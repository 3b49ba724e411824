"""The 2-bit wgmma packed GEMM at 256-row weight tiles (qgemm_tc_kernel<2, 128, false, 2>) against the 128-row kernel.

Both tile heights give every output element the same wgmma k16 steps in the same order and the same epilogue
arithmetic, so on any input they must agree bit for bit.  The shapes reach ragged N at 256 rows (144 = 9 row blocks,
4224 = 16.5 tiles), ragged M, one k super-block (K = 128), K = 11008, and more than 2 x 132 tiles with K / 64 not a
multiple of the 7-stage ring, so CTAs start tiles at different ring slots and phases.  The exactly representable cases
of oracle/exact.py check the 256-row kernel against fp16(exact result) on its own, and the default route is checked to
pick the 256-row kernel at the benchmark's shapes.
"""
import pytest
import torch

from exact_util import SMS, assert_fp16_bits_equal
from oracle import exact as ex

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
RING_256 = 7            # stages of the 2-bit 256-row ring at BN = 128: (227 KB - 36 KB epilogue) // 24 KB

# (N, K, M)
RANDOM_SHAPES = [
    (4096, 4096, 2048), (11008, 4096, 2048), (4096, 11008, 2048),    # the benchmark's GEMMs
    (144, 4096, 300), (4224, 4096, 300),                             # ragged N at 256 rows
    (4096, 4096, 65), (11008, 4096, 2125),                           # ragged M
    (4096, 128, 2048), (144, 11008, 129),                            # one super-block, K = 11008
    (4096, 11008, 2125),                                             # 272 tiles, K/64 = 172 = 4 mod 7
]


def tiles_256(N, M):
    return -(-N // 256) * -(-M // 128)


@pytest.fixture
def tc_rows():
    from quip_b200 import _lib
    lib = _lib.load()

    def set_rows(rows):
        _lib.check(lib.quip_config(b'tc_rows', rows))
    yield set_rows
    set_rows(0)


def random_case(N, K, M, symmetric, bias, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    codes = torch.randint(0, 4, (N, K), dtype=torch.uint8, device=DEV, generator=g)
    scales = torch.rand(N, device=DEV, generator=g) * 0.02 + 0.001
    zeros = scales * 1.5 + (torch.rand(N, device=DEV, generator=g) - 0.5) * 0.01
    x = torch.randn(M, K, device=DEV, generator=g).half()
    b = (torch.randn(N, device=DEV, generator=g) * 0.5).half() if bias else None
    return codes, scales, zeros, x, b


def run(codes, scales, zeros, x, b, symmetric):
    from gpu_util import run_qgemm_dev
    return run_qgemm_dev(codes, scales, zeros, 2, x, path=2, bias=b, symmetric=symmetric)


def test_shapes_reach_the_cases():
    assert tiles_256(4096, 2125) > 2 * SMS and (11008 // 64) % RING_256 != 0
    assert (4224 // 256) * 256 != 4224 and 144 < 256
    for N, K in [(4096, 4096), (11008, 4096), (4096, 11008)]:     # the benchmark's shapes route to 256 rows
        assert tiles_256(N, 2048) >= SMS


@pytest.mark.parametrize('symmetric', [True, False])
@pytest.mark.parametrize('bias', [True, False])
def test_256_rows_equal_128_rows_bit_for_bit(tc_rows, symmetric, bias):
    for (N, K, M) in RANDOM_SHAPES:
        codes, scales, zeros, x, b = random_case(N, K, M, symmetric, bias, seed=N * 31 + K * 7 + M + int(bias))
        tc_rows(128)
        z128 = run(codes, scales, zeros, x, b, symmetric)
        tc_rows(256)
        z256 = run(codes, scales, zeros, x, b, symmetric)
        assert not torch.isnan(z256).any(), (N, K, M)
        if not torch.equal(z128.view(torch.int16), z256.view(torch.int16)):
            diff = (z128.view(torch.int16) != z256.view(torch.int16)).nonzero()
            m, n = diff[0].tolist()
            pytest.fail(f'N={N} K={K} M={M} sym={symmetric} bias={bias}: {diff.shape[0]} outputs differ, first '
                        f'(m={m}, n={n}: tile row {n % 256}, token {m % 128}) 128-row {z128[m, n].item()} vs '
                        f'256-row {z256[m, n].item()}')
        del codes, x, z128, z256
        torch.cuda.empty_cache()


def test_default_route_is_256_rows_at_the_benchmark_shapes(tc_rows):
    for (N, K) in [(4096, 4096), (11008, 4096), (4096, 11008)]:
        codes, scales, zeros, x, b = random_case(N, K, 2048, False, False, seed=N + K)
        tc_rows(0)
        z0 = run(codes, scales, zeros, x, b, False)
        tc_rows(256)
        z256 = run(codes, scales, zeros, x, b, False)
        assert torch.equal(z0.view(torch.int16), z256.view(torch.int16)), (N, K)


EXACT_SHAPES = [(11008, 4096, 300), (144, 11008, 65), (4224, 640, 129), (4096, 11008, 2048 + 77)]


@pytest.mark.parametrize('symmetric', [True, False])
@pytest.mark.parametrize('bias', [True, False])
def test_256_rows_bit_exact(tc_rows, symmetric, bias):
    from gpu_util import run_qgemm
    tc_rows(256)
    for (N, K, M) in EXACT_SHAPES:
        xmax = ex.gemm_xmax(2, K, symmetric)
        c = ex.make_gemm_case(2, N, K, M, symmetric=symmetric, bias=bias, xmax=xmax,
                              seed=2 * 1000003 + N * 7 + K * 3 + M + 2 * int(symmetric) + int(bias))
        ex.check_mma(c)
        z, _ = run_qgemm(c.codes, c.scales, c.zeros, 2, c.X, path=2, bias=c.bias, symmetric=symmetric)
        want = ex.gemm_exact_torch(c, 'cuda').float().half().cpu().numpy()
        assert_fp16_bits_equal(z, want, f'qgemm_tc 256 rows N={N} K={K} M={M} sym={symmetric} bias={bias} '
                                         f'tiles={tiles_256(N, M)}', bn=128)
        torch.cuda.empty_cache()
