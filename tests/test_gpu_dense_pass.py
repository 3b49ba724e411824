"""The wgmma dense pass at 256-token tiles (qgemm_tc_kernel<2, W, true, 2>) against the 128-token kernel.

At both tile shapes every output element sees the same wgmma k16 steps in the same order, fp32 accumulation and one
fp16 rounding; only the tile's token count and column width differ.  So on any input the two must agree bit for bit.
The shapes reach every instantiated column width (96, 112, 128, 144, 152, 160, 176), ragged M (300, 2047), more tiles
than two waves with K / 64 not a multiple of the 3-stage ring (4096 tokens), and the shared (Kronecker) factor.  The
exactly representable cases of oracle/exact.py check the 256-token kernel against fp16(exact result) on its own, and
the default route is checked to pick the 256-token kernel at the benchmark's shape.
"""
import ctypes as C

import pytest
import torch

from exact_util import SMS, assert_fp16_bits_equal
from oracle import exact as ex
from test_gpu_exact import PASS_XMAX, _pass_exact_dev

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'

# (p, nblk, M, shared)
RANDOM_CASES = [
    (688, 16, 2048, False), (688, 16, 300, False), (688, 16, 2047, False), (688, 16, 4096, False),   # 7B down / gate, up
    (224, 32, 300, False), (128, 8, 129, True), (96, 4, 64, False),          # test_gpu_tcgen05 big-block shapes
    (688, 16, 2048, True),                                                   # shared (Kronecker) factor
    (144, 16, 300, False), (448, 8, 600, False), (160, 8, 257, True),        # widths 144, 3 x 152, 160
]
EXACT_CASES = [(688, 16, 2048, False), (688, 4, 300, True), (224, 32, 300, False), (96, 32, 300, False),
               (448, 8, 600, False), (144, 8, 257, False), (160, 8, 129, True), (128, 64, 300, True)]


def dense_cols(p):
    """Factor columns per 256-token tile (qgemm_tc.cu dense_cols)."""
    t = -(-p // 184)
    return 8 * -(-p // (8 * t))


@pytest.fixture
def dense_tile():
    from quip_b200 import _lib
    lib = _lib.load()

    def set_tile(tokens):
        _lib.check(lib.quip_config(b'dense_tile', tokens))
    yield set_tile
    set_tile(0)


def run_pass_dev(x, f, p, nblk):
    """One contiguous block-diagonal pass on the tensor cores (impl 2) on device tensors."""
    from quip_b200 import _lib
    lib = _lib.load()
    out = torch.empty_like(x)
    ps = _lib.QuipPass(p=p, nblk=nblk, strided=0, shared=int(f.shape[0] == 1 and nblk > 1), factors=f.data_ptr())
    _lib.check(lib.quip_rot_pass(C.byref(ps), _lib.ptr(x), _lib.ptr(out), x.shape[0], p * nblk, 2,
                                 C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    return out


def random_case(p, nblk, M, shared, seed):
    g = torch.Generator(device=DEV).manual_seed(seed)
    x = torch.randn(M, p * nblk, device=DEV, generator=g).half()
    f = (torch.randn(1 if shared else nblk, p, p, device=DEV, generator=g) / p ** 0.5).half().contiguous()
    return x, f


@pytest.mark.parametrize('p,nblk,M,shared', RANDOM_CASES)
def test_256_tokens_equal_128_tokens_bit_for_bit(dense_tile, p, nblk, M, shared):
    x, f = random_case(p, nblk, M, shared, seed=p + nblk + M)
    dense_tile(128)
    want = run_pass_dev(x, f, p, nblk)
    dense_tile(256)
    got = run_pass_dev(x, f, p, nblk)
    assert torch.isfinite(want.float()).all()
    diff = (got.view(torch.int16) != want.view(torch.int16))
    assert not diff.any(), f'p={p} nblk={nblk} M={M} shared={shared}: {int(diff.sum())} elements differ'


@pytest.mark.parametrize('p,nblk,M,shared', EXACT_CASES)
def test_256_tokens_bit_exact(dense_tile, p, nblk, M, shared):
    X, F = ex.make_pass_case(p, nblk, shared, M, xmax=PASS_XMAX, seed=p * 1000 + nblk + M)
    ex.check_pass(X, F)
    dense_tile(256)
    got = run_pass_dev(torch.from_numpy(X).to(DEV), torch.from_numpy(F).to(DEV).contiguous(), p, nblk)
    assert_fp16_bits_equal(got.cpu().numpy(), _pass_exact_dev(X, F, p, nblk, False),
                           f'dense pass 256 tokens p={p} nblk={nblk} M={M} shared={shared}')


def test_default_route_by_shape(dense_tile):
    """The 688-wide pass of the benchmark (2048 tokens) runs 256 x 176 tiles; at 300 tokens they would not fill the
    SMs (4 x 2 x 16 = 128 tiles), so the 128-token kernel runs."""
    from torch.profiler import ProfilerActivity, profile
    assert dense_cols(688) == 176 and 4 * 2 * 16 < SMS <= 4 * 8 * 16
    dense_tile(0)
    for M, want in ((2048, 'qgemm_tc_kernel<2, 176, true, 2>'), (300, 'qgemm_tc_kernel<2, 128, true, 1>')):
        x, f = random_case(688, 16, M, False, seed=M)
        run_pass_dev(x, f, 688, 16)
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            run_pass_dev(x, f, 688, 16)
        names = [e.name for e in prof.events() if 'qgemm_tc_kernel' in e.name]
        assert names and all(want in n for n in names), (M, names)
