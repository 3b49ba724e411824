"""The wgmma packed GEMM (quip_qgemm path 2, qgemm_tc_kernel<BITS, BN, false>) on exactly representable inputs,
compared bit for bit with fp16(exact result) (oracle/exact.py; own file: see tests/test_gpu_kernels.py).

The fp32 accumulators hold the exact value in any order (check_mma proves it per case), so the output does not
depend on the tile schedule, the ring slot a tile starts at or the order of the wgmma: any dropped, repeated or
misplaced term, stale fragment or wrong epilogue rounding shows as a differing fp16 bit pattern.  The shapes reach
  * BN = 64 (M <= 64) and BN = 128 (M > 64) tiles, ragged M and ragged N (N = 144, 11008 = 86 x 128);
  * one k super-block (K = 128), an odd number of them (K = 640), K = 4096 and K = 11008;
  * more tiles than CTAs at both BN, and for every bits value a case with >= 3 x 132 tiles whose K/64 stages are not
    a multiple of the ring depth (9 / 8 / 7 at BN = 128), so CTAs walk several tiles that start at different ring
    slots and phases.
"""
import pytest
import torch

from exact_util import SMS, assert_fp16_bits_equal, tc_bn, tc_stages, tc_tiles
from oracle import exact as ex

pytestmark = pytest.mark.gpu

# (N, K, M), and the least number of tiles each must produce
TC_SHAPES = [
    ((144, 128, 33), 2),           # BN 64: one super-block, ragged N
    ((256, 640, 64), 2),           # BN 64: odd number of super-blocks
    ((28672, 640, 64), SMS + 1),   # BN 64: 224 tiles on 132 CTAs
    ((11008, 4096, 300), SMS + 1), # BN 128: N = 86 x 128, 258 tiles, ragged M
    ((144, 11008, 65), 2),         # BN 128: ragged N, K = 11008, one token beyond the BN = 64 tile
    ((4096, 11008, 2048 + 77), 3 * SMS),   # BN 128: 544 tiles; K/64 = 172 = 1 / 4 / 4 mod 9 / 8 / 7
]


def tc_case(bits, N, K, M, symmetric, bias):
    xmax = ex.gemm_xmax(bits, K, symmetric)
    return ex.make_gemm_case(bits, N, K, M, symmetric=symmetric, bias=bias, xmax=xmax,
                             seed=bits * 1000003 + N * 7 + K * 3 + M + 2 * int(symmetric) + int(bias))


def tc_cases():
    """Every case of this file, for the host-side budget test."""
    for bits in (2, 3, 4):
        for symmetric in (True, False):
            for bias in (True, False):
                for (N, K, M), _ in TC_SHAPES:
                    yield (bits, N, K, M, symmetric, bias)


@pytest.mark.parametrize('bits', [2, 3, 4])
@pytest.mark.parametrize('symmetric', [True, False])
@pytest.mark.parametrize('bias', [True, False])
def test_wgmma_gemm_bit_exact(bits, symmetric, bias):
    from gpu_util import run_qgemm
    for (N, K, M), min_tiles in TC_SHAPES:
        bn = tc_bn(M)
        tiles = tc_tiles(N, M)
        assert tiles >= min_tiles, (N, K, M, tiles)
        if min_tiles >= 3 * SMS:
            assert (K // 64) % tc_stages(bits, bn) != 0, (bits, K, tc_stages(bits, bn))
        c = tc_case(bits, N, K, M, symmetric, bias)
        ex.check_mma(c)
        z, _ = run_qgemm(c.codes, c.scales, c.zeros, bits, c.X, path=2, bias=c.bias, symmetric=symmetric)
        want = ex.gemm_exact_torch(c, 'cuda').float().half().cpu().numpy()   # exact in fp32: one rounding
        assert_fp16_bits_equal(z, want, f'qgemm_tc bits={bits} N={N} K={K} M={M} sym={symmetric} bias={bias} '
                                         f'BN={bn} tiles={tiles}', bn=bn)
        torch.cuda.empty_cache()
