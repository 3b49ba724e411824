"""Helpers of the bit-exact kernel tests (tests/test_gpu_exact*.py, tests/test_exact_cases.py)."""
import numpy as np

from oracle import exact as ex

TC_BM = 128
SMS = 132                                          # H100 SXM: one persistent GEMM CTA per SM


def sb_words(bits):
    return {2: 128, 3: 192, 4: 256}[bits]


def tc_bn(M):
    """Token tile of the wgmma GEMM (qgemm_tc.cu qgemm_tc): 128 above 64 tokens, else 64."""
    return 128 if M > 64 else 64


def tc_stages(bits, BN):
    """Ring depth of qgemm_tc_kernel<BITS, BN, false> (TcCfg in qgemm_tc.cu)."""
    stage = (TC_BM // 16) * sb_words(bits) * 4 + BN * 64 * 2
    epi = 2 * max(BN * 72, 64 * (BN + 8)) * 2
    return min((227 * 1024 - epi - 1024 - 256) // stage, 16)


def tc_tiles(N, M):
    return -(-N // TC_BM) * -(-M // tc_bn(M))


def fit_xmax(make, check, top=64):
    """The case of the largest power-of-two xmax <= top that passes `check` (make(xmax) -> case)."""
    x = top
    while True:
        c = make(x)
        try:
            check(c)
            return c
        except ex.BudgetError:
            if x == 1:
                raise
            x //= 2


def assert_fp16_bits_equal(got, want, what, bn=None):
    """Compare fp16 arrays bit for bit; on a mismatch report the count, the first (m, n) and, for the GEMM, its tile."""
    g = np.ascontiguousarray(got, np.float16).view(np.uint16)
    w = np.ascontiguousarray(want, np.float16).view(np.uint16)
    assert g.shape == w.shape, (what, g.shape, w.shape)
    bad = np.argwhere(g != w)
    if len(bad):
        m, n = (int(v) for v in bad[0])
        tile = f', tile (m // {bn}, n // 128) = ({m // bn}, {n // 128})' if bn else ''
        raise AssertionError(f'{what}: {len(bad)} of {g.size} outputs differ from fp16(exact); first at (m, n) = '
                             f'({m}, {n}){tile}: got {got[m, n]!r} want {want[m, n]!r}')
