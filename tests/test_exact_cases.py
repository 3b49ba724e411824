"""The exact-case constructors and budget checks of oracle/exact.py, on the CPU.

* every case the bit-exact GPU tests use passes the budget check of its datapath;
* the float64 reference equals an fp32 evaluation of the kernels' own arithmetic bit for bit, in several summation
  orders (natural, k reversed, random k chunks): the premise that the fp32 result does not depend on the order;
* an over-budget case is rejected.
"""
import numpy as np
import pytest

from exact_util import assert_fp16_bits_equal
from oracle import exact as ex

ORDERS = ['natural', 'reversed', 'chunks']


def test_gpu_cases_pass_their_budgets():
    from test_gpu_exact import exact_cases, pass_cases
    from test_gpu_exact_tc import tc_case, tc_cases
    n = 0
    for args in tc_cases():
        ex.check_mma(tc_case(*args))
        n += 1
    for c, checks in exact_cases():
        for chk in checks:
            chk(c)
        n += 1
    for X, F in pass_cases():
        ex.check_pass(X, F)
        n += 1
    assert n > 100


@pytest.mark.parametrize('bits', [2, 3, 4])
@pytest.mark.parametrize('symmetric', [True, False])
@pytest.mark.parametrize('K', [128, 640, 11008])
def test_mma_arithmetic_is_order_independent(bits, symmetric, K):
    c = ex.make_gemm_case(bits, 48, K, 6, symmetric=symmetric, bias=True, xmax=ex.gemm_xmax(bits, K, symmetric),
                          seed=bits + K)
    bits_used = ex.check_mma(c)
    want = ex.to_fp16(ex.gemm_exact(c))
    for order in ORDERS:
        assert_fp16_bits_equal(ex.gemm_f32_mma(c, order, seed=K), want, f'mma fp32 {order}')
    if K == 11008:
        assert bits_used['epilogue'] > 20          # the case uses most of the fp32 significand
        # the fp16 rounding is not trivial: most exact outputs need more than fp16's 11 significant bits
        assert np.mean(ex.gemm_exact(c) != want.astype(np.float64)) > 0.3


@pytest.mark.parametrize('bits', [2, 3, 4])
@pytest.mark.parametrize('K', [1024, 11008])
def test_qgemv_fp16_arithmetic_is_order_independent(bits, K):
    from test_gpu_exact import gv16_case
    c = gv16_case(bits, 40, K, 8, False)
    want = ex.to_fp16(ex.gemm_exact(c))
    for order in ORDERS:
        assert_fp16_bits_equal(ex.gemm_f32_gv16(c, order, seed=K), want, f'qgemv fp16 fp32 {order}')


@pytest.mark.parametrize('p,nblk,strided', [(16, 8, True), (43, 4, False), (688, 2, False)])
def test_pass_arithmetic_is_order_independent(p, nblk, strided):
    X, F = ex.make_pass_case(p, nblk, False, 5, xmax=32, seed=p)
    ex.check_pass(X, F)
    from oracle import butterfly as obf
    want = ex.to_fp16(obf.apply_pass(X.astype(np.float64), F.astype(np.float64), p, nblk, strided))
    for order in ORDERS:
        assert_fp16_bits_equal(ex.pass_f32(X, F, p, nblk, strided, order, seed=p), want, f'pass fp32 {order}')


def test_i8_limbs_reassemble_the_tokens():
    c = ex.make_gemm_case(2, 16, 1024, 5, symmetric=False, bias=False, xmax=16, seed=3, rows=('zero',),
                          pow2_amax=(5, 6))
    amax, q, (hi, mid, lo) = ex.i8_limbs(c.X)
    assert np.array_equal(65536 * hi + 256 * mid + lo, q)
    assert np.abs(hi).max() <= 64 and not mid.any() and not lo.any()
    assert amax[0] == 0 and not q[0].any()
    ex.check_i8(c)


def test_over_budget_cases_are_rejected():
    # 4-bit, K = 11008, all +64 token: (2^4 - 1) 11008 x 64 2 > 2^24 in the asymmetric epilogue
    c = ex.make_gemm_case(4, 16, 11008, 3, symmetric=False, bias=False, xmax=64, seed=1)
    with pytest.raises(ex.BudgetError):
        ex.check_mma(c)
    # the offset-free fp16 path has a far smaller budget at 4 bits: an all +16 token of 11008 is too much
    c = ex.make_gemm_case(4, 16, 11008, 3, symmetric=False, bias=False, xmax=16, seed=2)
    ex.check_mma(c)
    with pytest.raises(ex.BudgetError):
        ex.check_gv16(c)
    # int8 path: a token whose amax is not a power of two, and limb sums beyond 2^24
    c = ex.make_gemm_case(2, 16, 1024, 2, symmetric=False, bias=False, xmax=16, seed=3, rows=())
    c.X[0, 0] = 48
    c.X[0, 1:] = np.clip(c.X[0, 1:], -16, 16)
    with pytest.raises(ex.BudgetError, match='power-of-two'):
        ex.check_i8(c)
    c = ex.make_gemm_case(4, 16, 4096, 2, symmetric=False, bias=False, xmax=64, seed=4, rows=('max',),
                          pow2_amax=(5, 6))
    with pytest.raises(ex.BudgetError, match='limb'):
        ex.check_i8(c)
    # passes: factor entries off the 1/64 grid, and p max|x| 64 > 2^24
    X, F = ex.make_pass_case(16, 4, False, 3, xmax=8, seed=5)
    F[0, 0, 0] = np.float16(1 / 128)
    with pytest.raises(ex.BudgetError):
        ex.check_pass(X, F)
    X, F = ex.make_pass_case(688, 1, False, 2, xmax=64, seed=6)
    X[0] = 1024
    with pytest.raises(ex.BudgetError):
        ex.check_pass(X, F)
