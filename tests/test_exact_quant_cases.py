"""The exact quantizer cases of oracle/exact_quant.py, on the CPU.

* every case the bit-exact GPU tests use passes its budget;
* the float64 references equal the fp32 torch loops (oracle/ldlq.py, quantize.ldlq_round with kernels=False) bit for
  bit, at block sizes that do and do not divide d, with and without greedy passes, and for LDLQ-RG;
* the cases can tell rounding rules and a dropped feedback term apart: mutations that change well under 0.2 % of the
  codes, and so pass a 99.8 % agreement bar, change codes here;
* over-budget cases are rejected.
"""
import numpy as np
import pytest
import torch

from oracle import exact_quant as eq
from oracle.exact import BudgetError

CPU_CASES = [(70, 96, 2), (70, 200, 3), (70, 300, 4)]


def test_gpu_cases_pass_their_budgets():
    from test_gpu_exact_quant import cases
    n = 0
    for name, run in cases():
        try:
            run()
        except BudgetError as e:
            raise AssertionError(f'{name}: {e}') from e
        n += 1
    assert n > 250


@pytest.mark.parametrize('m,d,bits', CPU_CASES)
@pytest.mark.parametrize('passes', [0, 1, 2])
def test_exact_reference_equals_the_torch_loops(m, d, bits, passes):
    from oracle import ldlq as oldlq
    from quip_b200 import quantize as qz
    c = eq.make_ldlq_case(m, d, bits, seed=d + m)
    w, H = torch.from_numpy(c.w).float(), torch.from_numpy(c.H).float()
    assert torch.equal(torch.linalg.cholesky(H), torch.from_numpy(c.C).float())       # the premise
    want = torch.from_numpy(eq.ldlq_exact(c, passes)[0]).float()
    assert torch.equal(oldlq.ldlq_round(w, H, bits, passes), want)
    for block in (128, 32, 40):
        assert torch.equal(qz.ldlq_round(w, H, bits, passes, block=block, kernels=False), want), block
    wr, Hr = (torch.from_numpy(a).float() for a in c.scrambled())
    want_rg = want[:, c.perm]
    assert torch.equal(oldlq.ldlq_rg_round(wr, Hr, bits, passes), want_rg)
    for block in (128, 40):
        assert torch.equal(qz.ldlq_rg_round(wr, Hr, bits, passes, block=block), want_rg), block


def test_ldlq_cases_have_distinct_ascending_diagonals():
    from test_gpu_exact_quant import E2E_CASES, e2e_case
    for (m, d, bits) in E2E_CASES + CPU_CASES:
        dg = np.diag(eq.make_ldlq_case(m, d, bits, seed=d + m).H)
        assert np.all(np.diff(dg) > 0)
        assert dg[-1] == 2.0 ** np.round(np.log2(dg[-1]))
    c = e2e_case(70, 1416, 2)
    assert np.array_equal(np.argsort(np.diag(c.scrambled()[1])), np.argsort(c.perm))


@pytest.mark.parametrize('m,d,bits', CPU_CASES + [(1000, 200, 2), (70, 1416, 2)])
def test_cases_tell_the_tie_rule_and_a_dropped_term_apart(m, d, bits):
    c = eq.make_ldlq_case(m, d, bits, seed=d + m)
    q, st = eq.ldlq_exact(c)
    s = st['ldlq']
    assert s['ties'] > 0 and s['clamp_lo'] > 0 and s['clamp_hi'] > 0, s
    # round half to even instead of floor(v + 1/2)
    assert not np.array_equal(eq.ldlq_exact(c, rnd=np.rint)[0], q)
    # one feedback term dropped: the last |L| = 1 entry (the largest row of C)
    L = c.L
    k, i = np.argwhere(np.abs(L) == 1)[-1]
    L[k, i] = 0
    dropped = eq.ldlq_exact(c, L=L)[0]
    assert np.count_nonzero(dropped != q) > 0


def test_greedy_block_cases_contain_half_even_ties():
    from test_gpu_exact_quant import CNTS, MS, greedy_block_case
    for cnt in CNTS:
        for m in MS:
            c = greedy_block_case(m, cnt)
            st = eq.greedy_block_exact(c)[2]
            assert st['ties'] > 0, (m, cnt)
    # the first column visited of a tied row: rint lands on the even neighbour, not on floor(arg + 1/2)
    c = greedy_block_case(64, 5)
    i, r = 4, np.arange(0, 64, 3)
    arg = c.wr[r, i] - (c.pre[r, i] + c.s[r] @ c.Hb[:, i]) / c.Hb[i, i]
    assert np.all(arg - np.floor(arg) == 0.5)
    assert np.array_equal(eq.greedy_block_exact(c)[0][r, i], np.rint(arg))


def test_hessian_cases_reach_the_chunk_budget():
    X = eq.make_hessian_case(256, 8, seed=0)
    X[2:] = X[0]                                        # 255 tokens at the maximum and one of granularity 2^e_i
    X[1] = X[0] / 256
    assert eq.check_hessian(X)['chunk'] > 23.99
    X1 = eq.make_hessian_case(2, 16, seed=1)
    assert not X1[1].any() and np.all(X1[0] > 0)


def test_over_budget_cases_are_rejected():
    c = eq.make_ldlq_case(20, 96, 2, seed=0)
    # L off the 1/16 grid: a non-dyadic entry, and a dyadic one so fine that gran(w) gran(L) leaves no room
    for bad in (1 / 3, 2.0 ** -22):
        L = c.L
        L[50, 10] = bad
        with pytest.raises(BudgetError, match='LDLQ feedback'):
            eq.ldlq_exact(c, L=L)
    # feedback sums above 2^24 x granularity: w of magnitude 2^21 on the 2^-4 grid
    big = eq.LdlqCase(c.bits, c.C, c.w + 2.0 ** 21, c.perm)
    with pytest.raises(BudgetError):
        eq.ldlq_exact(big)
    # greedy: pre too fine for its magnitude
    g = eq.make_greedy_block_case(8, 16, seed=0)
    g.pre[0, 3] = 2.0 ** -30
    with pytest.raises(BudgetError, match='greedy'):
        eq.greedy_block_exact(g)
    # Hessian: 256 tokens beyond |x| = 2^8 overflow the fp32 chunk; a prefill too fine for the float64 carry
    X = eq.make_hessian_case(256, 8, seed=0, xmax=512)
    X[2:] = X[0]
    X[1] = X[0] / 512
    with pytest.raises(BudgetError, match='chunk'):
        eq.check_hessian(X)
    X = eq.make_hessian_case(4, 8, seed=0)
    H0 = np.full((8, 8), 2.0 ** -60)
    H0[0, 0] = 2.0 ** 10
    with pytest.raises(BudgetError, match='carry'):
        eq.check_hessian(X, H0)
