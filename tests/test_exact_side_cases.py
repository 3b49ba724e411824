"""The whole-side cases of oracle/exact_side.py, on the CPU.

* every case tests/test_gpu_exact_side.py runs passes its budgets on the routes it is evaluated on;
* each route's float64 oracle equals an fp32 evaluation of that route's arithmetic bit for bit, in several summation
  orders (natural, reversed, random chunks);
* an over-budget case is rejected;
* the two-pass and one-launch oracles differ on a clear fraction of outputs, so the one-launch test can tell the two
  kernels apart (the fp16 rounding of the intermediate is not trivial).
"""
import numpy as np
import pytest

from exact_util import assert_fp16_bits_equal
from oracle import exact_side as es

ORDERS = ['natural', 'reversed', 'chunks']
ROUTES = [('two_pass', 'two_pass'), ('side_fewtok', 'side_fewtok'), ('side_fewtok', 'two_pass')]


def test_gpu_cases_pass_their_budgets():
    from test_gpu_exact_side import side_cases
    n = 0
    for c, routes in side_cases():
        for r in routes:
            es.check_case(c, *r)
        n += 1
    assert n > 120


@pytest.mark.parametrize('family,K,N,M,geometry', [('A', 2048, 768, 5, None), ('A', 768, 2048, 3, None),
                                                   ('B', 2048, 2048, 7, None), ('A', 2048, 1024, 2, 'hand'),
                                                   ('B', 768, 2048, 4, None)])
def test_route_oracles_equal_fp32_simulation(family, K, N, M, geometry):
    from test_gpu_exact_side import HAND_64x32
    c = es.fit_case(family, K, N, M, routes=ROUTES[:2], seed=K + N + M,
                    v_geometry=HAND_64x32 if geometry else None)
    for r in ROUTES:
        want = es.forward(c, *r)[0]
        for order in ORDERS:
            assert_fp16_bits_equal(es.simulate_f32(c, *r, order, seed=M), want, f'{family} {r} {order}')


def test_over_budget_cases_are_rejected():
    c = es.make_case('A', 2048, 2048, 4, seed=1, xmax=64, v_kind=('dense', 64), u_kind=('dense', 64))
    with pytest.raises(es.BudgetError):
        es.check_case(c)
    c = es.make_case('B', 4096, 4096, 4, seed=1, xmax=2048)
    with pytest.raises(es.BudgetError):
        es.check_case(c)


@pytest.mark.parametrize('family', ['A', 'B'])
def test_intermediate_rounding_is_not_trivial(family):
    """side_fewtok keeps the intermediate in fp32: on these cases that changes a clear fraction of the outputs (on
    the N side: family A keeps x2 coarse for the GEMM, so its K side rounds nothing)."""
    c = es.fit_case(family, 2048, 2048, 4, routes=ROUTES[:2], seed=11)
    y0 = es.forward(c, 'two_pass', 'two_pass')[0]
    y1 = es.forward(c, 'side_fewtok', 'side_fewtok')[0]
    assert np.mean(y0.view(np.uint16) != y1.view(np.uint16)) > 0.05


def test_selection_codes_cover_every_column():
    for (K, N) in [(4096, 11008), (11008, 4096), (2048, 2048)]:
        c = es.make_case('A', K, N, 1, seed=K + N)
        assert np.all(c.codes.sum(0) >= 1) and np.all(c.codes.sum(1) >= 1)
        assert c.codes.max() == 1


def test_route_plan_matches_the_forward():
    """plan() mirrors quip_qlinear_forward's choices on the shapes of the GPU file."""
    c = es.make_case('A', 4096, 11008, 2, seed=0)
    assert es.plan(c, dict(side_fewtok=1)) == dict(v='side_fewtok', u='side_fewtok', launches=3)
    c = es.make_case('A', 4096, 11008, 3, seed=0)
    assert es.plan(c, dict(side_fewtok=1))['u'] == 'two_pass'            # 11008 at 3 tokens exceeds shared memory
    c = es.make_case('A', 4096, 4096, 33, seed=0)
    assert es.plan(c, {}) == dict(v='side_fused', u='side_fused', launches=3)
    assert es.plan(c, dict(side_fused=0)) == dict(v='two_pass', u='two_pass', launches=8)
    c = es.make_case('A', 8192, 1024, 33, seed=0, perm=False, scale=None, bias=False)
    assert es.plan(c, {}) == dict(v='two_pass', u='two_pass', launches=6)   # 32 x 32 blocks: no one-kernel side
    c = es.make_case('A', 2048, 2048, 33, seed=0, v_geometry=[(64, 32, True), (32, 64, False)])
    assert es.side_fused_ok(c.vp, 2048) and c.vp[0].p == 64
