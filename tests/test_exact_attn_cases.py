"""The exact decode-attention cases of oracle/exact_attn.py, on the CPU.

* every case the bit-exact GPU tests use passes its budget, and the grid cases launch all 32 instantiations of the split
  kernel at both chunk sizes;
* an fp32 restatement of the kernel's algorithm (oracle/exact_attn.simulate) equals the reference bit for bit at both
  chunk sizes and in any summation order;
* off fp16 ties the reference equals fp16 of the float64 oracles (kvfp8.attention, test_gpu_generate._reference);
* each plausible kernel defect changes the result on a named case;
* over-budget cases are rejected.
"""
import dataclasses
import functools

import numpy as np
import pytest
import torch

from oracle import exact_attn as ea
from oracle.exact import BudgetError

from test_gpu_exact_attn import GRID, MAX_LENS, NKV, cases, grid_case
from test_gpu_generate import _chunk, _reference


@functools.lru_cache(maxsize=None)
def _grid(fp8, hd, G, chunk, max_len):
    return grid_case(fp8, hd, G, chunk, max_len)


def _bits(a):
    return np.ascontiguousarray(a, np.float16).view(np.uint16)


def _changed(got, want):
    """Outputs whose values differ (NaN equals NaN; +0 equals -0, whose sign a float64 sum leaves to chance)."""
    return ~((got == want) | (np.isnan(got) & np.isnan(want)))


def test_gpu_cases_pass_their_budgets():
    n = 0
    for name, make in cases():
        try:
            ea.check_budget(make())
        except BudgetError as e:
            raise AssertionError(f'{name}: {e}') from e
        n += 1
    assert n > 200


def test_grid_cases_cover_every_instantiation_at_both_chunks():
    """(cache dtype, head_dim, G, chunk) of the kernel launch each grid case makes: all 2 x 2 x 8 x 2."""
    seen = set()
    for fp8, hd, G in GRID:
        for chunk in (64, 128):
            for max_len in MAX_LENS:
                c = _grid(fp8, hd, G, chunk, max_len)
                B, nh, nkv, hd_, max_len_ = c.shape
                seen.add((c.fp8, hd_, nh // nkv, _chunk(B, nkv, max_len_)))
    assert seen == {(f, hd, G, ch) for f in (False, True) for hd in (64, 128) for G in range(1, 9) for ch in (64, 128)}


SIM_CASES = [(False, 64, 3, 64, 424), (False, 128, 8, 64, 37), (True, 64, 3, 64, 424), (True, 128, 5, 64, 424),
             (True, 64, 1, 64, 1), (False, 128, 2, 128, 424)]


@pytest.mark.parametrize('spec', SIM_CASES, ids=[str(s) for s in SIM_CASES])
def test_fp32_restatement_equals_the_reference(spec):
    c = _grid(*spec)
    want, _ = ea.reference(c)
    for chunk in (64, 128):
        for order in ('natural', 'reversed', 'random'):
            got = ea.simulate(c, chunk=chunk, order=order, seed=chunk)
            assert np.array_equal(_bits(got), _bits(want)), (spec, chunk, order)


def test_reference_equals_the_float64_oracles_off_ties():
    """fp16 of float64 softmax attention equals the reference wherever the fp32 quotient is not an fp16 midpoint; the
    cases do contain midpoints (the 'tie' heads), where the two may differ."""
    from oracle import kvfp8
    ties = 0
    for fp8, hd, G in GRID:
        if G not in (1, 3, 8):
            continue
        c = _grid(fp8, hd, G, 64, MAX_LENS[-1])
        want, nt = ea.reference(c)
        ties += nt
        t = {k: torch.from_numpy(np.ascontiguousarray(v)) for k, v in
             dict(q=c.q, kn=c.k_new, vn=c.v_new, kc=c.k_cache, vc=c.v_cache, pos=c.positions).items()}
        if fp8:
            kc, vc = t['kc'].view(torch.float8_e4m3fn), t['vc'].view(torch.float8_e4m3fn)
            f64 = kvfp8.attention(t['q'], t['kn'], t['vn'], kc, vc, torch.from_numpy(c.k_scale),
                                  torch.from_numpy(c.v_scale), t['pos'], c.scale)
        else:
            f64 = _reference(t['q'], t['kn'], t['vn'], t['kc'], t['vc'], t['pos'], c.scale)
        f64 = f64.numpy().astype(np.float16)
        O, L = ea.exact_sums(c, np.arange(len(c.positions)))
        tie = ea.is_fp16_tie(O.astype(np.float32) / L.astype(np.float32)[..., None])
        same = f64 == want                      # as values: a float64 sum leaves the sign of an exact zero to chance
        assert same[~tie].all(), (fp8, hd, G, np.argwhere(~same & ~tie)[:3])
    assert ties >= 20, ties


# mutation -> the grid case (fp8, hd, G, chunk, max_len) that shows it
MUTATION_CASES = {
    'range_short': (False, 64, 3, 64, 424),          # attend over 0 .. pos - 1
    'range_long': (False, 64, 3, 64, 424),           # 0 .. pos + 1
    'cache_at_pos': (False, 64, 3, 64, 424),         # the cache's slot pos instead of k_new / v_new
    'gqa_mod': (False, 64, 3, 64, 424),              # kv head h % nkv instead of h // G
    'combine_short': (False, 64, 3, 64, 424),        # one chunk too few in the combine
    'rcp': (False, 64, 5, 64, 424),                  # O * fp32(1 / L) instead of O / L
    'f64': (False, 64, 5, 64, 424),                  # float64 softmax rounded once to fp16
    'ks_prev': (True, 64, 3, 64, 424),               # the k scale of slot j - 1
    'ks_next': (True, 64, 3, 64, 424),
    'vs_prev': (True, 64, 3, 64, 424),
    'vs_next': (True, 64, 3, 64, 424),
    'l_sv': (True, 64, 3, 64, 424),                  # l accumulates p * s_v instead of p
}


def test_every_mutation_has_a_case():
    assert set(MUTATION_CASES) == set(ea.MUTATIONS)


@pytest.mark.parametrize('mutation', list(MUTATION_CASES))
def test_mutation_changes_the_result(mutation):
    spec = MUTATION_CASES[mutation]
    c = _grid(*spec)
    want, _ = ea.reference(c)
    got = ea.simulate(c, mutation=mutation)
    assert _changed(got, want).any(), f'{mutation} not caught by grid case {spec}'


def test_rcp_and_f64_mutations_meet_ties_only():
    """The reciprocal multiply and the float64 softmax differ from the reference only where the fp32 quotient is an
    fp16 midpoint: a tie, which round to nearest even resolves."""
    c = _grid(*MUTATION_CASES['rcp'])
    want, ties = ea.reference(c)
    assert ties > 0
    O, L = ea.exact_sums(c, np.arange(len(c.positions)))
    tie = ea.is_fp16_tie(O.astype(np.float32) / L.astype(np.float32)[..., None])
    for m in ('rcp', 'f64'):
        diff = _changed(ea.simulate(c, mutation=m), want)
        assert diff.any() and not (diff & ~tie).any(), m


def test_over_budget_cases_are_rejected():
    spec = (False, 64, 3, 64, 424)
    # a score scale so small that the selected and the other slots score within DELTA of each other
    c = _grid(*spec)
    small = dataclasses.replace(c, scale=2.0 ** -12)
    with pytest.raises(BudgetError, match='score gap'):
        ea.check_budget(small)
    # one selected slot of a multi-slot head scores a different value
    c = ea.make_case(False, 64, 3, NKV, 424, c.positions, 64, seed=2)
    b, h = next((b, h) for b in range(len(c.positions)) for h in range(c.q.shape[1])
                if c.kinds[b][h] == 'rand7' and c.sel[b, h].sum() == 7)
    j = int(np.nonzero(c.sel[b, h])[0][0])
    d = int(np.nonzero(c.q[b, h])[0][0])
    if j == int(c.positions[b]):
        c.k_new[b, h // c.G, d] *= 2
    else:
        c.k_cache[b, h // c.G, j, d] *= 2
    with pytest.raises(BudgetError, match='maximum bit for bit'):
        ea.check_budget(c)
    # sums too wide: a dimension of magnitude 2^15 on the 1/8 grid over every slot of a 424-slot row
    c = ea.make_case(False, 64, 3, NKV, 424, c.positions, 64, seed=3)
    c.v_cache[:, :, :, 7] = 2.0 ** 15
    c.v_new[:, :, 7] = 2.0 ** 15
    with pytest.raises(BudgetError, match='sum of V'):
        ea.check_budget(c)
    # e4m3: the same case with an appended V scale so fine that a slot's products leave no room
    c = ea.make_case(True, 64, 3, NKV, 424, c.positions, 64, seed=4)
    c.v_scale[:, :, 0] = 2.0 ** -20
    with pytest.raises(BudgetError, match='sum of V'):
        ea.check_budget(c)
