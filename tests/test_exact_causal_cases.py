"""The exact multi-token cases of oracle/exact_causal.py, on the CPU.

* every case the bit-exact GPU tests use passes its budget; the grid cases launch all 32 instantiations of the extend
  kernel and all 32 of the prefill kernel, with query tiles that split a token's heads and diagonal blocks that start
  mid-tile;
* fp32 restatements of both kernels' algorithms (simulate_extend, simulate_prefill) equal the reference bit for bit in
  any summation order;
* off fp16 ties the reference equals fp16 of the float64 oracles of test_gpu_speculative and test_gpu_prefill_chunked;
* each plausible kernel defect changes the result on a named case;
* over-budget cases are rejected.
"""
import dataclasses
import functools

import numpy as np
import pytest
import torch

from oracle import exact_causal as ec
from oracle.exact import BudgetError

from test_gpu_exact_causal import EXTEND_T, GRID, PREFILL_T, cases, extend_case, extend_max_lens, prefill_case


@functools.lru_cache(maxsize=None)
def _ext(fp8, hd, G, T, max_len):
    return extend_case(fp8, hd, G, T, max_len)


@functools.lru_cache(maxsize=None)
def _pf(fp8, hd, G, T):
    return prefill_case(fp8, hd, G, T)


def _case(spec):
    return _ext(*spec[1:]) if spec[0] == 'extend' else _pf(*spec[1:])


def _bits(a):
    return np.ascontiguousarray(a, np.float16).view(np.uint16)


def _changed(got, want):
    """Outputs whose values differ (NaN equals NaN; +0 equals -0, whose sign a float64 sum leaves to chance)."""
    return ~((got == want) | (np.isnan(got) & np.isnan(want)))


def test_gpu_cases_pass_their_budgets():
    n = 0
    for name, make in cases():
        try:
            ec.check_budget(make())
        except BudgetError as e:
            raise AssertionError(f'{name}: {e}') from e
        n += 1
    assert n > 480


def _tiles(c):
    """(straddle, mid_diag) of a prefill case: a counted token whose G query rows lie in two 64-row tiles, and a tile
    whose first token's slot is not at a block start while a block edge lies inside the tile's slots."""
    B, T, nh, nkv, hd, max_len = c.shape
    G = c.G
    straddle = mid = False
    for b in range(B):
        n, p = c.count(b), int(c.positions[b])
        for i in range(n):
            straddle |= (i * G) // ec.TILE != (i * G + G - 1) // ec.TILE
        for t in range(-(-G * T // ec.TILE)):
            i_lo = t * ec.TILE // G
            if i_lo >= n:
                continue
            i_hi = min((min(t * ec.TILE + ec.TILE - 1, G * T - 1)) // G, n - 1)
            first, last = p + i_lo, p + i_hi
            mid |= first % ec.BLOCK != 0 and last // ec.BLOCK > first // ec.BLOCK
    return straddle, mid


def test_grid_cases_cover_every_instantiation_and_the_tile_edges():
    """(kernel, cache dtype, head_dim, G) of each grid case's launch: all 2 x 2 x 2 x 8; prefill cases where a token's
    heads straddle two query tiles (G = 3, 5, 6, 7) and where a diagonal block starts mid-tile."""
    seen, straddle, mid = set(), set(), set()
    for fp8, hd, G in GRID:
        for T in EXTEND_T:
            for max_len in extend_max_lens(T):
                c = _ext(fp8, hd, G, T, max_len)
                seen.add(('extend', c.fp8, c.shape[4], c.G))
        for T in PREFILL_T:
            c = _pf(fp8, hd, G, T)
            seen.add(('prefill', c.fp8, c.shape[4], c.G))
            s, m = _tiles(c)
            if s:
                straddle.add(G)
            if m:
                mid.add(G)
    assert seen == {(k, f, hd, G) for k in ('extend', 'prefill') for f in (False, True) for hd in (64, 128)
                    for G in range(1, 9)}
    assert {3, 5, 6, 7} <= straddle, straddle
    assert set(range(1, 9)) <= mid, mid
    s, _ = _tiles(_pf(False, 64, 3, 22))                    # T = 22 at G = 3: token 21 owns rows 63 .. 65
    assert s


SIM_CASES = [('extend', False, 64, 3, 5, 232), ('extend', True, 128, 8, 8, 232), ('extend', True, 64, 1, 2, 2),
             ('extend', False, 128, 5, 3, 232), ('prefill', False, 64, 3, 22), ('prefill', True, 64, 5, 22),
             ('prefill', True, 128, 2, 100), ('prefill', False, 128, 8, 7)]


@pytest.mark.parametrize('spec', SIM_CASES, ids=[str(s) for s in SIM_CASES])
def test_fp32_restatement_equals_the_reference(spec):
    c = _case(spec)
    want, _ = ec.reference(c)
    for order in ('natural', 'reversed', 'random'):
        got = ec.simulate(c, order=order, seed=len(order))
        assert np.array_equal(_bits(got), _bits(want)), (spec, order)


def _f64_oracle(c):
    """fp16 of the float64 oracle of the kernel's existing tests, over the caches as the call leaves them."""
    import test_gpu_prefill_chunked as tp
    import test_gpu_speculative as ts
    kc, vc, ks, vs = c.caches_after()
    t = torch.from_numpy
    kc, vc = t(kc), t(vc)
    if c.fp8:
        kc, vc, ks, vs = kc.view(torch.float8_e4m3fn), vc.view(torch.float8_e4m3fn), t(ks), t(vs)
    q, pos = t(c.q), t(c.positions)
    if c.kernel == 'extend':
        out = ts._reference(q, kc, vc, pos, c.scale, ks, vs)
    else:
        out = tp._reference(q, kc, vc, pos, t(c.counts), c.scale, ks, vs)
    return out.numpy().astype(np.float16)


def test_reference_equals_the_float64_oracles_off_ties():
    """fp16 of float64 softmax attention equals the reference wherever the fp32 quotient is not an fp16 midpoint; the
    cases do contain midpoints (the 'tie' heads), where the two may differ."""
    ties = 0
    specs = [('extend', fp8, hd, G, 5, 232) for fp8 in (False, True) for hd in (64, 128) for G in (1, 3, 8)]
    specs += [('prefill', fp8, hd, G, T) for fp8 in (False, True) for hd in (64, 128) for G in (1, 3, 8)
              for T in (7, 100)]
    for spec in specs:
        c = _case(spec)
        want, nt = ec.reference(c)
        ties += nt
        f64 = _f64_oracle(c)
        rows = np.array([b for b in range(len(c.positions)) if c.count(b) > 0])
        O, L = ec.exact_sums(c, rows)
        with np.errstate(invalid='ignore', divide='ignore'):
            tie = ec.is_fp16_tie(O.astype(np.float32) / L.astype(np.float32)[..., None])
        comp = (L > 0)[..., None]
        same = f64[rows] == want[rows]
        assert same[~tie & comp].all(), (spec, np.argwhere(~same & ~tie & comp)[:3])
    assert ties >= 20, ties


# mutation -> the case that shows it: ('extend', fp8, hd, G, T, max_len) or ('prefill', fp8, hd, G, T)
EXT = ('extend', False, 64, 3, 5, 232)
EXT8 = ('extend', True, 64, 3, 5, 232)
PF = ('prefill', False, 64, 3, 22)
PF8 = ('prefill', True, 64, 3, 100)
EXT_TIE = ('extend', False, 64, 5, 5, 232)         # cases with ties that rcp and f64 resolve the other way
PF_TIE = ('prefill', False, 64, 5, 22)
MUTATION_CASES = {
    'extend': {
        'mask_short': EXT,                  # token i sees up to pos + i - 1
        'mask_long': EXT,                   # up to pos + i + 1
        'mask_tile': EXT,                   # every token masked at the last token
        'token_of_row': EXT,                # query row r masked as token r % T instead of r / G
        'gqa_mod': EXT,                     # kv head h % nkv instead of h / G
        'stale_new': EXT,                   # the cache's old content at the new slots
        'ks_prev': EXT8, 'ks_next': EXT8, 'vs_prev': EXT8, 'vs_next': EXT8,   # the scale of slot j -+ 1
        'l_sv': EXT8,                       # l accumulates p s_v instead of p
        'combine_pos': EXT,                 # the combine's chunk count from pos, not pos + i
        'rcp': EXT_TIE,                     # O * fp32(1 / L) instead of O / L
        'f64': EXT_TIE,                     # float64 softmax rounded once to fp16
    },
    'prefill': {
        'mask_short': PF, 'mask_long': PF, 'mask_tile': PF, 'token_of_row': PF, 'gqa_mod': PF, 'stale_new': PF,
        'no_rescale': PF,                   # alpha taken as 1
        'c_stale': PF8,                     # f = alpha / sm, the last block's c forgotten
        'ks_prev': PF8, 'ks_next': PF8, 'vs_prev': PF8, 'vs_next': PF8, 'l_sv': PF8,
        'count_long': PF,                   # tokens past the count computed, not zeroed
        'rcp': PF_TIE, 'f64': PF_TIE,
    },
}


def test_every_mutation_has_a_case():
    assert set(MUTATION_CASES['extend']) == set(ec.EXTEND_MUTATIONS)
    assert set(MUTATION_CASES['prefill']) == set(ec.PREFILL_MUTATIONS)


@pytest.mark.parametrize('kernel,mutation', [(k, m) for k in MUTATION_CASES for m in MUTATION_CASES[k]])
def test_mutation_changes_the_result(kernel, mutation):
    spec = MUTATION_CASES[kernel][mutation]
    c = _case(spec)
    want, _ = ec.reference(c)
    got = ec.simulate(c, mutation=mutation)
    assert _changed(got, want).any(), f'{mutation} not caught by {spec}'


@pytest.mark.parametrize('kernel', ['extend', 'prefill'])
def test_rcp_and_f64_mutations_meet_ties_only(kernel):
    """The reciprocal multiply and the float64 softmax differ from the reference only where the fp32 quotient is an
    fp16 midpoint: a tie, which round to nearest even resolves."""
    c = _case(MUTATION_CASES[kernel]['rcp'])
    want, ties = ec.reference(c)
    assert ties > 0
    O, L = ec.exact_sums(c, np.arange(len(c.positions)))
    with np.errstate(invalid='ignore', divide='ignore'):
        tie = ec.is_fp16_tie(O.astype(np.float32) / L.astype(np.float32)[..., None])
    for m in ('rcp', 'f64'):
        diff = _changed(ec.simulate(c, mutation=m), want)
        assert diff.any() and not (diff & ~tie).any(), m


def test_over_budget_cases_are_rejected():
    c = _pf(False, 64, 3, 22)
    # a score scale so small that the selected and the other slots score within DELTA of each other
    with pytest.raises(BudgetError, match='score gap'):
        ec.check_budget(dataclasses.replace(c, scale=2.0 ** -12))
    # one selected old slot of a multi-slot head scores a different value
    c = _pf(False, 64, 3, 22)
    b, h, j = next((b, h, int(j)) for b in range(len(c.positions)) for h in range(c.q.shape[2])
                   if c.kinds[b][h] == 'rand7' for j in np.nonzero(c.sel[b, h])[0][:1] if j < c.positions[b])
    d = int(np.nonzero(c.q[b, :, h].any(0))[0][0])
    kc = c.k_cache.copy()
    kc[b, h // c.G, j, d] *= 2
    with pytest.raises(BudgetError, match='maximum bit for bit'):
        ec.check_budget(dataclasses.replace(c, k_cache=kc))
    # a new token's key (the appended value is what the budget reads, not the decoy) of a 'new' head
    b, h, i = next((b, h, i) for b in range(len(c.positions)) for h in range(c.q.shape[2]) for i in range(1, c.count(b))
                   if c.kinds[b][h] == 'new' and not c.zero[b, i, h])
    dd = int(np.nonzero(c.q[b, i, h])[0][0])
    kn = c.k_new.copy()
    kn[b, i, h // c.G, dd] *= 2
    with pytest.raises(BudgetError, match='maximum bit for bit'):
        ec.check_budget(dataclasses.replace(c, k_new=kn))
    # sums too wide: a dimension of magnitude 2^15 on the 1/8 grid over every slot
    vc, vn = c.v_cache.copy(), c.v_new.copy()
    vc[:, :, :, 7] = 2.0 ** 15
    vn[:, :, :, 7] = 2.0 ** 15
    with pytest.raises(BudgetError, match='sum of V'):
        ec.check_budget(dataclasses.replace(c, v_cache=vc, v_new=vn))
    # e4m3: an old V scale so fine that a slot's products leave no room
    c = _pf(True, 64, 3, 22)
    vs = c.v_scale.copy()
    vs[:, :, 0] = 2.0 ** -20
    with pytest.raises(BudgetError, match='sum of V|fp16 normal'):
        ec.check_budget(dataclasses.replace(c, v_scale=vs))
