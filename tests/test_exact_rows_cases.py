"""The exact vocabulary rows of oracle/exact_rows.py, on the CPU.

* every case's premise holds: values on the fp16 grid, every value other than a tie at least GAP below the maximum
  (after temperature, in fp32), and the tie counts and positions each case claims;
* the cases reach every edge of each kernel's split of the row that tests/test_gpu_exact_rows.py relies on;
* the exact rule equals the float64 oracles (oracle/loglik.py, topk_logprobs.py, beam.py, sampling.py) on every case,
  and no sampling case is ambiguous to oracle/sampling.py.
"""
import math

import numpy as np
import pytest
import torch

from oracle import exact_rows as er
from oracle.beam import candidates as beam_oracle
from oracle.loglik import token_logprobs as lp_oracle
from oracle.sampling import sample_row, uniform
from oracle.topk_logprobs import topk_row

from test_gpu_exact_rows import BEAM_V, BIG_V, ROW_V, TOP_N, lse_cases, sample_cases


def _ulps(a, b):
    a, b = np.float32(a), np.float32(b)
    return abs(int(a.view(np.int32)) - int(b.view(np.int32)))


def _premise(row, T=1.0):
    """Values on the grid; every finite value other than a tie at least GAP below the maximum after temperature."""
    assert er.on_grid(row.x), row.name
    if row.m == -np.inf:
        assert (row.x == -np.inf).all(), row.name
        return
    z = row.x.astype(np.float32) / np.float32(T)
    zm = np.float32(np.float32(row.m) / np.float32(T))
    other = np.isfinite(z) & (row.x != np.float16(row.m))
    assert (z[np.isfinite(z)] <= zm).all(), row.name
    assert ((z[other] - zm).astype(np.float32) <= -er.GAP).all(), row.name
    assert row.ties.size >= 1, row.name


@pytest.mark.parametrize('V', ROW_V + BEAM_V + BIG_V)
def test_lse_rows_hold_their_premise_and_claims(V):
    rows = lse_cases(V)
    buf, ld = er.layout(rows)
    assert ld >= V and ld % 8 == 1
    for r, row in enumerate(rows):
        _premise(row)
        assert row.mis == r % 8 and np.array_equal(buf[r * ld:r * ld + V], row.x)
        c = row.claims
        if 'lead_thread' in c:                       # thread j's first unit is -inf; a later one holds a tie
            us = er.units(V, row.mis, c['lead_thread'])
            assert (row.x[list(us[0])] == -np.inf).all() and row.x[c['lead_at']] == np.float16(row.m)
            assert any(c['lead_at'] in u for u in us[1:])
        else:                                        # no -inf leads a thread whose later units hold a tie
            for j in range(min(er.THREADS, V)):
                us = er.units(V, row.mis, j)
                if len(us) > 1 and (row.x[list(us[0])] == -np.inf).all() and row.m != -np.inf:
                    assert not any((row.x[list(u)] == np.float16(row.m)).any() for u in us[1:]), (row.name, j)
        for i in c.get('tie_at', ()):
            assert row.x[i] == np.float16(row.m)


def test_lse_rows_reach_every_edge_of_the_split():
    seen = set()
    for V in ROW_V:
        rows = lse_cases(V)
        if V >= 16:
            assert {r.mis for r in rows} == set(range(8)), V
        for row in rows:
            head, nvec, body_end = er.split(V, row.mis)
            t = set(row.ties.tolist())
            c = row.claims
            if 'lead_thread' in c:
                us = er.units(V, row.mis, c['lead_thread'])
                first = 'head' if len(us[0]) == 1 and us[0][0] < head else 'group'
                later = 'tail' if c['lead_at'] >= body_end else 'group'
                seen.add(('lead', first, later, 'max' if row.ties.size == 1 else 'ties'))
            if 'tie_at' in c:
                seen |= {('head', i < head) for i in t}
                seen |= {('tail',) for i in t if i >= body_end}
                seen |= {('last group',) for i in t if nvec and head + 8 * (nvec - 1) <= i < body_end}
                for k, side in ((nvec - er.THREADS - 1, 'pair'), (nvec - er.THREADS, 'single')):
                    if k >= 0 and t & set(range(head + 8 * k, head + 8 * k + 8)):
                        seen.add(('two loads', side))
    want = {('lead', 'head', 'group', 'max'), ('lead', 'head', 'group', 'ties'), ('lead', 'group', 'group', 'max'),
            ('lead', 'group', 'group', 'ties'), ('lead', 'head', 'tail', 'max'), ('head', True), ('head', False),
            ('tail',), ('last group',), ('two loads', 'pair'), ('two loads', 'single')}
    assert want <= seen, want - seen


def test_topk_rows_reach_both_tie_paths():
    """Rows with exactly TIE_CAP and TIE_CAP + 1 ties at the threshold key of n = 20 (collected, and scanned in
    segments), with keys above and below it that differ in the low byte only."""
    seen = set()
    for V in ROW_V:
        for row in lse_cases(V):
            if 'threshold_ties' in row.claims:
                lv = np.float16(row.claims['level'])
                k = er.topn(row, TOP_N)
                assert row.x[k[-1]] == lv and row.x[k[0]] == np.float16(row.m)
                above = np.unique(row.x[k[1:]][row.x[k[1:]] != lv])
                assert above.size == 1 and (above.view(np.uint16) >> 8) == (lv.view(np.uint16) >> 8)
                seen.add(int((row.x == lv).sum()))
    assert seen == {er.TIE_CAP, er.TIE_CAP + 1}


def test_beam_rows_hold_more_than_c_ties_at_the_c_th_key():
    over = 0
    for V in ROW_V:
        for row in lse_cases(V):
            if 'level' in row.claims and 'threshold_ties' not in row.claims:
                lv = np.float16(row.claims['level'])
                k = er.topn(row, 64)
                over += row.ties.size == 1 and row.x[k[-1]] == lv and int((row.x == lv).sum()) > 64
    assert over >= 10


@pytest.mark.parametrize('V', ROW_V + BEAM_V + BIG_V[:1])
def test_lse_rule_equals_the_float64_oracles(V):
    rows = lse_cases(V)
    big = V in BIG_V
    for r, row in enumerate(rows):
        n = row.ties.size
        L = er.fp32_logs(n if row.m != -np.inf else 0)[0]
        rng = np.random.default_rng(r)
        t = np.array([er.first_max(row), row.ties[-1], *rng.integers(0, V, 4), -1, V])
        want, gr = lp_oracle(np.repeat(row.x[None], t.size, 0), t)
        for j, tj in enumerate(t):
            got = er.logprob(row, tj, L)
            assert gr[j] == int(0 <= tj < V and tj == er.first_max(row)), (row.name, tj)
            if np.isnan(want[j]):
                assert np.isnan(got), (row.name, tj)
            elif n == 1:
                assert got == want[j], (row.name, tj)    # exactly x - m
            else:
                assert _ulps(got, want[j]) <= 1, (row.name, tj, got, want[j])
        if big:
            continue
        ids, vals = topk_row(row.x, TOP_N)
        assert np.array_equal(er.topn(row, TOP_N), ids[ids >= 0]), row.name
        for C in (1, 8, 64):
            score = np.float32(-1.0) - np.float32(0.25) * np.float32(r % 7)
            ws, wi = beam_oracle(torch.from_numpy(row.x[None]), torch.tensor([score]), 3, C)
            s, i = er.beam(row, score, C, L, 0)
            assert np.array_equal(i, wi[0].numpy()), (row.name, C)
            assert np.array_equal(s.view(np.int32), ws[0].numpy().view(np.int32)) or (
                np.isnan(s) == np.isnan(ws[0].numpy())).all() and np.array_equal(s[~np.isnan(s)],
                                                                                  ws[0].numpy()[~np.isnan(s)]), row.name


@pytest.mark.parametrize('V', ROW_V)
def test_sample_rows_hold_their_premise_and_claims(V):
    rows = sample_cases(V)
    seg = er.sample_seg(V)
    for row in rows:
        if er.is_greedy(row):
            assert er.on_grid(row.x)
            continue
        for T in (row.T, 0.5, 2.0):                  # any temperature up to 2 keeps the premise (sample_at mixes rows)
            _premise(row, T)
        kept = er.sample_kept(row)
        if row.claims.get('topk_cut'):
            assert row.k < row.ties.size and kept.size <= row.k
            if V > 2 * seg:
                assert len(set((kept // seg).tolist())) >= 2, row.name   # the kept ties cross warps
    kinds = {r.name.split('/')[-1] for r in rows}
    assert {'edges', 'topk_cross', 'greedy', 'greedy_nan'} <= kinds
    edges = next(r for r in rows if r.name.endswith('/edges'))
    want = {i for i in (seg - 1, seg, 15 * seg - 1, 15 * seg, 4095, 4096, 4097, V - 1) if i < V}
    assert want <= set(edges.ties.tolist()), V


@pytest.mark.parametrize('V', ROW_V)
def test_sample_rule_equals_the_oracle(V):
    for row in sample_cases(V):
        o = sample_row(row.x, row.T, row.k, row.p, row.seed, row.step)
        assert er.sample(row) == o['token'], row.name
        n = 1 if er.is_greedy(row) else er.sample_kept(row).size
        if n <= 1000:                                # the oracle's margin is relative to the kept mass
            assert not o['ambiguous'], row.name
        if er.is_greedy(row) and np.isnan(row.x.astype(np.float32)).any():
            assert er.sample(row) == int(np.flatnonzero(np.isnan(row.x.astype(np.float32)))[0])


def test_flat_row_rule():
    row = er.flat_sample_row()
    assert row.V == (1 << 24) - 1
    for t in range(6):
        w24 = int(round(uniform(row.seed, t) * 2 ** 24))
        assert er.sample(row, t) == (w24 * row.V) >> 24
    # one more tie would make the fixed-point sum of the kept weights 2^24 * 2^40 = 2^64, which wraps to 0
    assert (row.V + 1) * 2 ** 40 == 2 ** 64 and row.V * 2 ** 40 < 2 ** 64
    assert math.isclose(uniform(row.seed, 0) * 2 ** 24, round(uniform(row.seed, 0) * 2 ** 24))
