"""The vocabulary-row kernels on the exact rows of oracle/exact_rows.py, bit for bit.

quip_token_logprobs, quip_token_topk_logprobs, quip_beam_candidates, quip_sample and quip_sample_at run on rows whose
sums of exp are exact, with ties and -inf placed at the edges of each kernel's split of the row and at every 16-byte
misalignment.  Ids, tokens and is_greedy must match exactly, and every fp32 value must match the rule for one logf(n)
within 1 ulp of fp32(log n) that is shared by every row with the same n (n = 1: logf(1) = 0, every value exact).  The
same positions filled with random finite values, +inf or NaN are compared with the float64 oracles.  Each launch is
repeated and must give the same bits.
"""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from oracle import exact_rows as er
from oracle.beam import candidates as beam_oracle
from oracle.loglik import token_logprobs as lp_oracle
from oracle.topk_logprobs import topk_row
from quip_b200 import _lib, fused

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')

# the edge cases of V: tiny rows, 4096 +- 8 and 8192 +- 8 (every thread's first group, and the two-loads boundary of
# logprob_row), the sampler's 4096 stride, vocabulary sizes, and the top of the accepted range
ROW_V = [1, 7, 8, 9, 16, 17, 4088, 4104, 8184, 8200, 4095, 4096, 4097, 32000, 32001, 50272, 128256]
BIG_V = [(1 << 24) - 1, 1 << 24]
BEAM_V = [2, 63, 64, 65]                # V < C, V = C and V = C + 1 for C = 64 (the small ROW_V cover C = 1 and 8)
TOP_N = 20


def _same(a, b):
    """Equal bits, or both NaN."""
    a, b = np.asarray(a, np.float32), np.asarray(b, np.float32)
    return (a.view(np.int32) == b.view(np.int32)) | (np.isnan(a) & np.isnan(b))


def lse_cases(V):
    return er.lse_rows(V, seed=V, count=4 if V > (1 << 20) else 16)


def sample_cases(V):
    return er.sample_rows(V, seed=V + 1)


@functools.lru_cache(maxsize=None)
def _rows(V):
    rows = lse_cases(V)
    buf, ld = er.layout(rows)
    x = torch.from_numpy(buf).to(DEV)[:len(rows) * ld].view(len(rows), ld)[:, :V]
    return rows, x


class _Logs:
    """The logf(n) a kernel used for each n: one value per n for every row, within 1 ulp of fp32(log n)."""

    def __init__(self):
        self.seen = {}

    def fit(self, row, ok):
        """The first candidate L for which ok(L) holds, checked against the other rows with this n; None if none."""
        n = row.ties.size if row.m != -np.inf else 0
        for L in er.fp32_logs(n):
            if ok(L) and self.seen.setdefault(n, L) == L:
                return L
        return None


def _targets(row, rng):
    V, x = row.V, row.x
    ninf = np.flatnonzero(x == -np.inf)
    neg = np.flatnonzero(np.isfinite(x) & (x != np.float16(row.m)))
    pick = lambda a, d: int(a[rng.integers(0, a.size)]) if a.size else d
    return [er.first_max(row), int(row.ties[-1]) if row.ties.size else V - 1, pick(ninf, 0), pick(neg, V - 1), -1, V,
            int(rng.integers(0, V))]


@pytest.mark.parametrize('V', ROW_V + BIG_V)
def test_token_logprobs_exact(V):
    rows, x = _rows(V)
    rng = np.random.default_rng(V)
    tg = np.array([_targets(r, rng) for r in rows], np.int64)
    got, greedy = [], []
    for j in range(tg.shape[1]):
        t = torch.from_numpy(tg[:, j].copy()).to(DEV)
        outs = []
        for _ in range(2):
            lp = torch.full((len(rows),), 7.0, device=DEV)
            gr = torch.full((len(rows),), 7, dtype=torch.uint8, device=DEV)
            fused.token_logprobs(x, t, lp, gr)
            outs.append((lp.cpu().numpy(), gr.cpu().numpy()))
        assert np.array_equal(outs[0][0].view(np.int32), outs[1][0].view(np.int32)) and np.array_equal(*[o[1] for o in outs])
        got.append(outs[0][0])
        greedy.append(outs[0][1])
    got, greedy = np.stack(got, 1), np.stack(greedy, 1)
    logs, bad = _Logs(), []
    for r, row in enumerate(rows):
        want_gr = [int(0 <= t < V and t == er.first_max(row)) for t in tg[r]]
        L = logs.fit(row, lambda L: all(_same(got[r, j], er.logprob(row, t, L)) for j, t in enumerate(tg[r])))
        if L is None or list(greedy[r]) != want_gr:
            bad.append((row.name, list(tg[r]), got[r].tolist(), greedy[r].tolist()))
    assert not bad, bad


def _top(x, rows, tokens, n):
    R = len(rows)
    cols = torch.zeros(R, dtype=torch.long, device=DEV)
    outs = []
    for _ in range(2):
        lp = torch.full((R, 1), 7.0, device=DEV)
        ids = torch.full((R, 1, n), 9, dtype=torch.long, device=DEV)
        top = torch.full((R, 1, n), 7.0, device=DEV)
        fused.token_topk_logprobs(x, tokens, cols, lp, ids, top)
        outs.append((lp[:, 0].cpu().numpy(), ids[:, 0].cpu().numpy(), top[:, 0].cpu().numpy()))
    (lp, ids, top), again = outs
    assert np.array_equal(ids, again[1]) and np.array_equal(top.view(np.int32), again[2].view(np.int32))
    assert np.array_equal(lp.view(np.int32), again[0].view(np.int32))
    return lp, ids, top


@pytest.mark.parametrize('n', [1, 5, TOP_N])
@pytest.mark.parametrize('V', ROW_V + BIG_V)
def test_topk_logprobs_exact(V, n):
    if V in BIG_V and n != TOP_N:
        pytest.skip('one n at the top of the range')
    rows, x = _rows(V)
    tokens = torch.tensor([er.first_max(r) for r in rows], device=DEV)
    lp, ids, top = _top(x, rows, tokens, n)
    logs, bad = _Logs(), []
    for r, row in enumerate(rows):
        want = np.full(n, -1, np.int64)
        k = er.topn(row, n)
        want[:k.size] = k
        L = logs.fit(row, lambda L: (_same(lp[r], er.logprob(row, int(tokens[r]), L)) and
                                     all(_same(top[r, j], er.logprob(row, int(i), L)) for j, i in enumerate(want))))
        if L is None or not np.array_equal(ids[r], want):
            bad.append((row.name, ids[r].tolist(), want.tolist(), top[r].tolist()))
    assert not bad, bad
    for j in range(n):                            # the same bits as quip_token_logprobs on each id
        w = torch.empty(len(rows), device=DEV)
        fused.token_logprobs(x, torch.from_numpy(ids[:, j].copy()).to(DEV), w, torch.empty(len(rows), dtype=torch.uint8,
                                                                                             device=DEV))
        assert np.array_equal(w.cpu().numpy().view(np.int32), top[:, j].view(np.int32)), j


def _beam(x, scores, K, C):
    R = x.shape[0]
    outs = []
    for _ in range(2):
        cs = torch.full((R, C), 7.0, device=DEV)
        ci = torch.full((R, C), 9, dtype=torch.int32, device=DEV)
        fused.beam_candidates(x, scores, K, C, cs, ci)
        outs.append((cs.cpu().numpy(), ci.cpu().numpy()))
    (cs, ci), (cs2, ci2) = outs
    assert np.array_equal(cs.view(np.int32), cs2.view(np.int32)) and np.array_equal(ci, ci2)
    return cs, ci


@pytest.mark.parametrize('C', [1, 8, 64])
@pytest.mark.parametrize('V', ROW_V + BEAM_V + BIG_V[:1])
def test_beam_candidates_exact(V, C):
    rows, x = _rows(V)
    K = 3
    score = np.float32(-1.0) - np.float32(0.25) * (np.arange(len(rows)) % 7).astype(np.float32)
    cs, ci = _beam(x, torch.from_numpy(score).to(DEV), K, C)
    logs, bad = _Logs(), []
    for r, row in enumerate(rows):
        want = {}

        def ok(L):
            want[L] = er.beam(row, score[r], C, L, r % K)
            return np.array_equal(ci[r], want[L][1]) and _same(cs[r], want[L][0]).all()
        if logs.fit(row, ok) is None:
            bad.append((row.name, ci[r].tolist(), cs[r].tolist(), [w[1].tolist() for w in want.values()][:1]))
    assert not bad, bad


# ---- sampling

def _settings(rows):
    t = lambda a, dt: torch.tensor(a, dtype=dt, device=DEV)
    return (t([r.T for r in rows], torch.float32), t([r.k for r in rows], torch.int32),
            t([r.p for r in rows], torch.float32), t([r.seed for r in rows], torch.int64))


@functools.lru_cache(maxsize=None)
def _sample_rows(V):
    return sample_cases(V)


@pytest.mark.parametrize('V', ROW_V)
def test_sample_exact(V):
    rows = _sample_rows(V)
    x = torch.from_numpy(np.stack([r.x for r in rows])).to(DEV)
    T, k, p, seed = _settings(rows)
    for step in (0, 7777, (1 << 32) + 5):
        toks = []
        for _ in range(2):
            out = torch.full((len(rows),), -5, dtype=torch.long, device=DEV)
            fused.sample(x, T, k, p, seed, torch.tensor([step], device=DEV), out)
            toks.append(out.cpu().numpy())
        assert np.array_equal(*toks)
        want = [er.sample(r, step) for r in rows]
        bad = [(r.name, int(g), w) for r, g, w in zip(rows, toks[0], want) if g != w]
        assert not bad, (step, bad)


@pytest.mark.parametrize('Tn', [1, 3, 8])
@pytest.mark.parametrize('V', [9, 4096, 4097, 32001])
def test_sample_at_agrees_with_sample(V, Tn):
    """Row b * T + i: row (b + i) of the non-NaN rows with the settings of b at step steps[b] + i, as quip_sample
    gives it."""
    rows = [r for r in _sample_rows(V) if not np.isnan(r.x.astype(np.float32)).any()]
    B = len(rows)
    x = torch.from_numpy(np.stack([[rows[(b + i) % B].x for i in range(Tn)] for b in range(B)])).to(DEV)
    T, k, p, seed = _settings(rows)
    steps = torch.tensor([r.step for r in rows], device=DEV)
    outs = []
    for _ in range(2):
        out = torch.full((B, Tn), -5, dtype=torch.long, device=DEV)
        fused.sample_at(x, T, k, p, seed, steps, out)
        outs.append(out.cpu().numpy())
    assert np.array_equal(*outs)
    want = np.array([[er.sample(rows[(b + i) % B], rows[b].step + i, rows[b]) for i in range(Tn)] for b in range(B)])
    assert np.array_equal(outs[0], want), [(rows[b].name, i) for b, i in np.argwhere(outs[0] != want)]
    for i in range(Tn):                           # quip_sample on the same rows, one shared step per launch
        for b in range(B):
            one = torch.empty(1, dtype=torch.long, device=DEV)
            fused.sample(x[b:b + 1, i].contiguous(), T[b:b + 1], k[b:b + 1], p[b:b + 1], seed[b:b + 1],
                         steps[b:b + 1] + i, one)
            assert int(one) == outs[0][b, i], (rows[b].name, i)


def test_sample_flat_row_at_the_top_of_the_range():
    """V = 2^24 - 1 equal values: every token is kept and the draw picks the floor(w24 V / 2^24)-th."""
    row = er.flat_sample_row()
    x = torch.zeros(1, row.V, dtype=torch.float16, device=DEV)
    T, k, p, seed = _settings([row])
    for step in range(4):
        out = torch.empty(1, dtype=torch.long, device=DEV)
        fused.sample(x, T, k, p, seed, torch.tensor([step], device=DEV), out)
        assert int(out) == er.sample(row, step), step
    w = x.view(1, 1, row.V)
    out = torch.empty(1, 1, dtype=torch.long, device=DEV)
    fused.sample_at(w, T, k, p, seed, torch.tensor([5], device=DEV), out)
    assert int(out) == er.sample(row, 5)


def test_sample_refuses_v_of_2_to_the_24():
    """At V = 2^24 the fixed-point sum of 2^24 weights of 2^40 would wrap: the wrappers and the C ABI refuse it, and
    nothing is launched."""
    V = 1 << 24
    x = torch.zeros(1, V, dtype=torch.float16, device=DEV)
    T, k, p, seed = _settings([er.SampleRow('flat', x, 0.0)])
    step = torch.zeros(1, dtype=torch.long, device=DEV)
    out = torch.full((1,), -5, dtype=torch.long, device=DEV)
    with pytest.raises(ValueError, match='sample'):
        fused.sample(x, T, k, p, seed, step, out)
    with pytest.raises(ValueError, match='sample_at'):
        fused.sample_at(x.view(1, 1, V), T, k, p, seed, step, out.view(1, 1))
    lib = _lib.load()
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    ptrs = [t.data_ptr() for t in (x, T, k, p, seed, step, out)]
    with pytest.raises(_lib.QuipError, match='bad sizes'):
        _lib.check(lib.quip_sample(*ptrs, 1, V, st))
    with pytest.raises(_lib.QuipError, match='bad sizes'):
        _lib.check(lib.quip_sample_at(*ptrs, 1, 1, V, st))
    torch.cuda.synchronize()
    assert int(out) == -5


# ---- the same positions with random values, +inf and NaN, against the float64 oracles

@functools.lru_cache(maxsize=None)
def _random_rows(V):
    """Each exact row with its finite values redrawn at random; rows 3 and 11 get +inf, rows 5 and 13 a NaN, at a tie."""
    rows, _ = _rows(V)
    g = np.random.default_rng(V + 2)
    buf, ld = er.layout(rows)
    out = []
    for r, row in enumerate(rows):
        x = row.x.copy()
        fin = np.isfinite(x)
        x[fin] = np.round(g.standard_normal(int(fin.sum())) * 3, 1).astype(np.float16)
        if r % 8 in (3, 5) and row.ties.size:
            x[row.ties[0]] = np.inf if r % 8 == 3 else np.nan
        buf[r * ld:r * ld + V] = x
        out.append(x)
    return np.stack(out), torch.from_numpy(buf).to(DEV)[:len(rows) * ld].view(len(rows), ld)[:, :V]


@pytest.mark.parametrize('V', [9, 17, 4097, 8200, 32001, 128256])
def test_random_rows_at_the_same_positions_match_the_oracles(V):
    xs, x = _random_rows(V)
    R = xs.shape[0]
    rng = np.random.default_rng(V)
    t = rng.integers(0, V, R)
    lp = torch.empty(R, device=DEV)
    gr = torch.empty(R, dtype=torch.uint8, device=DEV)
    fused.token_logprobs(x, torch.from_numpy(t).to(DEV), lp, gr)
    want, wgr = lp_oracle(xs, t)
    m = np.abs(np.where(np.isfinite(xs), xs, 0).astype(np.float64)).max(1)
    got = lp.cpu().numpy().astype(np.float64)
    close = (np.abs(got - want) <= 1e-5 + 1e-6 * m) | (np.isnan(got) & np.isnan(want)) | (got == want)
    assert close.all(), [(r, got[r], want[r]) for r in np.flatnonzero(~close)]
    assert np.array_equal(gr.cpu().numpy(), wgr)
    _, ids, top = _top(x, [None] * R, torch.from_numpy(t).to(DEV), TOP_N)
    for r in range(R):
        wi, wv = topk_row(xs[r], TOP_N)
        assert np.array_equal(ids[r], wi), r
        assert np.allclose(top[r].astype(np.float64), wv, atol=2e-5, rtol=0, equal_nan=True), r
    scores = torch.full((R,), -1.5, device=DEV)
    for C in (1, 8, 64):
        cs, ci = _beam(x, scores, 2, C)
        ws, wi = beam_oracle(torch.from_numpy(xs), scores.cpu(), 2, C)
        assert np.array_equal(ci, wi.numpy()), C
        torch.testing.assert_close(torch.from_numpy(cs), ws, rtol=2e-6, atol=2e-5, equal_nan=True)
