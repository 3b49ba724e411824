"""Constructed vocabulary rows whose answers are exact, for the row kernels.  TEST INFRASTRUCTURE ONLY.

The kernels are quip_sample / quip_sample_at (csrc/sample.cu), quip_token_logprobs and quip_token_topk_logprobs
(csrc/logprob.cu, csrc/topk_logprobs.cu, both on the row pass of csrc/logprob_row.cuh) and quip_beam_candidates
(csrc/beam.cu).  A row holds three kinds of value:

  * n copies of its maximum m;
  * negligible values with x - m <= -GAP (after temperature, in fp32 as the kernel computes it): e^-128 ~ 2.6e-56 is far
    below the smallest fp32 subnormal, so fp32 expf of them is exactly 0;
  * -inf.

Every value is an fp16 multiple of 1/8 of magnitude below 2048, so every difference x - m is exact in fp32.  Then each kernel's sum of exp is exactly n, whatever the order, and:

  * logprobs: (x - m) - L with L = logf(n); n = 1 gives L = 0, so the value is x - m bit for bit.  For n > 1, L is
    within 1 ulp of fp32(log n) and the same for every row with that n;
  * top-n: ids by the fp16 ranking, values as above;
  * beam candidates: s = ((x - m) - L) + score, exact for n = 1 when the score is on a coarse grid; ranking and indices
    are exact for any n;
  * sampling: the n tied weights are exactly 2^40 and every other weight 0.  Top-k keeps the first min(k, n) ties in
    index order, top-p the first max(1, ceil(p n_k)) of those (p n_k 2^40 is exact in double), and the token is the
    floor(w24 n_kept / 2^24)-th kept tie, w24 the top 24 bits of the Philox word.  Greedy rows with NaN take the first
    NaN.

Cases place ties and -inf by each kernel's split of the row (the constants below), at every 16-byte misalignment.
"""
import math
from dataclasses import dataclass, field
from fractions import Fraction

import numpy as np

from .sampling import uniform

# The work split of the row kernels, mirrored from their constants.
#   logprob_row.cuh (LP_THREADS) and beam.cu `sweep` (BC_THREADS): THREADS threads.  A row whose address is mis
#     elements past a 16-byte boundary splits into head = (8 - mis) & 7 scalars (thread i takes scalar i), nvec 16-byte
#     groups of GROUP values (thread k % THREADS takes group k, in k order; logprob_row keeps two loads in flight while
#     k + THREADS < nvec) and tail scalars (thread i takes body_end + i).
#   sample.cu (SP_THREADS, SP_U, SP_WARPS): index i belongs to thread i % THREADS, SP_STRIDE indices per loop; select
#     gives each of WARPS warps the contiguous segment of sample_seg(V) indices.
#   topk_logprobs.cu (TK_TIE_CAP, LP_WARPS): up to TIE_CAP ties at the threshold key are ranked in shared memory, more
#     are scanned by WARPS warps over contiguous segments of ceil(V / WARPS).
THREADS = 512
GROUP = 8
SP_STRIDE = 8 * THREADS
WARPS = 16
TIE_CAP = 64
GAP = 128
SAMPLE_MAX_V = (1 << 24) - 1        # quip_sample's bound: V * 2^40 < 2^64
MAXES = (0.0, 5.0, -100.0, 100.5)   # m; m - GAP - 0.25 stays on the fp16 1/8 grid


def split(V, mis):
    """(head, nvec, body_end) of a row mis elements past a 16-byte boundary."""
    head = min(V, (8 - mis) & 7)
    nvec = (V - head) // GROUP
    return head, nvec, head + GROUP * nvec


def units(V, mis, j):
    """The index ranges thread j reads, in its order: head scalar, groups j, j + THREADS, ..., tail scalar."""
    head, nvec, body_end = split(V, mis)
    out = [range(j, j + 1)] if j < head else []
    out += [range(head + GROUP * k, head + GROUP * (k + 1)) for k in range(j, nvec, THREADS)]
    if body_end + j < V:
        out.append(range(body_end + j, body_end + j + 1))
    return out


def sample_seg(V):
    return -(-V // (WARPS * 32)) * 32


def on_grid(x):
    """Every finite value a multiple of 1/8 below 2048 in magnitude."""
    f = x[np.isfinite(x)].astype(np.float64)
    return bool(np.all((f * 8 == np.round(f * 8)) & (np.abs(f) < 2048)))


@dataclass
class Row:
    name: str
    x: np.ndarray                   # fp16 (V,)
    m: float
    mis: int = 0                    # element offset of the row from a 16-byte boundary
    claims: dict = field(default_factory=dict)

    @property
    def V(self):
        return self.x.size

    @property
    def ties(self):
        return np.flatnonzero(self.x == np.float16(self.m))


def _base(V, m, rng, gap, ninf=0.03):
    """Negligible values m - gap - 1 - j (j < 256 integer) with a share of -inf, so the level m - gap is free."""
    x = (m - gap - 1 - rng.integers(0, 256, V)).astype(np.float16)
    x[rng.random(V) < ninf] = -np.inf
    return x


def _put(x, pos, v):
    pos = np.unique(np.asarray([p for p in pos if 0 <= p < x.size], dtype=np.int64))
    x[pos] = v
    return pos


# ---- rows for the log-sum-exp kernels (logprobs, top-n, beam)

def lse_edges(V, mis):
    """Indices at the edges of the split: the head, the first and last groups, both sides of the two-loads boundary,
    the tail."""
    head, nvec, body_end = split(V, mis)
    e = [0, head - 1, head, head + GROUP - 1, body_end - 1, body_end, V - 1]
    for k in (THREADS - 1, THREADS, nvec - THREADS - 1, nvec - THREADS, nvec - 2 * THREADS):
        if 0 <= k < nvec:
            e += [head + GROUP * k, head + GROUP * k + GROUP - 1]
    return sorted({i for i in e if 0 <= i < V})


def _lead_threads(V, mis):
    """Threads that read at least two units, the first in the head when there is one: the bug-1 pattern."""
    head, nvec, _ = split(V, mis)
    cand = [head - 1, THREADS - 1, head, 0, nvec % THREADS, (nvec - 1) % THREADS if nvec else 0, 37]
    return [j for j in dict.fromkeys(cand) if 0 <= j < THREADS and len(units(V, mis, j)) >= 2]


LSE_KINDS = ('lead_max', 'lead_ties', 'edges', 'edge_max', 'beam_over', 'topk_cap', 'all_ninf', 'flat')


def lse_rows(V, seed, count=16):
    """count rows of width V, row r at misalignment r % 8, cycling through the patterns."""
    rng = np.random.default_rng(seed)
    rows = []
    for r in range(count):
        mis, m = r % 8, MAXES[r % len(MAXES)]
        x = _base(V, m, rng, GAP)
        kind = LSE_KINDS[(r + r // 8) % 8]              # the second round shifts each kind to another misalignment
        claims = {}
        leads = _lead_threads(V, mis)
        if kind in ('lead_max', 'lead_ties') and not leads:
            kind = 'edges'
        if kind == 'flat' and V > (1 << 17):
            kind = 'edge_max'
        if kind in ('lead_max', 'lead_ties'):
            j = leads[0]
            us = units(V, mis, j)
            x[list(us[0])] = -np.inf
            later = us[1 + int(rng.integers(0, len(us) - 1))]
            at = int(later[int(rng.integers(0, len(later)))])
            extra = [] if kind == 'lead_max' else list(rng.integers(0, V, 2))
            for i in extra:
                if i not in us[0]:
                    x[i] = m
            x[at] = m
            claims = dict(lead_thread=j, lead_at=at)
        elif kind == 'edges':
            claims = dict(tie_at=[int(i) for i in _put(x, lse_edges(V, mis), m)])
        elif kind == 'edge_max':
            e = lse_edges(V, mis)
            claims = dict(tie_at=[int(i) for i in _put(x, [e[(r // 8) % len(e)]], m)])
        elif kind == 'beam_over':                          # one maximum, then more than 64 ties of the next level
            x[int(rng.integers(0, V))] = m
            x[rng.integers(0, V, min(V, 100))] = m - GAP
            claims = dict(level=m - GAP)
        elif kind == 'topk_cap':                           # 5 values above 64 or 65 ties (n = 20: threshold ties)
            cap = TIE_CAP + r % 2
            if V > cap + 6:
                pos = rng.permutation(V)
                x[pos[:1]] = m
                x[pos[1:5]] = m - GAP                      # three levels whose fp16 keys differ in the low byte only
                seg = -(-V // WARPS)
                edge = [w * seg + d for w in range(1, WARPS) for d in (-1, 0)]
                tie = list(dict.fromkeys([i for i in edge if i not in pos[:5]] + list(pos[5:5 + cap])))[:cap]
                x[tie] = m - GAP - 0.125
                x[pos[cap + 5:cap + 9]] = m - GAP - 0.25
                claims = dict(threshold_ties=cap, level=m - GAP - 0.125)
            else:
                x[:] = -np.inf
                kind = 'all_ninf'
        elif kind == 'all_ninf':
            x[:] = -np.inf
        else:
            x[:] = m
        if kind != 'all_ninf' and not (x == np.float16(m)).any():
            x[int(rng.integers(0, V))] = m
        if kind not in ('lead_max', 'lead_ties', 'all_ninf'):  # no other -inf leads a thread's share
            h = x[:split(V, mis)[0]]
            h[h == -np.inf] = m - GAP - 1
        rows.append(Row(f'V{V}/r{r}/mis{mis}/{kind}', x, m if kind != 'all_ninf' else -np.inf, mis, claims))
    return rows


def layout(rows):
    """(buffer (R * ld + 8,) fp16, ld) holding row r at element r * ld, with ld = 1 (mod 8): row r is r % 8 elements past
    a 16-byte boundary of a 16-byte aligned buffer."""
    V = rows[0].V
    ld = V + ((1 - V) % 8)
    buf = np.zeros(len(rows) * ld + 8, dtype=np.float16)
    for r, row in enumerate(rows):
        assert row.mis == r % 8 and row.V == V
        buf[r * ld:r * ld + V] = row.x
    return buf, ld


def fp32_logs(n):
    """The values logf(n) may take: 0 for n = 1, fp32(log n) and its neighbours otherwise."""
    if n <= 1:
        return [np.float32(0)]
    c = np.float32(math.log(n))
    return [c, np.nextafter(c, np.float32(-np.inf)), np.nextafter(c, np.float32(np.inf))]


def logprob(row, t, L):
    """fp32 (x_t - m) - L, NaN outside [0, V) and for rows of -inf ((-inf) - (-inf))."""
    if not 0 <= t < row.V:
        return np.float32(np.nan)
    with np.errstate(invalid='ignore'):
        return np.float32(np.float32(np.float32(row.x[t]) - np.float32(row.m)) - np.float32(L))


def first_max(row):
    return int(row.ties[0]) if row.ties.size else 0


def _rank(key, c):
    """Indices of the c largest keys (not NaN), key descending, then index ascending."""
    c = min(c, key.size)
    idx = np.arange(key.size)
    if c < key.size:
        idx = np.flatnonzero(key >= np.partition(key, key.size - c)[key.size - c])
    return idx[np.argsort(-key[idx], kind='stable')][:c]


def topn(row, n):
    """The first min(n, V) ids ranked by fp16 value descending, -0 == +0, ties by lower id."""
    return _rank(row.x.astype(np.float64) + 0.0, n)


def beam_key(s):
    from .beam import order_key
    return order_key(s)


def beam(row, score, C, L, beam_index=0):
    """(values (C,) fp32, flat ids (C,) int32) of quip_beam_candidates."""
    V = row.V
    x = row.x.astype(np.float32)
    if row.m == -np.inf:
        s = np.full(V, -np.inf, np.float32)
    else:
        s = ((x - np.float32(row.m)) - np.float32(L)).astype(np.float32) + np.float32(score)
    order = _rank(beam_key(s), C)
    vs = np.full(C, np.nan, np.float32)
    ids = np.full(C, -1, np.int32)
    vs[:order.size] = s[order]
    ids[:order.size] = order + beam_index * V
    return vs, ids


# ---- rows for the sampler

@dataclass
class SampleRow(Row):
    T: float = 1.0
    k: int = 0
    p: float = 1.0
    seed: int = 0
    step: int = 0


def _p_for(n, rng):
    """A top-p whose p n is far from an integer (the float64 oracle's margin), or 1."""
    for p in (0.3, 0.55, 0.7, 0.85, 0.45, 0.62):
        q = float(np.float32(p)) * n
        if abs(q - round(q)) > max(2e-4 * q, 0.05) and math.ceil(q) < n:
            return p
    return 1.0


def sample_kept(row):
    """The kept ties of a non-greedy row, in index order."""
    ties = row.ties
    K = min(row.k, row.V) if row.k > 0 else row.V
    nk = min(K, ties.size)
    if row.p < 1:
        nk = max(1, math.ceil(Fraction(float(np.float32(row.p))) * nk))
    return ties[:nk]


def is_greedy(row):
    return not (row.T > 0) or row.k == 1


def sample(row, step=None, settings=None):
    """The token of quip_sample for row under its settings (or those of `settings`) at its step (or `step`)."""
    s = settings or row
    t = s.step if step is None else step
    if is_greedy(s):
        x = row.x.astype(np.float32)
        nan = np.flatnonzero(np.isnan(x))
        return int(nan[0]) if nan.size else int(np.argmax(x))
    r = SampleRow(row.name, row.x, row.m, T=s.T, k=s.k, p=s.p)
    kept = sample_kept(r)
    w24 = int(round(uniform(s.seed, t) * 2 ** 24))
    return int(kept[(w24 * kept.size) >> 24])


def draw_margin(n, seed, t):
    """Distance of w24 n / 2^24 from the nearest integer."""
    q = Fraction(int(round(uniform(seed, t) * 2 ** 24)) * n, 1 << 24)
    return float(min(q - math.floor(q), math.ceil(q) - q)) if q.denominator != 1 else 0.0


def sample_edges(V):
    seg = sample_seg(V)
    e = [0, 1, THREADS - 1, THREADS, SP_STRIDE - 1, SP_STRIDE, SP_STRIDE + 1, V - 1, V - 2]
    e += [w * seg + d for w in range(1, WARPS) for d in (-1, 0)]
    return sorted({i for i in e if 0 <= i < V})


def sample_rows(V, seed, count=12, gap=2 * GAP):
    """count rows of width V with settings; gap 256 keeps the premise for every temperature up to 2."""
    rng = np.random.default_rng(seed)
    rows = []
    edges = sample_edges(V)
    for r in range(count):
        m = MAXES[r % len(MAXES)]
        x = _base(V, m, rng, gap)
        kind = ('edges', 'edge_one', 'topk_cross', 'topp', 'topk_topp', 'tempered', 'greedy', 'greedy_nan',
                'edges_topk', 'spread', 'flat', 'tempered_topp')[r % 12]
        T, k, p, claims = 1.0, 0, 1.0, {}
        if kind == 'flat' and V > SP_STRIDE + 1:
            kind = 'spread'
        if kind in ('edges', 'edges_topk', 'tempered', 'tempered_topp'):
            _put(x, edges, m)
        elif kind == 'edge_one':
            _put(x, [edges[(r + V) % len(edges)]], m)
        elif kind in ('topk_cross', 'topp', 'topk_topp', 'spread'):
            seg = sample_seg(V)                             # a few ties in every warp's segment
            pos = [w * seg + int(o) for w in range(WARPS) for o in rng.integers(0, seg, 3)]
            _put(x, pos, m)
        elif kind == 'greedy':
            _put(x, edges[::3], m)
            T = 0.0
        elif kind == 'greedy_nan':
            _put(x, edges[::2], m)
            _put(x, [edges[len(edges) // 2], V - 1], np.nan)
            k = 1                                           # greedy by k == 1 (the 'greedy' rows by T = 0)
        else:
            x[:] = m
        x[0] = -np.inf if kind == 'spread' and x[0] != np.float16(m) else x[0]
        n = int((x == np.float16(m)).sum())
        if n == 0:
            x[V // 2] = m
            n = 1
        if kind in ('topk_cross', 'edges_topk', 'topk_topp'):
            k = max(1, n // 2 + 1) if n > 2 else 2
            if k == 1:
                k = 2
            claims['topk_cut'] = k < n
        if kind in ('topp', 'topk_topp', 'tempered_topp'):
            p = _p_for(min(k, n) if k else n, rng)
        if kind.startswith('tempered'):
            T = (0.5, 0.75, 2.0)[r % 3]
        row = SampleRow(f'V{V}/s{r}/{kind}', x, m, claims=claims, T=T, k=k, p=p, seed=int(rng.integers(0, 2 ** 63)))
        nk = 1 if is_greedy(row) else sample_kept(row).size
        step = int(rng.integers(0, 1000))
        while nk <= 1000 and draw_margin(nk, row.seed, step) <= max(2e-4 * nk, 1e-3):
            step += 1
        row.step = step
        rows.append(row)
    return rows


def flat_sample_row(V=SAMPLE_MAX_V, seed=20250107, step=3):
    """Every value equal: n = V ties, every one kept; the token is the floor(w24 V / 2^24)-th."""
    return SampleRow(f'V{V}/flat', np.zeros(V, np.float16), 0.0, seed=seed, step=step)
