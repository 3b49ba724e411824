"""Sampled token selection (include/quip_b200.h, quip_sample) restated in numpy and Python ints.

The rule for one row x (V logits) with temperature T, top-k k, top-p p, seed and step t:
  greedy (T <= 0, T NaN or k == 1): the first index of max x;  z = float32(x) / float32(T) (IEEE);  rank z descending,
  ties by index;  the first K = min(k, V) (k > 0; else V) in rank order are the candidates;  e = exp(z - max z);  if p < 1
  the shortest rank-order prefix of the candidates with sum e >= p * sum over the candidates (at least one);  u from
  Philox4x32-10;  walking the kept tokens in index order, the first whose running sum of e exceeds u * S (else the last).

z is float32 as the kernel computes it, so the ranking and the top-k set agree bit for bit; e and the sums are float64.
`sample_row` also reports whether the case is ambiguous: a decision within a relative margin DELTA of its boundary, where
the kernel's fp32 exp and fixed-point sums may legitimately decide the other way.
"""
import numpy as np

DELTA = 1e-4
M0, M1 = 0xD2511F53, 0xCD9E8D57
W0, W1 = 0x9E3779B9, 0xBB67AE85
MASK = 0xFFFFFFFF


def philox4x32_10(counter, key):
    """Philox4x32-10 (Salmon, Moraes, Dror, Shaw, SC'11 / Random123) of 4 counter words under 2 key words."""
    c = [int(v) & MASK for v in counter]
    k0, k1 = int(key[0]) & MASK, int(key[1]) & MASK
    for r in range(10):
        if r:
            k0, k1 = (k0 + W0) & MASK, (k1 + W1) & MASK
        p0, p1 = M0 * c[0], M1 * c[2]
        c = [(p1 >> 32) ^ c[1] ^ k0, p1 & MASK, (p0 >> 32) ^ c[3] ^ k1, p0 & MASK]
    return c


def uniform(seed, t):
    """u in [0, 1) of (seed, step): the first Philox word of counter (t lo, t hi, 0, 0), key (seed lo, seed hi), top 24
    bits."""
    seed, t = int(seed) % 2 ** 64, int(t) % 2 ** 64
    w = philox4x32_10([t & MASK, t >> 32, 0, 0], [seed & MASK, seed >> 32])[0]
    return (w >> 8) * 2.0 ** -24


def is_greedy(T, k):
    return not (T > 0) or int(k) == 1


def sample_row(x, T, k, p, seed, t):
    """dict(token, kept (indices, rank order), probs (float64, over kept), ambiguous)."""
    x = np.asarray(x)
    V = x.shape[0]
    T, p = np.float32(T), np.float32(p)
    if is_greedy(T, k):
        i = int(np.argmax(x.astype(np.float32)))
        return dict(token=i, kept=np.array([i]), probs=np.ones(1), ambiguous=False)
    z = x.astype(np.float32) / T
    order = np.argsort(-z, kind='stable')
    K = min(int(k), V) if int(k) > 0 else V
    cand = order[:K]
    e = np.exp(z[cand].astype(np.float64) - np.float64(z[order[0]]))
    amb = False
    n = K
    if p < 1:
        cs = np.cumsum(e)
        target = float(p) * cs[-1]
        n = max(1, int(np.searchsorted(cs, target, side='left')) + 1) if target > 0 else 1
        n = min(n, K)
        if target > 0 and np.any(np.abs(cs - target) <= DELTA * target):
            amb = True
    kept, ek = cand[:n], e[:n]
    S = float(ek.sum())
    u = uniform(seed, t)
    idx = np.argsort(kept, kind='stable')                 # index order
    run = np.cumsum(ek[idx])
    thr = u * S
    j = int(np.searchsorted(run, thr, side='right'))       # first running sum > u * S
    j = min(j, n - 1)
    before = run[j - 1] if j else 0.0
    if abs(run[j] - thr) <= DELTA * S or (j and abs(before - thr) <= DELTA * S):
        amb = True
    return dict(token=int(kept[idx[j]]), kept=kept, probs=ek / S, ambiguous=amb)


def sample(logits, temperature, top_k, top_p, seeds, t):
    """Rows of logits (B, V) -> (tokens (B,) int64, ambiguous (B,) bool)."""
    logits = np.asarray(logits)
    B = logits.shape[0]
    out = [sample_row(logits[b], temperature[b], top_k[b], top_p[b], seeds[b], t) for b in range(B)]
    return (np.array([o['token'] for o in out], dtype=np.int64), np.array([o['ambiguous'] for o in out]))
