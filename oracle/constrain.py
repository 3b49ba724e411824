"""Constrained generation by a token automaton (include/quip_b200.h, quip_constrain_mask / quip_constrain_advance)
restated in numpy and Python ints.

The table packs S states: state s allows ids[k] and leads to next[k] for k in [lo_s, hi_s), lo_s = clamp(offsets[s],
0, nnz), hi_s = clamp(offsets[s + 1], lo_s, nnz).  delta(s, v) = next[k] where ids[k] == v in that range, else s; for
s outside [0, S), delta(s, v) = s.
  mask: a row with state s_0 and drafts d_1 .. d_i is left alone when s_i = delta(..delta(s_0, d_1).., d_i) lies
        outside [0, S); otherwise x_v <- x_v + (v allowed in s_i ? +0 : -inf) in x's dtype, for every v (ids outside
        [0, V) allow nothing);
  advance: the state walked over the committed tokens, in order.
"""
import numpy as np


def _range(offsets, nnz, s):
    lo = min(max(int(offsets[s]), 0), nnz)
    return lo, min(max(int(offsets[s + 1]), lo), nnz)


def delta(offsets, ids, next, s, v):
    S, nnz = len(offsets) - 1, len(ids)
    if not 0 <= s < S:
        return s
    lo, hi = _range(offsets, nnz, s)
    k = np.nonzero(np.asarray(ids[lo:hi], dtype=np.int64) == int(v))[0]
    return int(next[lo + k[0]]) if k.size else s


def walk(offsets, ids, next, s, tokens):
    for v in tokens:
        s = delta(offsets, ids, next, s, v)
    return int(s)


def mask_row(x, offsets, ids, next, s0, drafts=()):
    """The masked copy of one row x (1-D numpy array, fp16 or fp32) at state s0 after walking `drafts`."""
    x = np.array(x, copy=True)
    s = walk(offsets, ids, next, int(s0), drafts)
    if not 0 <= s < len(offsets) - 1:
        return x
    V = x.shape[0]
    lo, hi = _range(offsets, len(ids), s)
    bias = np.full(V, -np.inf, dtype=x.dtype)
    allowed = np.asarray(ids[lo:hi], dtype=np.int64)
    bias[allowed[(allowed >= 0) & (allowed < V)]] = 0
    with np.errstate(invalid='ignore'):
        return (x + bias).astype(x.dtype)


def advance(state, tokens, offsets, ids, next, counts=None, rows=None):
    """The advanced copy of state (B,) int32: entry n of tokens (N, T) walks state[rows[n]] (default n) over its first
    counts[n] (default T, clamped to [0, T]) tokens; rows outside [0, B) are skipped."""
    state = np.array(state, dtype=np.int32, copy=True)
    N, T = np.asarray(tokens).shape
    for n in range(N):
        b = n if rows is None else int(rows[n])
        if not 0 <= b < len(state):
            continue
        c = T if counts is None else min(max(int(counts[n]), 0), T)
        state[b] = walk(offsets, ids, next, int(state[b]), [int(v) for v in tokens[n][:c]])
    return state
