"""Logits processors of generation (include/quip_b200.h, quip_logits_process) restated in numpy and Python ints.

For a logits row x (fp16 or fp32) with history h (the decoder row's tokens by position, then its drafts), L = len(h),
n_new = L - prompt_len, penalty rho, n-gram size n, min_new m, eos ids and bad-word sequences:
  1. rho != 1: every distinct v of h in [0, V): x_v <- x_v < 0 ? x_v * rho : x_v / rho, in float32, rounded once to x's
     dtype;
  2. n >= 1: the last token of every n-gram of h whose first n - 1 tokens equal h's last n - 1 tokens gets -inf;
  3. bad words (one-token sequences equal to an eos id dropped): w bans w[-1] when len(w) == 1, or len(w) <= L and h ends
     with w[:-1]; with any bad words the row becomes x + bias (bias -inf at the banned tokens, +0 elsewhere);
  4. n_new < m: every eos id gets -inf.
"""
import numpy as np


def process_row(x, h, prompt_len, rho, n, m, eos, bad):
    """The processed copy of one row x (1-D numpy array); h a list of ints, bad a list of id lists."""
    x = np.array(x, copy=True)
    V, L = x.shape[0], len(h)
    eos = [int(e) for e in eos]
    pen, ng, ban_eos = np.float32(rho) != np.float32(1), 1 <= n <= L, bool(eos) and L - prompt_len < m
    if not (pen or ng or ban_eos or bad):
        return x
    if pen:
        r = np.float32(rho)
        for v in sorted({v for v in h if 0 <= v < V}):
            f = np.float32(x[v])
            x[v] = (f * r if f < 0 else f / r).astype(x.dtype)
    hard = set()
    if ng:
        for e in range(L - n + 1):
            if h[e:e + n - 1] == h[L - n + 1:]:
                hard.add(h[e + n - 1])
    if bad:
        keep = [w for w in bad if 1 <= len(w) <= 16 and not (len(w) == 1 and w[0] in eos)]
        biased = {w[-1] for w in keep if len(w) == 1 or (len(w) <= L and h[L - len(w) + 1:] == list(w[:-1]))}
        bias = np.zeros(V, dtype=np.float32)
        bias[[v for v in biased if 0 <= v < V]] = -np.inf
        with np.errstate(invalid='ignore'):
            x = (x.astype(np.float32) + bias).astype(x.dtype)
    if ban_eos:
        hard.update(eos)
    x[[v for v in hard if 0 <= v < V]] = -np.inf
    return x
