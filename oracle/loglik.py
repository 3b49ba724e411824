"""Float64 restatement of quip_token_logprobs (include/quip_b200.h) and of the reference harness's request windows.

token_logprobs: for fp16 logits (R, V) and int targets (R,), logprob = x_t - m - log sum exp(x - m) in float64 and
is_greedy = (t == the lowest index of the row's largest value); NaN rows and targets outside [0, V) give NaN and 0.

windows: BaseLM._loglikelihood_tokens (zeroShot/models/models_utils.py): requests grouped by their token sequence
ctx + cont (the first occurrence's split), ordered by (-length, tokens); input (ctx + cont)[-(max_length + 1):][:-1],
whose last len(cont) positions are scored against cont.
"""
import numpy as np


def token_logprobs(logits, targets):
    x = np.asarray(logits, dtype=np.float64)
    t = np.asarray(targets, dtype=np.int64)
    R, V = x.shape
    lp = np.full(R, np.nan)
    gr = np.zeros(R, dtype=np.uint8)
    for r in range(R):
        row = x[r]
        if np.isnan(row).any() or not 0 <= t[r] < V:
            continue
        m = row.max()
        lp[r] = (row[t[r]] - m) - np.log(np.exp(row - m).sum())
        gr[r] = int(np.argmax(row) == t[r])                     # np.argmax: the first index of the maximum
    return lp, gr


def windows(contexts, continuations, max_length):
    """[(inp, cont, caller indices)] in the harness's order."""
    groups = {}
    for i, (c, x) in enumerate(zip(contexts, continuations)):
        key = tuple(list(c) + list(x))
        groups.setdefault(key, (list(c), list(x), []))[2].append(i)
    order = sorted(groups, key=lambda k: (-len(k), k))
    return [(list(k)[-(max_length + 1):][:-1], groups[k][1], groups[k][2]) for k in order]
