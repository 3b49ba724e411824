"""quip_token_topk_logprobs (include/quip_b200.h) restated in numpy for one logits row.

Ranking on the fp16 values: logit descending, equal values (-0 == +0) by lower id; the first min(n, V) ids, then
(-1, NaN).  A row holding a NaN gives (-1, NaN) throughout.  Values by the formula of oracle/loglik.py in float64:
x_v - m - log sum exp(x - m).
"""
import numpy as np

from .loglik import token_logprobs


def topk_row(row, n):
    """(ids (n,) int64, logprobs (n,) float64) of one fp16 row."""
    x = np.asarray(row, dtype=np.float16).astype(np.float64)
    ids = np.full(n, -1, dtype=np.int64)
    vals = np.full(n, np.nan)
    if np.isnan(x).any():
        return ids, vals
    k = min(n, x.size)
    order = np.argsort(-x, kind='stable')[:k]                  # -(+0) == -(-0): ties stay in id order
    ids[:k] = order
    with np.errstate(invalid='ignore'):                         # +inf rows: inf - inf, NaN as the rule says
        vals[:k] = token_logprobs(np.repeat(x[None], k, 0), order)[0]
    return ids, vals
