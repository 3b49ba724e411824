"""Restatement of the beam-search candidate rule and the cache fork (include/quip_b200.h: quip_beam_candidates,
quip_kv_beam_fork) for the GPU tests, written independently of quip_b200/decode.py: the lse in float64, the ranking by
a full sort, and the fork as a gather of whole rows through the tables."""
import numpy as np
import torch


def order_key(s):
    """int64 keys of fp32 s: larger for larger s, -0 == +0, NaN lowest."""
    s = np.asarray(s, dtype=np.float32)
    u = np.where(s == 0, np.float32(0), s).view(np.uint32).astype(np.int64)
    k = np.where(u >= 2 ** 31, (~u) & 0xFFFFFFFF, u | 2 ** 31)
    return np.where(np.isnan(s), 0, k)


def candidates(logits, scores, K, C):
    """(R, C) fp32 values and int32 flat indices (r % K) * V + v of each row's top min(C, V) of
    s = ((x - m) - log sum exp(x - m)) + score (fp32 steps, the sum in float64), ranked by s descending (NaN last),
    then lower index; (NaN, -1) padding when V < C."""
    x = logits.float().cpu().numpy()
    sc = scores.float().cpu().numpy()
    R, V = x.shape
    out_s = np.full((R, C), np.nan, dtype=np.float32)
    out_i = np.full((R, C), -1, dtype=np.int32)
    for r in range(R):
        row = x[r]
        m = np.float32(row.max()) if not np.isnan(row).any() else np.float32(np.nan)
        if m == -np.inf:
            s = np.full(V, -np.inf, dtype=np.float32)
        else:
            logS = np.float32(np.log(np.exp(row.astype(np.float64) - np.float64(m)).sum()))
            s = ((row - m).astype(np.float32) - logS).astype(np.float32) + np.float32(sc[r])
        order = np.lexsort((np.arange(V), -order_key(s)))[:min(C, V)]
        out_s[r, :order.size] = s[order]
        out_i[r, :order.size] = order + (r % K) * V
    return torch.from_numpy(out_s), torch.from_numpy(out_i)


def gathered(pool, table):
    """Every row's slots through its table: pool (L, n_pages, nkv, 64, hd) or scales (L, n_pages, nkv, 64) ->
    (R, max_pages * 64, L, nkv[, hd]); unmapped pages read as NaN."""
    R, P = table.shape
    t = table.long()
    ok = (t >= 0) & (t < pool.shape[1])
    g = pool.float()[:, t.clamp(min=0, max=pool.shape[1] - 1)]             # (L, R, P, nkv, 64[, hd])
    g = torch.where(ok.view(1, R, P, *[1] * (g.dim() - 3)), g, torch.full_like(g, float('nan')))
    g = g.permute(1, 2, 4, 0, 3, 5) if g.dim() == 6 else g.permute(1, 2, 4, 0, 3)   # (R, P, 64, L, nkv[, hd])
    return g.reshape(R, P * 64, *g.shape[3:])
