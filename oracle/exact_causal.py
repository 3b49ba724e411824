"""Exactly representable multi-token cases for the extend- and prefill-attention kernels.  TEST INFRASTRUCTURE ONLY.

The kernels are quip_extend_attention's (csrc/attn_decode.cu: attn_extend_split_kernel and the multi-token
combine) and quip_kv_append followed by quip_prefill_attention (csrc/attn_prefill.cu), on fp16 and e4m3 caches.  Token i of row b
attends over slots 0 .. positions[b] + i.  The premise is the one of oracle/exact_attn.py, per (row, token): when
every score a token sees either equals its maximum bit for bit or lies at least DELTA = 128 below it, expf gives
exactly 1 or 0, and attention returns the mean of the V rows of the token's visible selected slots.  In detail:

  * the score of a visible selected slot is the token's maximum M; every other visible slot scores <= M - DELTA;
  * extend: per 64-slot chunk m, l = count and o = sum of V over the chunk's part of the visible set (e4m3: of
    p s_v / sm V, times sm, sm the largest v scale the token sees in the chunk); the combine merges the chunks
    0 .. (pos + i) / 64 and weighs a chunk without a selected slot by expf(m - M) = 0;
  * prefill: online softmax over 64-slot blocks.  alpha = expf(m_old - m_new) is 1 when m does not move and 0 when
    it first reaches M from a block without a selected slot (m_old <= M - DELTA), so such stale partials are wiped
    exactly as long as they are finite; later blocks add p = 0.  e4m3 keeps O' = O / c with c the last block's sm and
    rescales O' by alpha c / sm: a power of two (or 0), exact as long as O' stays above the fp32 normal range;
  * P is 0, 1, or s_v / sm (a power of two >= 2^-14, a normal fp16), so its fp16 rounding is exact;
  * Q.K and P.V on mma.sync are exact when every partial is a multiple of its granularity g and at most 2^24 g,
    the budget of oracle/exact.check_mma;
  * each kernel ends with one IEEE division O / L and one fp16 rounding.

So both kernels must return fp16_rn(fp32(O) / fp32(L)) bit for bit, O the sum of V over the token's visible selected
slots and L their count.  Prefill rows past a row's count are +0; rows the kernel must not look at are NaN.

Construction (make_case) follows exact_attn.make_case: head g of a kv group owns the dimensions d = g (mod G), q = c_g P
there, K = +-P there (+ on S_h), and the first dimensions of V spell the slot index.  The K vector of a slot is shared
by all tokens, so the selected set S_h is per head and token i sees S_h n [0, pos + i].  Per (token, head) q is
either 0 (uniform attention over 0 .. pos + i) or c_g P 2^(i mod 3).  Every S_h holds a slot <= pos, so no token sees
an empty set.  Kinds beyond exact_attn's: 'new' (slots pos + i of every counted token plus one older slot, so token i
averages i + 2 rows), 'last_new' (only the last counted token sees its own slot) and 'block_edge' (slots 64k - 1 and
64k around every block boundary).  Tie heads keep their 14 slots <= pos, so every token sees the whole tie.  Before
the call the new slots hold a decoy: K negated on the P dimensions and V reversed (e4m3: scales x 8).
"""
from dataclasses import dataclass, field

import numpy as np

from .exact import BudgetError, _fits
from .exact_attn import (DELTA, E4M3, E4M3_MAX, FLT_MAX, V_DEN, _merge_scales, _select, _walk, e4m3_bytes,
                         is_fp16_tie)
from .exact_quant import gran

BLOCK = 64                      # slots per chunk (extend) and per block (prefill)
TILE = 64                       # query rows per prefill CTA
KINDS = ('uniform', 'new', 'pos', 'last_new', 'zero', 'block_edge', 'all', 'chunk_last', 'boundary', 'rand3',
         'rand7', 'tie14')
ZERO_EVERY = 7                  # about one in ZERO_EVERY (token, head) pairs of a q != 0 head (not a tie) gets q = 0


@dataclass
class CausalCase:
    """One call of the extend kernel (kernel 'extend') or of kv_append + prefill attention ('prefill')."""
    kernel: str
    fp8: bool
    scale: float                # an fp32 value
    q: np.ndarray               # (B, T, nh, hd) fp16
    k_new: np.ndarray           # (B, T, nkv, hd) fp16
    v_new: np.ndarray
    k_cache: np.ndarray         # (B, nkv, max_len, hd) fp16 or uint8 (e4m3 bytes), before the call
    v_cache: np.ndarray
    k_scale: object             # (B, nkv, max_len) fp32, or None
    v_scale: object
    positions: np.ndarray       # (B,) int64
    counts: np.ndarray          # (B,) int64 (extend: T)
    sel: np.ndarray             # (B, nh, max_len) bool: S_h
    zero: np.ndarray            # (B, T, nh) bool: q = 0
    kinds: list = field(default_factory=list)   # (B, nh) kind names

    @property
    def shape(self):
        B, T, nh, hd = self.q.shape
        return B, T, nh, self.k_new.shape[2], hd, self.k_cache.shape[2]

    @property
    def G(self):
        return self.q.shape[2] // self.k_new.shape[2]

    def valid(self, b):
        B, T, nh, nkv, hd, max_len = self.shape
        p, n = int(self.positions[b]), int(self.counts[b])
        if self.kernel == 'extend':
            return 0 <= p <= max_len - T
        return p >= 0 and 0 <= n <= T and p + n <= max_len

    def count(self, b):
        """Tokens of row b the kernel computes (0 for a row it must not look at)."""
        return int(self.counts[b]) if self.valid(b) else 0

    def new_quantized(self):
        """(k bytes, k scale, v bytes, v scale) of k_new / v_new (B, T, nkv, ...) as kvfp8.quantize gives them."""
        if '_newq' not in self.__dict__:
            import torch
            from . import kvfp8
            out = []
            for x in (self.k_new, self.v_new):
                qb, s = kvfp8.quantize(torch.from_numpy(x))
                out += [qb.view(torch.uint8).numpy(), s.numpy()]
            self._newq = out
        return self._newq

    def caches_after(self):
        """(k_cache, v_cache, k_scale, v_scale) as the call must leave them: token i < count of row b at slot
        positions[b] + i (e4m3: quantized), nothing else changed."""
        kc, vc = self.k_cache.copy(), self.v_cache.copy()
        ks = None if self.k_scale is None else self.k_scale.copy()
        vs = None if self.v_scale is None else self.v_scale.copy()
        if self.fp8:
            kq, kqs, vq, vqs = self.new_quantized()
        for b in range(len(self.positions)):
            n, p = self.count(b), int(self.positions[b])
            if n == 0:
                continue
            sl = slice(p, p + n)
            if self.fp8:
                kc[b, :, sl], vc[b, :, sl] = kq[b, :n].transpose(1, 0, 2), vq[b, :n].transpose(1, 0, 2)
                ks[b, :, sl], vs[b, :, sl] = kqs[b, :n].T, vqs[b, :n].T
            else:
                kc[b, :, sl], vc[b, :, sl] = self.k_new[b, :n].transpose(1, 0, 2), self.v_new[b, :n].transpose(1, 0, 2)
        return kc, vc, ks, vs

    def slots(self, rows, pre=False):
        """K, V (R, nkv, max_len, hd) float64 in cache units and ks, vs (R, nkv, max_len) float64 (ones for fp16) of
        the rows as the kernel reads them (after the append), or as they were before the call (pre)."""
        if '_after' not in self.__dict__:
            self._after = self.caches_after()
        kc, vc, ksc, vsc = (self.k_cache, self.v_cache, self.k_scale, self.v_scale) if pre else self._after
        rows = np.asarray(rows)
        if self.fp8:
            return E4M3[kc[rows]], E4M3[vc[rows]], ksc[rows].astype(np.float64), vsc[rows].astype(np.float64)
        K, V = kc[rows].astype(np.float64), vc[rows].astype(np.float64)
        ones = np.ones(K.shape[:3])
        return K, V, ones, ones


def visible(c, rows):
    """(R, T, nh, max_len) bool: the slots each computed token sees with weight 1 -- S_h n [0, pos + i], or all of
    0 .. pos + i for q = 0 -- and live (R, T, max_len): the slots 0 .. pos + i of a computed token."""
    B, T, nh, nkv, hd, max_len = c.shape
    rows = np.asarray(rows)
    cnt = np.array([c.count(b) for b in rows])
    j = np.arange(max_len)
    t = np.arange(T)
    live = (j[None, None, :] <= (c.positions[rows][:, None] + t[None, :])[..., None]) & (t[None, :] < cnt[:, None])[..., None]
    vis = live[:, :, None, :] & (c.zero[rows][..., None] | c.sel[rows][:, None])
    return vis, live


def _row_blocks(c, elems=1 << 23):
    B, T, nh, nkv, hd, max_len = c.shape
    rows = np.array([b for b in range(B) if c.count(b) > 0], np.int64)
    step = max(1, elems // (T * nh * max_len + nkv * max_len * hd))
    return [rows[i:i + step] for i in range(0, len(rows), step)]


def _dots(c, rows, K, absolute=False):
    """q . K (R, T, nh, max_len) float64 (exact: small dyadic values)."""
    R, nkv, L, hd = K.shape
    T, G = c.q.shape[1], c.G
    q = c.q[rows].astype(np.float64).reshape(R, T, nkv, G, hd).transpose(0, 2, 1, 3, 4).reshape(R, nkv, T * G, hd)
    if absolute:
        q, K = np.abs(q), np.abs(K)
    d = np.matmul(q, K.transpose(0, 1, 3, 2))                              # (R, nkv, T G, L)
    return d.reshape(R, nkv, T, G, L).transpose(0, 2, 1, 3, 4).reshape(R, T, nkv * G, L)


def fp32_scores(c, rows, K, ks):
    """The kernels' scores (R, T, nh, max_len) fp32: fp32(d * scale), times the slot's k scale for e4m3."""
    s = (_dots(c, rows, K).astype(np.float32) * np.float32(c.scale)).astype(np.float32)
    if c.fp8:
        ksh = np.repeat(ks, c.G, axis=1).astype(np.float32)                # (R, nh, L)
        s = (s * ksh[:, None]).astype(np.float32)
    return s


# --------------------------------------------------------------------------------------------------------------
# budget and reference
# --------------------------------------------------------------------------------------------------------------
def check_budget(c):
    """Raise BudgetError unless the case meets the exactness premise (module docstring), per (row, token) with the
    live slots 0 .. pos + i.  Returns the bits used {'dot', 'sum', 'gap'}.  Granularities are taken over a block of
    rows and over all of a row's slots, which only makes the bounds stricter."""
    B, T, nh, nkv, hd, max_len = c.shape
    G = c.G
    bits = dict(dot=0.0, sum=0.0, gap=np.inf)
    for rows in _row_blocks(c):
        R = len(rows)
        what = f'rows {rows[0]}..{rows[-1]}'
        K, V, ks, vs = c.slots(rows)
        vis, live = visible(c, rows)
        for r, b in enumerate(rows):
            p, n = int(c.positions[b]), c.count(b)
            S = c.sel[b]
            if S[:, p + n:].any():
                raise BudgetError(f'{what}: row {b} selects a slot past its last token')
            if not S[:, :p + 1].any(1).all():
                raise BudgetError(f'{what}: row {b} has a head without a selected slot <= pos')
        dot = _dots(c, rows, K, absolute=True)
        bits['dot'] = max(bits['dot'], _fits(dot, gran(c.q[rows]) * gran(K), f'{what}: q . K'))
        s = fp32_scores(c, rows, K, ks)
        lv = live[:, :, None, :]
        s = np.where(lv, s, -np.inf).astype(np.float32)
        M = np.where(vis, s, -np.inf).max(3)
        comp = np.broadcast_to(live.any(2)[:, :, None], M.shape)           # computed (row, token, head)
        if not np.array_equal(M[comp], s.max(3)[comp]) or not np.all(np.where(vis, s == M[..., None], True)):
            raise BudgetError(f'{what}: the visible selected slots do not all score the token maximum bit for bit')
        with np.errstate(invalid='ignore'):
            gap = (s - M[..., None]).astype(np.float32)
        worst = float(np.where(vis | ~lv, -np.inf, gap).max(initial=-np.inf))
        if worst > -DELTA:
            raise BudgetError(f'{what}: score gap {-worst:.6g} below {DELTA:g}')
        bits['gap'] = min(bits['gap'], -worst)
        rl = live.any(1)                                                    # (R, max_len): slots any token reads
        W = V * vs[..., None] * rl[:, None, :, None]
        g = gran(W)
        tot = _sums(c, vis, np.abs(W))
        bits['sum'] = max(bits['sum'], _fits(tot, g, f'{what}: sum of V over a visible set'))
        # stale partials (chunks / blocks before the maximum, wiped by a weight of exactly 0) stay finite
        big = float(np.abs(W).sum(2).max(initial=0.0)) / float(vs.min(initial=1.0))
        if not (big < FLT_MAX and max_len < FLT_MAX):
            raise BudgetError(f'{what}: a stale partial overflows fp32')
        if c.fp8:
            # P = p s_v / sm a normal fp16; O' = O / c and its rescales alpha c / sm stay above the fp32 normal range
            vr = np.where(rl[:, None], vs, np.nan)
            lo, hi = np.nanmin(vr, 2), np.nanmax(vr, 2)
            if not np.all(lo / hi >= 2.0 ** -14):
                raise BudgetError(f'{what}: s_v / max s_v below the fp16 normal range')
            if not g / float(np.nanmax(hi)) >= 2.0 ** -126:
                raise BudgetError(f'{what}: O / c leaves the fp32 normal range')
    return bits


def _sums(c, vis, W):
    """sum over the visible slots of W (R, nkv, max_len, hd) -> (R, T, nh, hd)."""
    R, T, nh, L = vis.shape
    nkv, G = W.shape[1], c.G
    v = vis.reshape(R, T, nkv, G, L).transpose(0, 2, 1, 3, 4).reshape(R, nkv, T * G, L).astype(np.float64)
    O = np.matmul(v, W)                                                     # (R, nkv, T G, hd)
    return O.reshape(R, nkv, T, G, -1).transpose(0, 2, 1, 3, 4).reshape(R, T, nh, -1)


def exact_sums(c, rows):
    """-> (O (R, T, nh, hd), L (R, T, nh)) float64: the sum of the dequantized V rows over each token's visible set
    and its size (0 for a token that is not computed)."""
    _, V, _, vs = c.slots(rows)
    vis, _ = visible(c, rows)
    return _sums(c, vis, V * vs[..., None]), vis.sum(3).astype(np.float64)


def reference(c):
    """-> (out (B, T, nh, hd) fp16, ties): fp16_rn(fp32(O) / fp32(L)) per computed token; +0 for the tokens of a valid
    row past its count; NaN for rows the kernel must not look at.  ties counts outputs whose fp32 quotient is an fp16
    midpoint."""
    B, T, nh, nkv, hd, max_len = c.shape
    out = np.zeros((B, T, nh, hd), np.float16)
    for b in range(B):
        if not c.valid(b):
            out[b] = np.nan
    ties = 0
    for rows in _row_blocks(c):
        O, L = exact_sums(c, rows)
        comp = L > 0
        with np.errstate(divide='ignore', invalid='ignore'):
            quo = (O.astype(np.float32) / L.astype(np.float32)[..., None]).astype(np.float32)
        quo = np.where(comp[..., None], quo, np.float32(0))
        ties += int(is_fp16_tie(quo).sum())
        out[rows] = quo.astype(np.float16)
    return out, ties


# --------------------------------------------------------------------------------------------------------------
# the kernels' algorithms in fp32 numpy, with mutations
# --------------------------------------------------------------------------------------------------------------
EXTEND_MUTATIONS = ('mask_short', 'mask_long', 'mask_tile', 'token_of_row', 'gqa_mod', 'stale_new', 'ks_prev',
                    'ks_next', 'vs_prev', 'vs_next', 'l_sv', 'combine_pos', 'rcp', 'f64')
PREFILL_MUTATIONS = ('mask_short', 'mask_long', 'mask_tile', 'token_of_row', 'gqa_mod', 'stale_new', 'no_rescale',
                     'c_stale', 'ks_prev', 'ks_next', 'vs_prev', 'vs_next', 'l_sv', 'count_long', 'rcp', 'f64')
FP8_ONLY = ('c_stale', 'ks_prev', 'ks_next', 'vs_prev', 'vs_next', 'l_sv')


def _fma32(a, b, acc):
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(acc, np.float64)).astype(np.float32)


def _slot_order(n, order, rng):
    idx = np.arange(n)
    if order == 'reversed':
        return idx[::-1]
    if order == 'random':
        return rng.permutation(idx)
    return idx


def _row_setup(c, b, mutation, T_comp):
    """Per-row inputs of a simulation: K, V, ks, vs (nkv, max_len[, hd]) as read, kv head of each q head, the last
    slot lim (T, nh) each (token, head) sees, and the scores s (T, nh, max_len) fp32 (-inf past lim)."""
    B, T, nh, nkv, hd, max_len = c.shape
    G = c.G
    pos = int(c.positions[b])
    K, V, ks, vs = (a[0] for a in c.slots([b], pre=mutation == 'stale_new'))
    if mutation in ('ks_prev', 'ks_next', 'vs_prev', 'vs_next'):
        j = np.clip(np.arange(max_len) + (-1 if mutation.endswith('prev') else 1), 0, max_len - 1)
        if mutation[0] == 'k':
            ks = ks[:, j]
        else:
            vs = vs[:, j]
    kv = np.arange(nh) % nkv if mutation == 'gqa_mod' else np.arange(nh) // G
    tok = np.repeat(np.arange(T)[:, None], nh, 1)                           # (T, nh): the token of row r = i G + g
    if mutation == 'token_of_row':
        tok = (np.arange(T)[:, None] * G + np.arange(nh)[None, :] % G) % T
    lim = pos + tok + {'mask_short': -1, 'mask_long': 1}.get(mutation, 0)
    if mutation == 'mask_tile':                                             # every row masked at its tile's last token
        r = np.arange(T)[:, None] * G + np.arange(nh)[None, :] % G
        tile_last = np.minimum(((r // TILE) * TILE + TILE - 1) // G, T_comp - 1)
        lim = pos + tile_last
    lim = np.minimum(lim, max_len - 1)
    q = c.q[b].astype(np.float64)
    d = np.einsum('thd,hjd->thj', q, K[kv])
    s = (d.astype(np.float32) * np.float32(c.scale)).astype(np.float32)
    if c.fp8:
        s = (s * ks[kv][None].astype(np.float32)).astype(np.float32)
    seen = np.arange(max_len)[None, None, :] <= lim[..., None]
    s = np.where(seen, s, -np.inf).astype(np.float32)
    return K, V, ks, vs, kv, lim, s, seen


def _f64(c, b, K, V, ks, vs, kv, seen):
    q = c.q[b].astype(np.float64)
    d = np.einsum('thd,hjd->thj', q, K[kv]) * c.scale * (ks[kv][None] if c.fp8 else 1.0)
    d = np.where(seen, d, -np.inf)
    w = np.exp(d - d.max(2, keepdims=True))
    w /= w.sum(2, keepdims=True)
    return np.einsum('thj,hjd->thd', w, (V * vs[..., None])[kv]).astype(np.float16)


def _quotient(O, L, mutation):
    with np.errstate(divide='ignore', invalid='ignore'):
        if mutation == 'rcp':
            return (O * (np.float32(1) / L)[..., None]).astype(np.float32).astype(np.float16)
        return (O / L[..., None]).astype(np.float32).astype(np.float16)


def simulate_extend(c, order='natural', mutation=None, seed=0):
    """attn_extend_split_kernel + the combine in fp32: per 64-slot chunk the max m, p = expf(s - m), e4m3 P =
    fp16(p s_v / sm) with sm the largest v scale the token sees in the chunk, l = sum p and o = sm sum P V in `order`;
    then the combine over chunks 0 .. (pos + i) / 64 ascending, M = max m, w = expf(m - M), L = fmaf(l, w, L),
    O = fmaf(o, w, O), fp16_rn(O / L).  `mutation` (one of EXTEND_MUTATIONS) restates a plausible defect."""
    assert c.kernel == 'extend'
    B, T, nh, nkv, hd, max_len = c.shape
    rng = np.random.default_rng(seed)
    out = np.full((B, T, nh, hd), np.nan, np.float16)
    for b in range(B):
        if not c.valid(b):
            continue
        pos = int(c.positions[b])
        K, V, ks, vs, kv, lim, s, seen = _row_setup(c, b, mutation, T)
        if mutation == 'f64':
            out[b] = _f64(c, b, K, V, ks, vs, kv, seen)
            continue
        ns = (pos + (0 if mutation == 'combine_pos' else np.arange(T)[:, None])) // BLOCK + 1
        ns = np.broadcast_to(ns, (T, nh))
        nchunk = int(ns.max())
        ms, ls, os_ = [], [], []
        for k in range(nchunk):
            j0, j1 = k * BLOCK, min(max_len, (k + 1) * BLOCK)
            sk = s[:, :, j0:j1]
            m = sk.max(2)
            with np.errstate(invalid='ignore'):
                p = np.where(np.isfinite(m)[..., None], np.exp((sk - m[..., None]).astype(np.float32)), 0).astype(np.float32)
            svk = vs[kv, j0:j1][None]                                       # (1, nh, n)
            if c.fp8:
                sm = np.where(seen[:, :, j0:j1], svk, 0).max(2)
                sm = np.where(sm > 0, sm, 1).astype(np.float32)
                P = np.where(p > 0, p * (svk.astype(np.float32) * (np.float32(1) / sm)[..., None]), 0).astype(np.float16)
            else:
                sm = np.ones((T, nh), np.float32)
                P = p.astype(np.float16)
            P = P.astype(np.float32)
            lacc = np.zeros((T, nh), np.float32)
            oacc = np.zeros((T, nh, hd), np.float32)
            for i in _slot_order(j1 - j0, order, rng):
                lacc = (lacc + (p[..., i] * svk[..., i] if mutation == 'l_sv' else p[..., i])).astype(np.float32)
                oacc = _fma32(P[..., i, None], V[kv, j0 + i][None], oacc)
            ms.append(m)
            ls.append(lacc)
            os_.append((oacc * sm[..., None]).astype(np.float32))
        ms = np.array(ms)
        used = np.arange(nchunk)[:, None, None] < ns[None]
        M = np.where(used, ms, -np.inf).max(0)
        L = np.zeros((T, nh), np.float32)
        O = np.zeros((T, nh, hd), np.float32)
        for k in range(nchunk):
            with np.errstate(invalid='ignore'):
                w = np.exp((ms[k] - M).astype(np.float32)).astype(np.float32)
            L = np.where(used[k], _fma32(ls[k], w, L), L)
            O = np.where(used[k][..., None], _fma32(os_[k], w[..., None], O), O)
        out[b] = _quotient(O, L, mutation)
    return out


def simulate_prefill(c, order='natural', mutation=None, seed=0):
    """attn_prefill_kernel in fp32: 64-slot blocks 0 .. (pos + last token) / 64, online max m, alpha = expf(m - m_new),
    l = l alpha + sum p; e4m3 sm = the largest v scale the token sees in the block, f = alpha c / sm, c = sm and
    P = fp16(p s_v / sm); O = O f + sum P V in `order`; fp16_rn(O c / l).  Tokens past the count are +0.  `mutation`
    (one of PREFILL_MUTATIONS) restates a plausible defect."""
    assert c.kernel == 'prefill'
    B, T, nh, nkv, hd, max_len = c.shape
    rng = np.random.default_rng(seed)
    out = np.full((B, T, nh, hd), np.nan, np.float16)
    for b in range(B):
        if not c.valid(b):
            continue
        out[b] = 0
        n = c.count(b)
        T_comp = T if mutation == 'count_long' else n
        if T_comp == 0:
            continue
        K, V, ks, vs, kv, lim, s, seen = _row_setup(c, b, mutation, T_comp)
        if mutation == 'f64':
            out[b, :T_comp] = _f64(c, b, K, V, ks, vs, kv, seen)[:T_comp]
            continue
        nblk = int(lim[:T_comp].max()) // BLOCK + 1
        m = np.full((T, nh), -np.inf, np.float32)
        l = np.zeros((T, nh), np.float32)
        cc = np.ones((T, nh), np.float32)
        O = np.zeros((T, nh, hd), np.float32)
        for kb in range(nblk):
            j0, j1 = kb * BLOCK, min(max_len, (kb + 1) * BLOCK)
            x = s[:, :, j0:j1]
            mn = np.maximum(m, x.max(2))
            with np.errstate(invalid='ignore'):
                alpha = np.exp((m - mn).astype(np.float32)).astype(np.float32)
                p = np.exp((x - mn[..., None]).astype(np.float32)).astype(np.float32)
            if mutation == 'no_rescale':
                alpha = np.ones_like(alpha)
            m = mn
            svk = vs[kv, j0:j1][None].astype(np.float32)
            lsum = np.zeros((T, nh), np.float32)
            for i in _slot_order(j1 - j0, order, rng):
                lsum = (lsum + (p[..., i] * svk[..., i] if mutation == 'l_sv' else p[..., i])).astype(np.float32)
            l = (l * alpha + lsum).astype(np.float32)
            f = alpha
            if c.fp8:
                sm = np.where(seen[:, :, j0:j1], svk, 0).max(2).astype(np.float32)
                hit = sm > 0
                fs = ((alpha if mutation == 'c_stale' else alpha * cc) / np.where(hit, sm, 1)).astype(np.float32)
                f = np.where(hit, fs, alpha)
                cc = np.where(hit, sm, cc)
                vn = (np.float32(1) / np.where(hit, sm, 1)).astype(np.float32)
                p = np.where(hit[..., None] & (p > 0), p * (svk * vn[..., None]), p).astype(np.float32)
            O = (O * f[..., None]).astype(np.float32)
            P = p.astype(np.float16).astype(np.float32)
            acc = np.zeros((T, nh, hd), np.float32)
            for i in _slot_order(j1 - j0, order, rng):
                acc = _fma32(P[..., i, None], V[kv, j0 + i][None], acc)
            O = (O + acc).astype(np.float32)
        if c.fp8:
            O = (O * cc[..., None]).astype(np.float32)
        out[b, :T_comp] = _quotient(O, l, mutation)[:T_comp]
    return out


def simulate(c, **kw):
    with np.errstate(invalid='ignore', divide='ignore', over='ignore'):
        return (simulate_extend if c.kernel == 'extend' else simulate_prefill)(c, **kw)


# --------------------------------------------------------------------------------------------------------------
# case construction
# --------------------------------------------------------------------------------------------------------------
def _select_causal(kind, pos, n, rng):
    """S_h (slot indices in 0 .. pos + n - 1, one of them <= pos) of a head of a row with n >= 1 counted tokens."""
    hi = pos + n - 1
    if kind == 'new':
        S = list(range(pos, pos + n)) + ([int(rng.integers(0, pos))] if pos > 0 else [])
    elif kind == 'last_new':
        S = [int(rng.integers(0, pos + 1)), hi]
    elif kind == 'block_edge':
        S = [j for k in range(BLOCK, hi + 1, BLOCK) for j in (k - 1, k)]
    elif kind == 'pos':
        S = [pos]
    elif kind == 'tie14':
        S = list(_select(kind, pos, BLOCK, rng))                     # every token sees the whole tie
    else:
        S = list(_select(kind, hi, BLOCK, rng))
    if not any(j <= pos for j in S):
        S.append(int(rng.integers(0, pos + 1)))
    return np.unique(np.array(S, np.int64))


def make_case(kernel, fp8, hd, G, nkv, max_len, T, positions, counts=None, seed=0, scale=None):
    """A multi-token case (module docstring).  counts: the prefill counts (None: T for every row, the extend rule).
    Rows the kernel must not look at select nothing.  The cache is built in integer cache units (int8 K, int16 V in
    units of 1 / V_DEN for fp16), as in exact_attn.make_case."""
    assert kernel in ('extend', 'prefill')
    rng = np.random.default_rng(seed)
    positions = np.asarray(positions, np.int64)
    B, nh = len(positions), G * nkv
    counts = np.full(B, T, np.int64) if counts is None else np.asarray(counts, np.int64)
    scale = float(np.float32(scale if scale is not None else 1.0 / np.sqrt(hd)))
    g_of_d = np.arange(hd) % G
    P = rng.integers(1, 4, size=hd).astype(np.int8)
    P[:G] = 0                                                       # the first dimension of each head: free
    P2 = np.array([np.sum(P[g_of_d == g].astype(np.int64) ** 2) for g in range(G)])
    cg = np.ldexp(1.0, np.ceil(np.log2(8 * DELTA / (P2 * scale))).astype(int))
    c0 = CausalCase(kernel, fp8, scale, np.zeros((B, T, nh, hd), np.float16), None, None,
                    np.zeros((B, nkv, max_len, hd), np.float16), None, None, None, positions, counts, None, None)
    c0.k_new = np.zeros((B, T, nkv, hd), np.float16)
    cnt = np.array([c0.count(b) for b in range(B)])

    sel = np.zeros((B, nh, max_len), bool)
    zero = np.zeros((B, T, nh), bool)
    kinds = []
    for b in range(B):
        p, n = int(positions[b]), int(cnt[b])
        kinds.append([KINDS[(b * nh + h + seed) % len(KINDS)] if n > 0 else 'none' for h in range(nh)])
        for h, kind in enumerate(kinds[-1]):
            if kind == 'none':
                continue
            sel[b, h, _select_causal(kind, p, n, rng)] = True
            if kind == 'uniform':
                zero[b, :, h] = True
            elif kind != 'tie14':
                zero[b, :, h] = rng.integers(0, ZERO_EVERY, size=T) == 0
    own = g_of_d[None, :] == (np.arange(nh) % G)[:, None]           # (nh, hd): the dimensions of head h
    tscale = np.ldexp(1.0, np.arange(T) % 3)                        # q of token i: c_g P 2^(i mod 3)
    q = np.where(own, cg[g_of_d] * P, 0.0)[None, None] * tscale[None, :, None, None] * ~zero[..., None]

    sig = np.where(sel.reshape(B, nkv, G, max_len).transpose(0, 1, 3, 2), 1, -1).astype(np.int8)
    K = rng.integers(-8, 9, size=(B, nkv, max_len, hd), dtype=np.int8)
    K = np.where(P > 0, sig[..., g_of_d] * P, K)
    del sig
    slot = np.arange(max_len)
    if fp8:
        V = rng.integers(-16, 17, size=(B, nkv, max_len, hd), dtype=np.int16)
        V[..., 0], V[..., 1], V[..., 2] = slot // 256, (slot // 16) % 16, slot % 16
        ke = _walk(rng, (B, nkv, max_len), -2, 2)
        ve = _walk(rng, (B, nkv, max_len), -2, 2)
        _merge_scales(ke, sel, kinds, G)
    else:
        V = rng.integers(-32 * V_DEN, 32 * V_DEN + 1, size=(B, nkv, max_len, hd), dtype=np.int16)
        V[..., 0], V[..., 1] = (slot // 64) * V_DEN, (slot % 64) * V_DEN
        for b in range(B):                                          # ties: O / L = m exactly on dimension hd - 1 - g
            for h in range(nh):
                js = np.nonzero(sel[b, h])[0]
                if kinds[b][h] != 'tie14' or len(js) % 2:
                    continue
                k = int(rng.integers(1376, 2048)) // 2 * 2 + b % 2
                V[b, h // G, js, hd - 1 - h % G] = 2 * k + 1 + np.where(np.arange(len(js)) % 2, 1, -1)

    # new slots: k_new / v_new carry the intended content; the cache holds a decoy there before the call
    k_new = rng.integers(-8, 9, size=(B, T, nkv, hd)).astype(np.float64)
    v_new = rng.integers(-8, 9, size=(B, T, nkv, hd)).astype(np.float64)
    intended = []
    for b in range(B):
        p = int(positions[b])
        for i in range(int(cnt[b])):
            j = p + i
            kr, vr = K[b, :, j].astype(np.float64), V[b, :, j].astype(np.float64)
            if fp8:
                kr[:, 0] = E4M3_MAX * rng.choice([-1.0, 1.0], nkv)     # a free dimension: amax = 448
                vr[:, 3] = E4M3_MAX * rng.choice([-1.0, 1.0], nkv)
                k_new[b, i] = kr * np.ldexp(1.0, ke[b, :, j])[:, None]
                v_new[b, i] = vr * np.ldexp(1.0, ve[b, :, j])[:, None]
                intended.append((b, i, kr, vr, ke[b, :, j], ve[b, :, j]))
            else:
                k_new[b, i], v_new[b, i] = kr, vr / V_DEN
            K[b, :, j] = np.where(P > 0, -K[b, :, j], K[b, :, j][:, ::-1])
            V[b, :, j] = V[b, :, j][:, ::-1]
    if fp8:
        kc, vc = e4m3_bytes(K), e4m3_bytes(V)
        ksc = np.ldexp(1.0, ke).astype(np.float32)
        vsc = np.ldexp(1.0, ve).astype(np.float32)
        for b in range(B):
            p, n = int(positions[b]), int(cnt[b])
            ksc[b, :, p:p + n] *= 8
            vsc[b, :, p:p + n] *= 8
    else:
        kc, vc = K.astype(np.float16), (V / np.float32(V_DEN)).astype(np.float16)
        ksc = vsc = None
    q16, kn16, vn16 = q.astype(np.float16), k_new.astype(np.float16), v_new.astype(np.float16)
    assert np.array_equal(q16, q) and np.array_equal(kn16, k_new) and np.array_equal(vn16, v_new)
    c = CausalCase(kernel, fp8, scale, q16, kn16, vn16, kc, vc, ksc, vsc, positions, counts, sel, zero, kinds)
    if fp8:                                                         # the quantizer reproduces the intended bytes
        kq, kqs, vq, vqs = c.new_quantized()
        for b, i, kr, vr, kej, vej in intended:
            assert np.array_equal(E4M3[kq[b, i]], kr) and np.array_equal(kqs[b, i], np.ldexp(1.0, kej))
            assert np.array_equal(E4M3[vq[b, i]], vr) and np.array_equal(vqs[b, i], np.ldexp(1.0, vej))
    return c
