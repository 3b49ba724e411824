"""Exactly representable cases for the decode-attention kernels.  TEST INFRASTRUCTURE ONLY.

The kernels are quip_decode_attention's, on fp16 and e4m3 caches (csrc/attn_decode.cu).  Softmax is not exact in
general, because expf is not correctly rounded.  It is exact when every score of a head either equals the head's maximum
bit for bit or lies at least DELTA = 128 below it: expf(0) = 1, and e^-128 ~ 2.6e-56 is far below the smallest fp32
subnormal 2^-149 ~ 1.4e-45, so expf(x <= -128) = 0.  Attention then returns exactly the mean of the V rows of the
selected slots S_h, and the kernel's arithmetic reduces to sums a budget can prove exact:

  * in a chunk (64 or 128 slots) that holds a slot of S_h, m = the maximum, p = 1 on S_h and 0 elsewhere, l = the count
    and o = the sum of V over the chunk's part of S_h (e4m3: of p * s_v * V8, each product exact, see below);
  * a chunk without a slot of S_h has m_chunk <= M - DELTA, so the combine weighs it by expf(m_chunk - M) = 0, and
    fmaf(x, 0, acc) = acc as long as its l and o are finite;
  * the combine then holds L = |S_h| and O = sum_{j in S_h} V_j and returns fp16_rn(fp32(O) / fp32(L)), one IEEE fp32
    division and one fp16 round to nearest even.

Construction (make_case).  Head g of a kv group owns the dimensions d = g (mod G).  q_h = c_g P on those dimensions and 0
elsewhere, with P a pattern of small integers that is 0 on the group's first dimension.  K[j] holds sigma_{j,h} P there,
sigma = +1 on S_h and -1 elsewhere, so the score is +-c_g |P_g|^2 scale (times the slot's k scale for e4m3).  The
dimensions where P is 0 are free: random values there, and 448 in k_new for the e4m3 cache.  A head with q = 0 attends
uniformly over 0..pos.  V rows are small dyadic values; the first dimensions spell the slot index, so a mismatch can name
the slot that was read.  'tie' heads get V values m +- 1/8 around an fp16 midpoint m on a dimension of their own, so
O / L = m exactly: a tie that only round to nearest even resolves.

e4m3.  Cache bytes and power-of-two scales are written directly.  K scales are equal across each S_h of a q != 0 head
(the union of overlapping sets shares one scale) and random elsewhere; V scales change from slot to slot.  k_new / v_new
are 2^a times e4m3 values with amax 448, so the kernel's quantizer (s = amax / 448 = 2^a) stores exactly those bytes.

Budget (check_budget).  Per row, it raises BudgetError unless:
  * the dot products q . K are exact in fp32 in any order: sum |q K| <= 2^24 gran(q) gran(K);
  * after the kernel's fp32 roundings (d * scale, then * k_scale) every slot of S_h scores the row maximum bit for bit
    and every other slot scores at least DELTA below it, the difference taken in fp32 as the kernel takes it;
  * every partial sum of O (per slot group, warp, chunk, and in the combine) is exact in any order: for every (head,
    dimension), sum_{j in S_h} |s_v V_j| <= 2^24 times the granularity of the row's values (p s_v V is exact: s_v is a
    power of two and V an fp16 or e4m3 value);
  * the o and l of a chunk without a selected slot stay finite (at most 128 |V| s_v and 128).

Rounding of the quotient.  Under this budget, fp16_rn(fp32(O / L)) equals fp16_rn(O / L) rounded once from the exact
quotient, for L <= 2^13: an fp32 rounding can only change the fp16 result by landing on an fp16 midpoint m that O / L
is not, which needs |O - L m| < L ulp32(m) / 2 and so |O| > 2^24 times its granularity.  What the fp32 quotient pins is
the tie itself: when O / L = m exactly, round to nearest even decides, and a reciprocal multiply or a float64 softmax
(inexact weights 1 / L, nonzero e^-gap terms) can land on either side of m.
"""
from dataclasses import dataclass, field

import numpy as np

from .exact import BudgetError, _fits
from .exact_quant import gran

DELTA = 128.0
E4M3_MAX = 448.0
KINDS = ('uniform', 'pos', 'zero', 'all', 'chunk_last', 'boundary', 'rand3', 'rand7', 'tie14')
V_DEN = 8                       # fp16 V values are k / 8
FLT_MAX = float(np.finfo(np.float32).max)


def _e4m3_table():
    import torch
    return torch.arange(256, dtype=torch.int32).to(torch.uint8).view(torch.float8_e4m3fn).to(torch.float64).numpy()


E4M3 = _e4m3_table()


def e4m3_bytes(x):
    """float64 values that are e4m3 values -> their bytes (asserts exactness)."""
    import torch
    x = np.asarray(x, np.float32)
    out = torch.from_numpy(x).to(torch.float8_e4m3fn).view(torch.uint8).numpy()
    assert np.array_equal(E4M3.astype(np.float32)[out], x), 'not an e4m3 value'
    return out


@dataclass
class AttnCase:
    """One kernel call.  Arrays are numpy; caches are fp16, or e4m3 bytes (uint8) with fp32 scales."""
    fp8: bool
    chunk: int                  # the kernel's chunk for (B, nkv, max_len)
    scale: float                # an fp32 value
    q: np.ndarray               # (B, nh, hd) fp16
    k_new: np.ndarray           # (B, nkv, hd) fp16
    v_new: np.ndarray
    k_cache: np.ndarray         # (B, nkv, max_len, hd) fp16 or uint8
    v_cache: np.ndarray
    k_scale: object             # (B, nkv, max_len) fp32, or None
    v_scale: object
    positions: np.ndarray       # (B,) int64
    sel: np.ndarray             # (B, nh, max_len) bool: S_h (all False for a row out of range)
    kinds: list = field(default_factory=list)   # (B, nh) kind names

    @property
    def shape(self):
        B, nh, hd = self.q.shape
        nkv, max_len = self.k_cache.shape[1], self.k_cache.shape[2]
        return B, nh, nkv, hd, max_len

    @property
    def G(self):
        return self.q.shape[1] // self.k_new.shape[1]

    def valid(self, b):
        return 0 <= int(self.positions[b]) < self.k_cache.shape[2]

    def new_quantized(self):
        """(k bytes, k scale, v bytes, v scale) of k_new / v_new as the kernel quantizes them (oracle/kvfp8.quantize)."""
        if '_newq' not in self.__dict__:
            import torch
            from . import kvfp8
            out = []
            for x in (self.k_new, self.v_new):
                qb, s = kvfp8.quantize(torch.from_numpy(x))
                out += [qb.view(torch.uint8).numpy(), s.numpy()]
            self._newq = out
        return self._newq


def row_slots(c, rows, pre=False):
    """Rows (an index array) as the kernel reads them -> K, V (R, nkv, max_len, hd) float64 in cache units (fp16 values
    or e4m3 values) and ks, vs (R, nkv, max_len) float64 (ones for fp16).  Slot positions[b] of a valid row holds
    k_new / v_new (their quantization for e4m3), unless pre: then it holds what the cache held before the call."""
    rows = np.asarray(rows)
    if c.fp8:
        K, V = E4M3[c.k_cache[rows]], E4M3[c.v_cache[rows]]
        ks, vs = c.k_scale[rows].astype(np.float64), c.v_scale[rows].astype(np.float64)
    else:
        K, V = c.k_cache[rows].astype(np.float64), c.v_cache[rows].astype(np.float64)
        ks = vs = np.ones(K.shape[:3])
    if pre:
        return K, V, ks, vs
    i = np.array([r for r, b in enumerate(rows) if c.valid(b)], np.int64)
    if len(i):
        b, p = rows[i], c.positions[rows[i]]
        if c.fp8:
            kq, kqs, vq, vqs = c.new_quantized()
            ks, vs = ks.copy(), vs.copy()
            K[i, :, p], V[i, :, p], ks[i, :, p], vs[i, :, p] = E4M3[kq[b]], E4M3[vq[b]], kqs[b], vqs[b]
        else:
            K[i, :, p], V[i, :, p] = c.k_new[b], c.v_new[b]
    return K, V, ks, vs


def fp32_scores(c, rows, K, ks):
    """The kernel's scores (R, nh, n) fp32 of rows whose K / ks (R, nkv, n, hd) / (R, nkv, n) come from row_slots:
    fp32(d * scale), times k_scale for e4m3 (d is exact by the budget)."""
    R, nkv, n, hd = K.shape
    q = c.q[rows].astype(np.float64).reshape(R, nkv, -1, hd)
    d = np.einsum('rkgd,rkjd->rkgj', q, K)
    s = (d.astype(np.float32) * np.float32(c.scale)).astype(np.float32)
    if c.fp8:
        s = (s * ks[:, :, None].astype(np.float32)).astype(np.float32)
    return s.reshape(R, -1, n)


def _row_blocks(c, elems=1 << 22):
    """The valid rows in blocks of about `elems` cached values."""
    B, nh, nkv, hd, max_len = c.shape
    rows = np.array([b for b in range(B) if c.valid(b)], np.int64)
    step = max(1, elems // (nkv * max_len * hd))
    return [rows[i:i + step] for i in range(0, len(rows), step)]


# --------------------------------------------------------------------------------------------------------------
# budget and reference
# --------------------------------------------------------------------------------------------------------------
def check_budget(c):
    """Raise BudgetError unless the case meets the exactness premise (module docstring).  Returns the bits used
    {'dot': ..., 'sum': ..., 'gap': smallest score gap}.  The granularities are taken over a block of rows, which
    only makes the bounds stricter."""
    B, nh, nkv, hd, max_len = c.shape
    bits = dict(dot=0.0, sum=0.0, gap=np.inf)
    for rows in _row_blocks(c):
        K, V, ks, vs = row_slots(c, rows)
        live = np.arange(max_len)[None, :] <= c.positions[rows][:, None]          # (R, max_len): slots 0..pos
        sel = c.sel[rows]
        what = f'rows {rows[0]}..{rows[-1]}'
        if (sel & ~live[:, None]).any():
            raise BudgetError(f'{what}: a selected slot past the position')
        if not sel.any(2).all():
            raise BudgetError(f'{what}: a head with an empty selected set')
        q = c.q[rows].astype(np.float64).reshape(len(rows), nkv, -1, hd)
        dot = np.einsum('rkgd,rkjd->rkgj', np.abs(q), np.abs(K))
        bits['dot'] = max(bits['dot'], _fits(dot, gran(q) * gran(K), f'{what}: q . K'))
        s = fp32_scores(c, rows, K, ks)
        s = np.where(live[:, None], s, -np.inf).astype(np.float32)
        M = np.where(sel, s, -np.inf).max(2)
        if not np.array_equal(M, s.max(2)) or not np.all(np.where(sel, s == M[..., None], True)):
            raise BudgetError(f'{what}: the selected slots do not all score the row maximum bit for bit')
        gap = (s - M[..., None]).astype(np.float32)
        worst = float(np.where(sel | ~live[:, None], -np.inf, gap).max(initial=-np.inf))
        if worst > -DELTA:
            raise BudgetError(f'{what}: score gap {-worst:.6g} below {DELTA:g}')
        bits['gap'] = min(bits['gap'], -worst)
        terms = np.abs(V * vs[..., None]) * live[:, None, :, None]               # (R, nkv, max_len, hd)
        g = gran(V * vs[..., None] * live[:, None, :, None])
        tot = np.einsum('rkgj,rkjd->rkgd', sel.reshape(len(rows), nkv, -1, max_len).astype(np.float64), terms)
        bits['sum'] = max(bits['sum'], _fits(tot, g, f'{what}: sum of V over S_h'))
        if not float(terms.max(initial=0.0)) * 128 < FLT_MAX:
            raise BudgetError(f'{what}: a chunk partial overflows fp32')
    return bits


def exact_sums(c, rows):
    """-> (O (R, nh, hd), L (R, nh)) float64 of valid rows: the sums over S_h of the dequantized V rows, and |S_h|."""
    _, V, _, vs = row_slots(c, rows)
    R, nkv, max_len, hd = V.shape
    sel = c.sel[rows].astype(np.float64)
    O = np.einsum('rkgj,rkjd->rkgd', sel.reshape(R, nkv, -1, max_len), V * vs[..., None])
    return O.reshape(R, -1, hd), sel.sum(2)


def is_fp16_tie(x32):
    """fp32 values that lie exactly halfway between two adjacent fp16 values."""
    x = np.asarray(x32, np.float32).astype(np.float64)
    r16 = x.astype(np.float16)
    r = r16.astype(np.float64)
    nb = np.nextafter(r16, np.where(x > r, np.inf, -np.inf).astype(np.float16)).astype(np.float64)
    return (x != r) & (2 * np.abs(x - r) == np.abs(nb - r))


def reference(c):
    """-> (out (B, nh, hd) fp16, ties): fp16_rn(fp32(O) / fp32(L)) per head, NaN rows for positions out of range; ties
    counts outputs whose fp32 quotient is an fp16 midpoint."""
    B, nh, nkv, hd, max_len = c.shape
    out = np.full((B, nh, hd), np.nan, np.float16)
    ties = 0
    for rows in _row_blocks(c):
        O, L = exact_sums(c, rows)
        quo = O.astype(np.float32) / L.astype(np.float32)[..., None]
        ties += int(is_fp16_tie(quo).sum())
        out[rows] = quo.astype(np.float16)
    return out, ties


# --------------------------------------------------------------------------------------------------------------
# the kernel's algorithm in fp32 numpy, with mutations
# --------------------------------------------------------------------------------------------------------------
MUTATIONS = ('range_short', 'range_long', 'cache_at_pos', 'gqa_mod', 'combine_short', 'ks_prev', 'ks_next',
             'vs_prev', 'vs_next', 'l_sv', 'rcp', 'f64')
FP8_ONLY = ('ks_prev', 'ks_next', 'vs_prev', 'vs_next', 'l_sv')


def _fma32(a, b, acc):
    """fmaf in fp32 through float64: the product of two fp32 values is exact there; the sum is rounded twice, which the
    exact cases never notice."""
    return (np.asarray(a, np.float64) * np.asarray(b, np.float64) + np.asarray(acc, np.float64)).astype(np.float32)


def simulate(c, chunk=None, order='natural', mutation=None, seed=0):
    """The split-KV algorithm of csrc/attn_decode.cu in fp32: per chunk the max m, p = expf(s - m) (times s_v for
    e4m3), l = sum p and o = sum p V in `order` ('natural', 'reversed' or 'random'), then the ascending combine with
    M = max m, w = expf(m - M), L = fmaf(l, w, L), O = fmaf(o, w, O), and fp16_rn(O / L).  `mutation` (one of
    MUTATIONS) restates a plausible kernel defect instead; 'f64' is a float64 softmax rounded once to fp16."""
    B, nh, nkv, hd, max_len = c.shape
    chunk = chunk or c.chunk
    rng = np.random.default_rng(seed)
    kv = np.arange(nh) % nkv if mutation == 'gqa_mod' else np.arange(nh) // c.G
    out = np.full((B, nh, hd), np.nan, np.float16)
    for b in range(B):
        if not c.valid(b):
            continue
        pos = int(c.positions[b])
        K, V, ks, vs = (a[0] for a in row_slots(c, [b], pre=mutation == 'cache_at_pos'))
        if mutation in ('ks_prev', 'ks_next', 'vs_prev', 'vs_next'):
            pre = [a[0] for a in row_slots(c, [b], pre=True)]
            src = pre[2] if mutation[0] == 'k' else pre[3]
            step = -1 if mutation.endswith('prev') else 1
            j = np.arange(max_len)
            moved = src[:, np.clip(j + step, 0, max_len - 1)]
            moved[:, pos] = (ks if mutation[0] == 'k' else vs)[:, pos]     # the appended slot's scale is in shared memory
            if mutation[0] == 'k':
                ks = moved
            else:
                vs = moved
        n = pos + 1 + {'range_short': -1, 'range_long': 1}.get(mutation, 0)
        n = min(n, max_len)
        if mutation == 'f64':
            d = np.einsum('hd,hjd->hj', c.q[b].astype(np.float64), K[kv, :n]) * c.scale * ks[kv, :n]
            w = np.exp(d - d.max(1, keepdims=True))
            w /= w.sum(1, keepdims=True)
            out[b] = np.einsum('hj,hjd->hd', w, (V * vs[..., None])[kv, :n]).astype(np.float16)
            continue
        d = np.einsum('hd,hjd->hj', c.q[b].astype(np.float64), K[kv, :n])
        s = (d.astype(np.float32) * np.float32(c.scale)).astype(np.float32)
        if c.fp8:
            s = (s * ks[kv, :n].astype(np.float32)).astype(np.float32)
        ns = max(0, -(-n // chunk) - (mutation == 'combine_short'))
        ms, ls, os_ = [], [], []
        for k in range(ns):
            j0, j1 = k * chunk, min(n, (k + 1) * chunk)
            sk = s[:, j0:j1]
            m = sk.max(1)
            p = np.exp((sk - m[:, None]).astype(np.float32)).astype(np.float32)
            pv = (p * vs[kv, j0:j1].astype(np.float32)).astype(np.float32) if c.fp8 else p
            idx = np.arange(j1 - j0)
            if order == 'reversed':
                idx = idx[::-1]
            elif order == 'random':
                idx = rng.permutation(idx)
            lacc = np.zeros(nh, np.float32)
            oacc = np.zeros((nh, hd), np.float32)
            for i in idx:
                lacc = (lacc + (pv[:, i] if mutation == 'l_sv' else p[:, i])).astype(np.float32)
                oacc = _fma32(pv[:, i, None], V[kv, j0 + i], oacc)
            ms.append(m)
            ls.append(lacc)
            os_.append(oacc)
        M = np.max(ms, 0) if ms else np.full(nh, -np.inf, np.float32)
        L = np.zeros(nh, np.float32)
        O = np.zeros((nh, hd), np.float32)
        for m, l, o in zip(ms, ls, os_):
            w = np.exp((m - M).astype(np.float32)).astype(np.float32)
            L = _fma32(l, w, L)
            O = _fma32(o, w[:, None], O)
        with np.errstate(divide='ignore', invalid='ignore'):
            if mutation == 'rcp':
                quo = (O * (np.float32(1) / L)[:, None]).astype(np.float32)
            else:
                quo = (O / L[:, None]).astype(np.float32)
        out[b] = quo.astype(np.float16)
    return out


# --------------------------------------------------------------------------------------------------------------
# case construction
# --------------------------------------------------------------------------------------------------------------
def _select(kind, pos, chunk, rng):
    """S_h (sorted slot indices in 0..pos) of one head."""
    n = pos + 1
    if kind in ('uniform', 'all'):
        return np.arange(n)
    if kind == 'pos':
        return np.array([pos])
    if kind == 'zero':
        return np.array([0])
    if kind == 'chunk_last':                                        # the last valid slot of every chunk
        return np.minimum(np.arange(chunk - 1, pos + chunk, chunk), pos)
    if kind == 'boundary':                                          # 5 slots around the last chunk start <= pos
        e = max(chunk, (pos // chunk) * chunk)                      # (shifted into 0..pos when pos < chunk)
        lo = min(e - 2, max(0, n - 5))
        return np.arange(lo, min(n, lo + 5))
    size = {'rand3': 3, 'rand7': 7, 'tie14': 14}[kind]
    return np.sort(rng.choice(n, size=min(size, n), replace=False))


def _walk(rng, shape, lo, hi):
    """Random integer exponents in [lo, hi] along the last axis, each different from its predecessor."""
    e = rng.integers(lo, hi + 1, size=shape)
    for j in range(1, shape[-1]):
        same = e[..., j] == e[..., j - 1]
        e[..., j] = np.where(same, np.where(e[..., j] < hi, e[..., j] + 1, lo), e[..., j])
    return e


def _merge_scales(ke, sel, kinds, G):
    """One k-scale exponent per union of overlapping selected sets of the q != 0 heads of each (row, kv head)."""
    B, nkv, max_len = ke.shape
    for b in range(B):
        for k in range(nkv):
            lab = np.arange(max_len)
            for h in range(k * G, (k + 1) * G):
                if kinds[b][h] in ('uniform', 'none'):
                    continue
                hit = np.isin(lab, lab[sel[b, h]])
                lab[hit] = lab[hit].min()
            ke[b, k] = ke[b, k][lab]


def make_case(fp8, hd, G, nkv, max_len, positions, chunk, seed, scale=None):
    """A decode-attention case (module docstring).  positions may lie outside [0, max_len): such rows select nothing.
    The cache is built in integer cache units (int8 K, int16 V in units of 1 / V_DEN for fp16), which keeps the
    64-row, 4096-slot cases small."""
    rng = np.random.default_rng(seed)
    positions = np.asarray(positions, np.int64)
    B, nh = len(positions), G * nkv
    scale = float(np.float32(scale if scale is not None else 1.0 / np.sqrt(hd)))
    g_of_d = np.arange(hd) % G
    P = rng.integers(1, 4, size=hd).astype(np.int8)
    P[:G] = 0                                                       # the first dimension of each head: free
    P2 = np.array([np.sum(P[g_of_d == g].astype(np.int64) ** 2) for g in range(G)])
    # c_g: a power of two with c |P|^2 scale >= 8 DELTA, so that the gap holds for k scales down to 2^-2
    cg = np.ldexp(1.0, np.ceil(np.log2(8 * DELTA / (P2 * scale))).astype(int))
    valid = (positions >= 0) & (positions < max_len)

    sel = np.zeros((B, nh, max_len), bool)
    kinds = []
    for b in range(B):
        p = int(positions[b])
        kinds.append([KINDS[(b * nh + h + seed) % len(KINDS)] if valid[b] else 'none' for h in range(nh)])
        for h, kind in enumerate(kinds[-1]):
            if kind != 'none':
                sel[b, h, _select(kind, p, chunk, rng)] = True
    uniform = np.array([[k == 'uniform' for k in row] for row in kinds], bool).reshape(B, nh)
    own = g_of_d[None, :] == (np.arange(nh) % G)[:, None]          # (nh, hd): the dimensions of head h
    q = np.where(own, cg[g_of_d] * P, 0.0)[None] * ~uniform[..., None]

    # K[b, kvh, j, d] = sigma P[d] with sigma = +1 iff j is in S of head (kvh, d mod G); free where P = 0
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
                k = int(rng.integers(1376, 2048)) // 2 * 2 + b % 2    # m = (2k + 1) / 8 in (344, 512); even k ties down
                V[b, h // G, js, hd - 1 - h % G] = 2 * k + 1 + np.where(np.arange(len(js)) % 2, 1, -1)

    # slot pos: k_new / v_new carry the row's intended content; the cache holds something else before the call
    k_new = np.zeros((B, nkv, hd))
    v_new = np.zeros((B, nkv, hd))
    knew_f, vnew_f = np.zeros((B, nkv, hd)), np.zeros((B, nkv, hd))
    for b in range(B):
        p = int(positions[b]) if valid[b] else 0
        kr, vr = K[b, :, p].astype(np.float64), V[b, :, p].astype(np.float64)
        if fp8:
            kr[:, 0] = E4M3_MAX * rng.choice([-1.0, 1.0], nkv)         # a free dimension: amax = 448
            vr[:, 3] = E4M3_MAX * rng.choice([-1.0, 1.0], nkv)
            k_new[b] = kr * np.ldexp(1.0, ke[b, :, p])[:, None]
            v_new[b] = vr * np.ldexp(1.0, ve[b, :, p])[:, None]
        else:
            k_new[b], v_new[b] = kr, vr / V_DEN
        knew_f[b], vnew_f[b] = kr, vr
        if valid[b]:
            K[b, :, p] = np.where(P > 0, -K[b, :, p], K[b, :, p][:, ::-1])
            V[b, :, p] = V[b, :, p][:, ::-1]
    if fp8:
        kc, vc = e4m3_bytes(K), e4m3_bytes(V)
        ksc = np.ldexp(1.0, ke).astype(np.float32)
        vsc = np.ldexp(1.0, ve).astype(np.float32)
        rows = np.nonzero(valid)[0]
        ksc[rows, :, positions[rows]] *= 8                             # slot pos before the call: other scales
        vsc[rows, :, positions[rows]] *= 8
    else:
        kc, vc = K.astype(np.float16), (V / np.float32(V_DEN)).astype(np.float16)
        ksc = vsc = None
    q16, kn16, vn16 = q.astype(np.float16), k_new.astype(np.float16), v_new.astype(np.float16)
    assert np.array_equal(q16, q) and np.array_equal(kn16, k_new) and np.array_equal(vn16, v_new)
    c = AttnCase(fp8, chunk, scale, q16, kn16, vn16, kc, vc, ksc, vsc, positions, sel, kinds)
    if fp8:                                                         # the quantizer reproduces the intended bytes
        kq, kqs, vq, vqs = c.new_quantized()
        for b in np.nonzero(valid)[0]:
            p = int(positions[b])
            assert np.array_equal(E4M3[kq[b]], knew_f[b]) and np.array_equal(kqs[b], np.ldexp(1.0, ke[b, :, p]))
            assert np.array_equal(E4M3[vq[b]], vnew_f[b]) and np.array_equal(vqs[b], np.ldexp(1.0, ve[b, :, p]))
    return c
