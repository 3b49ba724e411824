"""Exactly representable cases for the quantizer kernels.  TEST INFRASTRUCTURE ONLY.

The kernels are the LDLQ and greedy column loops (csrc/ldlq.cu through quantize.ldlq_round) and the Hessian
accumulation (csrc/hessian.cu).  The construction follows oracle/exact.py: every partial sum is an integer multiple of a
granularity G and at most B in magnitude, so whenever B <= 2^24 G an fp32 accumulator holds it exactly in any summation
order.  A correct implementation then makes every rounding decision (ties included) on the exact value, and its codes
must equal those of a float64 restatement of the loop.

LDLQ.  H = C C^T with C unit lower triangular and a few off-diagonal entries k/16 (|k| <= 16) per row.  H is then exact
in fp32, its Cholesky factor is C itself (each step is an exact dyadic sum, a square root of 1 and a division by 1), and
the feedback matrix L = C - I is dyadic.  The rows of C are built so that diag(H) is strictly ascending with a
power-of-two maximum:
  * H / max diag(H), the greedy pass's matrix, is exact;
  * argsort(diag(H)) has no ties, so LDLQ-RG takes the same permutation on every device, and it sorts a scrambled copy
    of the case back to H = C C^T, whose factor is again C.  A scrambled H has no dyadic factor of its own.
w lies on a 2^-4 grid.  Two columns are exact half-integers: the last, which is rounded with no feedback, so the
rounding rule meets ties in w; and one inner column.  Rows 0 and 1 drive the clamps at 0 and 2^bits - 1.

The budget of a case is checked by its float64 reference while it runs.  For every column step it records the
order-independent bound |w_i| + sum_k |e_k L_ki| (greedy: |pre_i| + sum_k |s_k H_ki|) and raises BudgetError unless
it is <= 2^24 G.  That covers every FMA chain inside the kernels and every cuBLAS fp32 feedback GEMM of the host loop
(quantize.ldlq_round_cuda turns TF32 off).

Hessian.  X is fp16 integers |x| <= 2^8 times a per-feature power of two 2^e_i (outlier channels).  Every product of
the feature pair (i, j) is a multiple of 2^(e_i + e_j) and at most 2^16 times it, so a 256-token fp32 chunk sum is at
most 2^24 times its granularity: exact.  The float64 carry is exact far beyond any token count used here.
"""
from dataclasses import dataclass
from math import isqrt

import numpy as np

from .exact import BudgetError, _fits

W_DEN = 16                      # w on a 2^-4 grid
L_DEN = 16                      # off-diagonal entries of C: k / 16, |k| <= 16
F64_SPAN = float(1 << 53)
HS_CHUNK = 256                  # tokens summed in fp32 before the float64 carry (csrc/hessian.cu)


def gran_exp(a):
    """Elementwise exponent of the largest power of two dividing each entry; +inf for zeros and NaNs.

    A value that is not a short dyadic (1/3, 0.1) gets an exponent near -55, which no budget accepts."""
    a = np.asarray(a, np.float64)
    out = np.full(a.shape, np.inf)
    ok = np.isfinite(a) & (a != 0)
    m, e = np.frexp(np.abs(a[ok]))
    mi = np.ldexp(m, 53).astype(np.int64)
    low = mi & -mi
    out[ok] = e - 53 + np.log2(low.astype(np.float64))
    return out


def gran(a):
    """Largest power of two dividing every entry of a (1.0 for an all-zero array)."""
    g = gran_exp(a)
    return 1.0 if not np.isfinite(g).any() else float(2.0 ** g.min())


def _stats():
    return dict(ties=0, clamp_lo=0, clamp_hi=0, steps=0, bits=0.0)


# --------------------------------------------------------------------------------------------------------------
# the two column loops, in float64, with the kernels' rounding rules
# --------------------------------------------------------------------------------------------------------------
def half_up(v):
    """The LDLQ rule of the reference and the kernel: floor(v + 1/2)."""
    return np.floor(v + 0.5)


def ldlq_loop(base, w, L, top, st, rnd=half_up):
    """quip_ldlq_block on one block of n columns, rows independent: for j = n-1 .. 0
        v = base_j + sum_{k > j} e_k L_kj,   q_j = clamp(rnd(v), 0, top),   e_j = w_j - q_j.
    base (m, n), w (m, n), L (n, n): only the strictly lower part is read.  Returns (q, e) and adds to the stats `st`;
    raises BudgetError unless every feedback sum is exact in fp32."""
    m, n = base.shape
    Ls = np.tril(np.nan_to_num(L), -1)
    q = np.empty((m, n))
    e = np.zeros((m, n))
    G = min(gran(base), 0.5, min(gran(w), 1.0) * gran(Ls))
    worst = 0.0
    for j in range(n - 1, -1, -1):
        k = j + 1 + np.nonzero(Ls[j + 1:, j])[0]
        lk = Ls[k, j]
        v = base[:, j] + e[:, k] @ lk
        worst = max(worst, float((np.abs(base[:, j]) + np.abs(e[:, k]) @ np.abs(lk)).max(initial=0.0)) + 0.5)
        st['ties'] += int(np.count_nonzero(v - np.floor(v) == 0.5))
        r = rnd(v)
        st['clamp_lo'] += int(np.count_nonzero(r < 0))
        st['clamp_hi'] += int(np.count_nonzero(r > top))
        q[:, j] = np.clip(r, 0, top)
        e[:, j] = w[:, j] - q[:, j]
    st['steps'] += n
    st['bits'] = max(st['bits'], _fits(worst, G, 'LDLQ feedback sum'))
    return q, e


def greedy_sweep(pre, Hb, wr, s, st):
    """quip_greedy_block on one block of n columns, in place on wr / s (m, n): for i = n-1 .. 0
        hs = pre_i + sum_j s_j H_ji   (s as updated so far),
        wr_i <- rint(wr_i - hs / H_ii)   (half to even),   s_i moves with wr_i.
    The quotient and the difference are rounded to fp32 as the kernel does (both operands are fp32 values, and one
    rounding through float64 first does not change a correctly rounded / or -).  Raises BudgetError unless hs is
    exact in fp32."""
    n = Hb.shape[0]
    G = min(gran(pre), min(gran(s), 1.0) * gran(Hb))
    worst = 0.0
    for i in range(n - 1, -1, -1):
        k = np.nonzero(Hb[:, i])[0]
        hk = Hb[k, i]
        hs = pre[:, i] + s[:, k] @ hk
        worst = max(worst, float((np.abs(pre[:, i]) + np.abs(s[:, k]) @ np.abs(hk)).max(initial=0.0)))
        quo = (hs / Hb[i, i]).astype(np.float32).astype(np.float64)
        arg = (wr[:, i] - quo).astype(np.float32).astype(np.float64)
        st['ties'] += int(np.count_nonzero(arg - np.floor(arg) == 0.5))
        move = wr[:, i] - np.rint(arg)
        wr[:, i] -= move
        s[:, i] -= move
    st['steps'] += n
    st['bits'] = max(st['bits'], _fits(worst, G, 'greedy sum'))


# --------------------------------------------------------------------------------------------------------------
# end to end: quantize.ldlq_round / ldlq_rg_round
# --------------------------------------------------------------------------------------------------------------
@dataclass
class LdlqCase:
    bits: int
    C: np.ndarray               # (d, d) float64, unit lower triangular, off-diagonal k/16
    w: np.ndarray               # (m, d) float64 on the 2^-4 grid
    perm: np.ndarray            # (d,) the column order of the scrambled copy (LDLQ-RG input)

    @property
    def H(self):
        return self.C @ self.C.T

    @property
    def L(self):
        return self.C - np.eye(len(self.C))

    @property
    def top(self):
        return float((1 << self.bits) - 1)

    def scrambled(self):
        """(w, H) with the columns in `perm` order: ldlq_rg_round sorts them back to (w, C C^T)."""
        H = self.H
        return self.w[:, self.perm], H[self.perm][:, self.perm]


def _squares(n, cap, rng):
    """A random list of at most cap integers k in [1, L_DEN] with sum k^2 = n, or None."""
    ks, rem = [], n
    while rem:
        hi = min(L_DEN, isqrt(rem))
        if len(ks) == cap - 1:                          # the last slot must take the rest
            if hi * hi != rem:
                return None
            k = hi
        else:
            k = int(rng.integers((hi + 1) // 2, hi + 1))
        ks.append(k)
        rem -= k * k
    return ks


def make_ldlq_case(m, d, bits, seed):
    """An LDLQ case (see the module docstring).  Row i > 0 of C has entries whose squares sum to n_i / 256 with
    n_1 < n_2 < ..., so diag(H) = 1 + n_i / 256 is strictly ascending; the last row takes n = 256 (P - 1) with P the
    next power of two, as P - 1 entries of +-1."""
    assert d >= 8 and m >= 1
    rng = np.random.default_rng(seed)
    C = np.eye(d)
    step = max(1, 1600 // d)
    n_prev = 0

    def place(i, ks):
        cols = rng.choice(i, size=len(ks), replace=False)
        C[i, cols] = rng.choice([-1.0, 1.0], len(ks)) * np.asarray(ks, np.float64) / L_DEN

    for i in range(1, d - 1):
        n = n_prev + 1 + int(rng.integers(0, step))
        ks = None
        while ks is None:
            if n > L_DEN ** 2 * i:
                raise ValueError(f'row {i} of C cannot reach n = {n}')
            for _ in range(8):
                ks = _squares(n, i, rng)
                if ks is not None:
                    break
            else:
                n += 1
        place(i, ks)
        n_prev = n
    P = 1 << int(np.floor(np.log2(1 + n_prev / L_DEN ** 2)) + 1)
    assert P - 1 <= d - 1
    place(d - 1, [L_DEN] * (P - 1))
    dg = np.diag(C @ C.T)
    assert np.all(np.diff(dg) > 0) and dg[-1] == P
    top = (1 << bits) - 1
    w = rng.integers(-W_DEN // 2, W_DEN * top + W_DEN // 2 + 1, size=(m, d)) / W_DEN
    if m >= 2:
        w[0] = -1.25                                    # clamp at 0
        w[1] = top + 1.25                               # clamp at 2^bits - 1
    for col in (d - 1, int(rng.integers(0, d - 1))):
        w[:, col] = rng.integers(-1, top + 2, size=m) + 0.5
    return LdlqCase(bits, C, w, rng.permutation(d))


def ldlq_exact(c, greedy_passes=0, *, L=None, rnd=half_up):
    """float64 codes of quantize.ldlq_round(w, H, bits, greedy_passes) on the case -> (codes (m, d), stats).

    LDLQ: the column loop with clamp(floor(v + 1/2), 0, top).  Greedy: passes of greedy_sweep on H / max diag(H) with
    s = q - w, the clamp at the end of a pass not updating s, stopping early when a pass changes nothing.
    `L` and `rnd` replace the feedback matrix and the rounding rule: the tests use them to show that the cases can
    tell a dropped term or another tie rule apart.  stats: ties / clamps met by each stage, and the budget bits used."""
    L = c.L if L is None else L
    st = dict(ldlq=_stats(), greedy=_stats())
    q, _ = ldlq_loop(c.w, c.w, L, c.top, st['ldlq'], rnd)
    if greedy_passes:
        H = c.H
        Hn = H / np.diag(H).max()
        out = q.copy()
        s = q - c.w
        zero = np.zeros_like(c.w)
        for _ in range(greedy_passes):
            greedy_sweep(zero, Hn, out, s, st['greedy'])
            out = np.clip(out, 0, c.top)
            if np.array_equal(q, out):
                break
            q = out.copy()
        q = out
    return q, st


# --------------------------------------------------------------------------------------------------------------
# one kernel launch
# --------------------------------------------------------------------------------------------------------------
@dataclass
class LdlqBlockCase:
    """quip_ldlq_block inputs in row-major (m, cnt) form: base = w + host feedback (a 2^-7 grid), Lb with NaN on and
    above the diagonal (the kernel reads only the strictly lower part)."""
    bits: int
    base: np.ndarray
    w: np.ndarray
    Lb: np.ndarray


def make_ldlq_block_case(m, cnt, bits, seed):
    rng = np.random.default_rng(seed)
    top = (1 << bits) - 1
    w = rng.integers(-24, W_DEN * (top + 1) + 25, size=(m, cnt)) / W_DEN
    fb = rng.integers(-256, 257, size=(m, cnt)) / 128.0
    fb[:, -1] = 0                                       # half-integer w with no feedback at all: ties in w
    w[::2, -1] = rng.integers(-1, top + 2, size=len(w[::2])) + 0.5
    Lb = np.where(rng.random((cnt, cnt)) < min(1.0, 6.0 / cnt), rng.integers(-8, 9, size=(cnt, cnt)) / 8.0, 0.0)
    Lb[np.triu_indices(cnt)] = np.nan
    return LdlqBlockCase(bits, w + fb, w, Lb)


def ldlq_block_exact(c):
    """-> (q, err, stats) of one quip_ldlq_block launch."""
    st = _stats()
    q, e = ldlq_loop(c.base, c.w, c.Lb, float((1 << c.bits) - 1), st)
    return q, e, st


@dataclass
class GreedyBlockCase:
    """quip_greedy_block inputs in row-major (m, cnt) form: pre on a 2^-5 grid, Hb symmetric with power-of-two
    diagonal (so hs / H_ii is exact and half-even ties occur), wr integers, s on the 2^-4 grid."""
    pre: np.ndarray
    Hb: np.ndarray
    wr: np.ndarray
    s: np.ndarray


def make_greedy_block_case(m, cnt, seed):
    rng = np.random.default_rng(seed)
    U = np.where(rng.random((cnt, cnt)) < min(0.3, 3.0 / cnt), rng.integers(-8, 9, size=(cnt, cnt)) / 8.0, 0.0)
    Hb = np.triu(U, 1) + np.triu(U, 1).T + np.diag(np.ldexp(1.0, rng.integers(1, 4, size=cnt)))
    wr = rng.integers(-2, 18, size=(m, cnt)).astype(np.float64)
    s = rng.integers(-16, 17, size=(m, cnt)) / W_DEN
    pre = rng.integers(-128, 129, size=(m, cnt)) / 32.0
    # force a tie at the first column visited in every third row: hs / H_ii = wr - (wr + x + 1/2)
    i, r = cnt - 1, np.arange(0, m, 3)
    arg = wr[r, i] + rng.integers(-1, 1, size=len(r)) + 0.5
    pre[r, i] = (wr[r, i] - arg) * Hb[i, i] - s[r] @ Hb[:, i]
    return GreedyBlockCase(pre, Hb, wr, s)


def greedy_block_exact(c):
    """-> (wr, s, stats) after one quip_greedy_block launch."""
    st = _stats()
    wr, s = c.wr.copy(), c.s.copy()
    greedy_sweep(c.pre, c.Hb, wr, s, st)
    return wr, s, st


# --------------------------------------------------------------------------------------------------------------
# Hessian accumulation
# --------------------------------------------------------------------------------------------------------------
def make_hessian_case(T, K, seed, xmax=256, emin=-4, emax=4):
    """(T, K) fp16 activations x = n 2^e_i, |n| <= xmax, e_i per feature in [emin, emax].  Token 0 is +xmax 2^e_i on
    every feature, token 1 (when T > 1) is all zero.  The exponents depend on K only, as a layer's outlier channels
    stay the same across calibration batches (mixing scales within one chunk would cost budget bits)."""
    sc = np.ldexp(1.0, np.random.default_rng(K).integers(emin, emax + 1, size=K))
    rng = np.random.default_rng(seed)
    X = rng.integers(-xmax, xmax + 1, size=(T, K)) * sc
    X[0] = xmax * sc
    if T > 1:
        X[1] = 0
    out = X.astype(np.float16)
    assert np.array_equal(out.astype(np.float64), X)
    return out


def check_hessian(X, H0=None):
    """One quip_hessian_accumulate call on X (T, K) fp16 adding onto the float64 H0 (NaN entries: not written).

    Entry (i, j) of a chunk sum is a multiple of g_i g_j, g_i the granularity of feature i: exact in the fp32
    accumulator when sum over the chunk's tokens of |x_i x_j| <= 2^24 g_i g_j.  The float64 carry adds multiples of
    min(g_i g_j, gran(H0_ij)) and is exact while |H0_ij| + sum_t |x_i x_j| stays below 2^53 times that.
    Returns the bits used {'chunk': ..., 'carry': ...}."""
    x = np.abs(X.astype(np.float64))
    g = gran_exp(X).min(0)                              # per feature; +inf for an all-zero feature
    g = np.where(np.isfinite(g), g, 0.0).astype(np.int64)
    G = np.ldexp(1.0, g[:, None] + g[None, :])
    worst = 0.0
    for t0 in range(0, len(x), HS_CHUNK):
        a = x[t0:t0 + HS_CHUNK]
        worst = max(worst, float((a.T @ a / G).max(initial=0.0)))
    out = dict(chunk=_fits(worst, 1.0, 'fp32 chunk sum'))
    tot = x.T @ x
    Gc = G
    if H0 is not None:
        tot = np.where(np.isnan(H0), 0.0, tot + np.abs(np.nan_to_num(H0)))
        gh = gran_exp(H0)
        Gc = np.where(np.isfinite(gh), np.minimum(G, np.ldexp(1.0, np.where(np.isfinite(gh), gh, 0).astype(np.int64))), G)
    ratio = float((tot / Gc).max(initial=0.0))
    if not ratio <= F64_SPAN:
        raise BudgetError(f'float64 carry: bound exceeds 2^53 x granularity ({np.log2(ratio):.1f} bits)')
    out['carry'] = float(np.log2(max(ratio, 1.0)))
    return out


def hessian_exact(batches):
    """float64 sum of X^T X over the batches (exact under check_hessian)."""
    H = 0.0
    for X in batches:
        x = X.reshape(-1, X.shape[-1]).astype(np.float64)
        H = H + x.T @ x
    return H
