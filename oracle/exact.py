"""Exactly representable test cases for the packed GEMMs and the rotation passes.  TEST INFRASTRUCTURE ONLY.

With small-integer activations, power-of-two row scales, zero points that are integer multiples of the scale and
dyadic biases, every product and partial sum of the packed contraction is a dyadic number with few significant
bits.  Whenever those bits fit the 24 of an fp32 significand, the fp32 accumulators of every datapath (wgmma,
mma.sync, IMMA int32, FMAs) hold the exact value in any summation order, and the only rounding left is the final
fp32 -> fp16 round-to-nearest-even.  A correct kernel then returns exactly fp16(exact value), element by element,
whatever its split-K order, tile schedule or persistent walk: any missing, duplicated or misplaced term shows.

The budget checks below prove that premise for one case and one datapath, or raise BudgetError.  Each bound is
"every intermediate is an integer multiple of a granularity G and at most B in magnitude", which is exact in fp32
when B <= 2^24 G.  The bounds use the largest per-token L1 norm of the activations, so they are valid for every
summation order.
"""
from dataclasses import dataclass

import numpy as np

SPAN = float(1 << 24)           # integers up to 2^24 are exact in fp32
FP16_MAX = 65504.0


class BudgetError(ValueError):
    """The case does not satisfy the exactness premise of a datapath."""


def _fits(bound, gran, what):
    bound, gran = float(np.max(bound)), float(np.min(gran))
    if not bound <= SPAN * gran:
        raise BudgetError(f'{what}: bound {bound:.6g} exceeds 2^24 x granularity {gran:.3g} '
                          f'({np.log2(max(bound / gran, 1)):.2f} bits)')
    return np.log2(max(bound / gran, 1.0))


@dataclass
class GemmCase:
    """z = X . (scales * codes - zeros)^T (+ bias); scales = 2^-e per row."""
    bits: int
    codes: np.ndarray           # (N, K) uint8 in [0, 2^bits)
    e: np.ndarray               # (N,) int: scales = 2^-e
    zint: np.ndarray            # (N,) float64: zeros = scales * zint (zint = cbar on the symmetric grid)
    X: np.ndarray               # (M, K) fp16 integers
    bias: object                # (N,) fp16 dyadic, or None
    symmetric: bool

    @property
    def scales(self):
        return np.ldexp(1.0, -self.e).astype(np.float32)

    @property
    def zeros(self):
        return (np.ldexp(1.0, -self.e) * self.zint).astype(np.float32)

    @property
    def cbar(self):
        return ((1 << self.bits) - 1) / 2.0

    def xl1(self):
        """Largest per-token L1 norm of the activations (the bound of every partial sum of one output)."""
        return float(np.abs(self.X.astype(np.float64)).sum(1).max())


BIAS_GRAN = 1.0 / 8             # bias values are multiples of 1/8 in [-8, 8]: never finer than the outputs' 2^-(e+1)


def make_gemm_case(bits, N, K, M, *, symmetric, bias, xmax, seed, rows=('max', 'zero', 'pow2'), pow2_amax=None):
    """A packed-GEMM case whose exact result is a dyadic number in every output.

    codes uniform; per-row scales 2^-e with e drawn from six consecutive exponents (chosen so the largest possible
    output stays below the fp16 maximum); zeros = scale x an integer in [0, 2^bits) (asymmetric) or scale x cbar;
    bias = k/8 in fp16 or None; X integers in [-colmax_k, colmax_k] with a per-column magnitude profile
    (colmax_k in [xmax/4, xmax]), then the adversarial `rows`: 'max' a token of all +xmax, 'zero' an all-zero token,
    'pow2' a token whose amax is a power of two.
    pow2_amax = (lo, hi): every token gets amax = 2^a, a in [lo, hi], by one entry of +-2^a (its other entries stay
    below 2^lo), as the int8 few-token path needs; the 'max' row is then all +2^hi.
    """
    rng = np.random.default_rng(seed)
    codes = rng.integers(0, 1 << bits, size=(N, K), dtype=np.uint8)
    cbar = ((1 << bits) - 1) / 2.0
    zint = np.full(N, cbar) if symmetric else rng.integers(0, 1 << bits, size=N).astype(np.float64)
    base = xmax if pow2_amax is None else min(xmax, (1 << pow2_amax[0]) - 1)
    colmax = np.maximum(1, np.round(base * rng.uniform(0.25, 1.0, K))).astype(np.int64)
    X = rng.integers(-colmax, colmax + 1, size=(M, K)).astype(np.float64)
    if pow2_amax is not None:
        a = rng.integers(pow2_amax[0], pow2_amax[1] + 1, size=M)
        X[np.arange(M), rng.integers(0, K, M)] = np.ldexp(1.0, a) * rng.choice([-1.0, 1.0], M)
    r = 0
    for kind in rows:
        if r >= M:
            break
        if kind == 'max':
            X[r] = float(1 << pow2_amax[1]) if pow2_amax is not None else float(xmax)
        elif kind == 'zero':
            X[r] = 0.0
        elif kind == 'pow2':
            top = float(1 << int(np.log2(xmax)))
            X[r] = np.clip(X[r], -top, top)
            X[r, rng.integers(0, K)] = -top
        r += 1
    X = X.astype(np.float16)
    assert np.array_equal(X.astype(np.float64), np.round(X.astype(np.float64)))
    # six scale exponents, the smallest one large enough that no output can reach the fp16 maximum
    smax = float(np.abs(X.astype(np.float64)).sum(1).max())
    worst = ((1 << bits) - 1) * smax + 8.0
    e_lo = max(3, int(np.ceil(np.log2(max(worst / (0.9 * FP16_MAX), 1.0)))))
    e = rng.integers(e_lo, e_lo + 6, size=N)
    b = (rng.integers(-64, 65, size=N) * BIAS_GRAN).astype(np.float16) if bias else None
    return GemmCase(bits, codes, e, zint, X, b, bool(symmetric))


def gemm_xmax(bits, K, symmetric):
    """Largest power of two <= 64 that keeps a case with an all +xmax token inside the wgmma / mma.sync budget."""
    per = ((1 << bits) - 1) * (1 if symmetric else 2)
    x = 64
    while x > 1 and per * K * x + 2.0 ** 20 > SPAN:         # 2^20: the bias, 8 / 2^-(e+1) for e up to 16
        x //= 2
    return x


# --------------------------------------------------------------------------------------------------------------
# budgets, one per datapath
# --------------------------------------------------------------------------------------------------------------
def _check_range(c, l1):
    """|z| = |2^-e sum_k (c_k - zint) x_k + b| stays below the fp16 maximum."""
    sc = np.ldexp(1.0, -c.e)
    bound = sc * np.maximum(c.zint, ((1 << c.bits) - 1) - c.zint) * l1
    if c.bias is not None:
        bound = bound + np.abs(c.bias.astype(np.float64))
    if not np.all(bound < FP16_MAX):
        raise BudgetError(f'output bound {bound.max():.6g} reaches the fp16 maximum')
    return bound


def check_mma(c):
    """wgmma GEMM (qgemm_tc.cu) and the mma.sync split-K kernel (qgemm_skinny.cu).

    Both expand a code to A = (c - cbar)/2^bits in fp16 (common.cuh dq2/dq3/dq4, frag_natural: mask | one,
    minus (1 + cbar/2^bits)), a multiple of 2^-(bits+1) with |A| < 1/2, and accumulate A x in fp32: every partial
    sum is a multiple of 2^-(bits+1) and at most max|A| * sum_k |x_k|.
    Epilogue (qgemm_tc.cu:246-247, qgemm_skinny.cu:187-191 / 213-214): v = P_n acc + b_n + R_n xsum with
    P_n = scale 2^bits = 2^(bits-e) (exact scaling), R_n = scale cbar - zero = 2^-e (cbar - zint), a multiple of
    2^-(e+1) when cbar is a half integer, xsum an integer (fp32 row sums of integers, exact below 2^24).  Every
    partial of v (the split-K partials of the skinny kernel included) is a multiple of 2^-(e+1) (bias: of 1/8) and
    at most |P_n| max|A| L1 + |R_n| L1 + |b_n|.
    """
    l1 = c.xl1()
    bits = c.bits
    amax = c.cbar / (1 << bits)
    out = dict(acc=_fits(amax * l1, 2.0 ** -(bits + 1), 'fp32 accumulator'))
    out['xsum'] = _fits(l1, 1.0, 'row sum')
    sc = np.ldexp(1.0, -c.e)
    gran = sc / 2
    bound = (1 << bits) * sc * amax * l1 + sc * np.abs(c.cbar - c.zint) * (0 if c.symmetric else l1)
    if c.bias is not None:
        bound = bound + np.abs(c.bias.astype(np.float64))
        gran = np.minimum(gran, BIAS_GRAN)
    out['epilogue'] = _fits(bound / gran, 1.0, 'epilogue')
    _check_range(c, l1)
    return out


GV16_DIV = {2: (64.0, 4.0), 4: (256.0, 16.0)}       # 4^(e+1) of the two mantissa fields (e = 2 / e = 0)


def gv16_pos_scale(bits):
    """Token pre-scale 4^(e-2) of each of a lane's 8 consecutive k (qgemv.cu gv_scale): 1 or 1/16."""
    if bits == 2:
        return np.array([1, 1, 1, 1, 1 / 16, 1 / 16, 1 / 16, 1 / 16])
    return np.array([1, 1, 1 / 16, 1 / 16, 1, 1, 1 / 16, 1 / 16])


def check_gv16(c):
    """fp16 whole-K few-token kernel (qgemv.cu:15-26, qgemv_kernel).

    2-/4-bit: the codes are read in place as A_k = 1 + c_k/4^(e+1), the tokens pre-scaled by 4^(e-2) (e = 2: x_k;
    e = 0: x_k/16, exact in fp16 for |x| <= 2^10), so A_k B_k = 4^(e-2) x_k + c_k x_k / 2^(bits+4): a multiple of
    2^-(bits+4), and |A_k B_k| <= |x_k| (1 + (2^bits - 1)/2^(bits+4)).  The accumulator and the warp reduction s hold
    T_m + 2^-(bits+4) sum c x exactly when L1 (1 + (2^bits-1)/2^(bits+4)) <= 2^24 2^-(bits+4), i.e. sum_k |x_k| below
    about 2^18 (2-bit) or 2^16 (4-bit): the offset T_m costs bits+4 of the 24 bits, not 6, for 4-bit.
    T_m (multiple of 1/16) and S_m (integer) come from the constant-A MMA, exact below 2^20 and 2^24.
    Epilogue (qgemv.cu:346): A1 (s - T) = sum c x (A1 = 2^(bits+4)), an integer; v = sc sum c x - zero S + bias, a
    multiple of 2^-e (bias: 1/8).
    3-bit: the recentring expansion A = (c - 3.5)/8 as in check_mma, T = 0, and 8 s + 3.5 S = sum c x.
    """
    l1 = c.xl1()
    bits = c.bits
    out = {}
    if bits == 3:
        out['acc'] = _fits(c.cbar / 8 * l1, 1 / 16, 'fp32 accumulator')
        out['epi_sum'] = _fits(8 * (c.cbar / 8) * l1 + 3.5 * l1, 0.5, 'A1 (s - T) + A2 S')
    else:
        g = 2.0 ** -(bits + 4)
        out['acc'] = _fits((1 + ((1 << bits) - 1) * g) * l1, g, 'fp32 accumulator (T + sum c x / 2^(bits+4))')
        out['T'] = _fits(l1, 1 / 16, 'token sum T')
        out['epi_sum'] = _fits(((1 << bits) - 1) * l1, 1.0, 'A1 (s - T)')
    out['S'] = _fits(l1, 1.0, 'token sum S')
    sc = np.ldexp(1.0, -c.e)
    gran = sc / 2 if c.symmetric else sc                 # zero = 2^-e cbar on the symmetric grid
    bound = sc * ((1 << bits) - 1) * l1 + sc * np.abs(c.zint) * l1
    if c.bias is not None:
        bound = bound + np.abs(c.bias.astype(np.float64))
        gran = np.minimum(gran, BIAS_GRAN)
    out['epilogue'] = _fits(bound / gran, 1.0, 'epilogue')
    _check_range(c, l1)
    return out


GV_QMAX = float(1 << 22)


def i8_limbs(X):
    """The int8 path's token split (qgemv.cu gv_quantize_tokens): q = round(x 2^22/amax) in balanced base 256."""
    x = X.astype(np.float64)
    amax = np.abs(x).max(1, keepdims=True)
    inv = np.where(amax > 0, GV_QMAX / np.where(amax > 0, amax, 1), 0.0)
    q = np.rint(x * inv).astype(np.int64)
    lo = ((q & 0xFF) ^ 0x80) - 0x80
    v = (q - lo) >> 8
    mid = ((v & 0xFF) ^ 0x80) - 0x80
    hi = (v - mid) >> 8
    return amax[:, 0], q, (hi, mid, lo)


def check_i8(c):
    """int8 tensor path of the few-token kernels (qgemv.cu:9-13, qgemv_i8_* kernels; 2- and 4-bit).

    Each token is split once into round(x 2^22/amax) = 65536 hi + 256 mid + lo.  With amax = 2^a (or an all-zero
    token) x 2^22/amax is an exact integer, and for a <= 6 the mid and lo limbs vanish.  IMMA sums c' limb in int32
    (exact), c' = c on rows g and 4c / 16c on rows g+8 (masked in place); the epilogue converts each limb sum to
    fp32 (exact while c'max sum |limb| <= 2^24), forms tokf rs (65536 L0 + 256 L1 + L2) = sum c x with
    tokf = amax/2^22 and rs = 1 / 1/4 / 1/16 (powers of two), then v = sc sum c x - zero S + bias as in check_gv16.
    """
    if c.bits not in (2, 4):
        raise BudgetError('the int8 path takes 2- and 4-bit codes only')
    x = c.X.astype(np.float64)
    amax, q, limbs = i8_limbs(c.X)
    nz = amax > 0
    a = np.log2(amax[nz])
    if not np.array_equal(a, np.round(a)):
        raise BudgetError('every token of an int8 case must have a power-of-two amax (or be all zero)')
    if not np.array_equal(q.astype(np.float64), x * np.where(amax > 0, GV_QMAX / np.where(amax > 0, amax, 1), 0)[:, None]):
        raise BudgetError('x 2^22 / amax is not an integer')
    cmax = {2: 12.0, 4: 240.0}[c.bits]
    out = {}
    total, low = 0.0, 16
    for li, (w, L) in enumerate(zip((16, 8, 0), limbs)):
        b = cmax * float(np.abs(L).sum(1).max())
        out[f'limb{li}'] = _fits(b, 1.0, f'fp32 conversion of limb {li} sums')
        total += b * 2.0 ** w
        if np.any(L != 0):
            low = min(low, w)
    out['dot'] = _fits(total, 2.0 ** low, '65536 L0 + 256 L1 + L2')
    l1 = c.xl1()
    out['S'] = _fits(l1, 1.0, 'token sum S')
    sc = np.ldexp(1.0, -c.e)
    gran = sc / 2 if c.symmetric else sc                 # zero = 2^-e cbar on the symmetric grid
    bound = sc * ((1 << c.bits) - 1) * l1 + sc * np.abs(c.zint) * l1
    if c.bias is not None:
        bound = bound + np.abs(c.bias.astype(np.float64))
        gran = np.minimum(gran, BIAS_GRAN)
    out['epilogue'] = _fits(bound / gran, 1.0, 'epilogue')
    _check_range(c, l1)
    return out


# --------------------------------------------------------------------------------------------------------------
# references
# --------------------------------------------------------------------------------------------------------------
def dequant(c):
    """(N, K) float64 weights scales * codes - zeros (exact: 2^-e times small integers)."""
    return np.ldexp(1.0, -c.e)[:, None] * (c.codes.astype(np.float64) - c.zint[:, None])


def gemm_exact(c):
    """float64 result (exact: at most ~40 significant bits per output)."""
    z = c.X.astype(np.float64) @ dequant(c).T
    if c.bias is not None:
        z += c.bias.astype(np.float64)[None, :]
    return z


def gemm_exact_torch(c, device):
    """gemm_exact on `device` in float64 (exact in any order, so fine for the large shapes)."""
    import torch
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(device)
    sc = t(np.ldexp(1.0, -c.e))
    W = sc[:, None] * (t(c.codes).double() - t(c.zint)[:, None])
    z = t(c.X).double() @ W.T
    if c.bias is not None:
        z += t(c.bias).double()[None, :]
    return z


def to_fp16(z):
    """The single rounding a correct kernel performs: round to nearest even, fp16."""
    return np.asarray(z, np.float64).astype(np.float16)


def _k_orders(K, order, rng):
    if order == 'natural':
        return [np.arange(K)]
    if order == 'reversed':
        return [np.arange(K)[::-1]]
    cuts = np.sort(rng.choice(np.arange(1, K), size=min(K - 1, 7), replace=False))
    chunks = np.split(np.arange(K), cuts)
    return [chunks[i] for i in rng.permutation(len(chunks))]


def _f32_dot(X32, A32, order, rng):
    """sum_k X[m,k] A[n,k] in fp32, k visited in the given order: chunks accumulated one after another."""
    acc = np.zeros((X32.shape[0], A32.shape[0]), np.float32)
    for idx in _k_orders(X32.shape[1], order, rng):
        for k in (idx if order == 'reversed' else [idx]):
            k = np.atleast_1d(k)
            acc = (acc + (X32[:, k] @ A32[:, k].T).astype(np.float32)).astype(np.float32)
    return acc


def gemm_f32_mma(c, order, seed=0):
    """The wgmma / mma.sync arithmetic in fp32 with k summed in `order` ('natural', 'reversed', 'chunks')."""
    rng = np.random.default_rng(seed)
    f = np.float32
    A = ((c.codes.astype(f) - f(c.cbar)) / f(1 << c.bits)).astype(f)
    X = c.X.astype(f)
    acc = _f32_dot(X, A, order, rng)
    sc = c.scales
    P = (sc * f(1 << c.bits)).astype(f)
    v = (P[None, :] * acc).astype(f)
    if c.bias is not None:
        v = (v + c.bias.astype(f)[None, :]).astype(f)
    if not c.symmetric:
        R = (sc * f(c.cbar) - c.zeros).astype(f)
        xsum = X.sum(1, dtype=f)
        v = (v + R[None, :] * xsum[:, None]).astype(f)
    return v.astype(np.float16)


def gemm_f32_gv16(c, order, seed=0):
    """The fp16 few-token kernel's arithmetic (offset-free 2-/4-bit expansion, T and S, (A1, A2) epilogue) in fp32."""
    rng = np.random.default_rng(seed)
    f = np.float32
    K = c.codes.shape[1]
    X = c.X.astype(f)
    if c.bits == 3:
        A = ((c.codes.astype(f) - f(3.5)) / f(8)).astype(f)
        B, T, a1, a2 = X, np.zeros(X.shape[0], f), f(8), f(3.5)
    else:
        ps = np.tile(gv16_pos_scale(c.bits), K // 8).astype(f)
        big, small = GV16_DIV[c.bits]
        div = np.where(ps == 1, big, small).astype(f)
        A = (f(1) + c.codes.astype(f) / div[None, :]).astype(f)
        B = (X * ps[None, :]).astype(np.float16).astype(f)
        T = B.sum(1, dtype=f)
        a1, a2 = f(big), f(0)
    s = _f32_dot(B, A, order, rng)
    S = X.sum(1, dtype=f)
    inner = (a1 * (s - T[:, None]) + a2 * S[:, None]).astype(f)
    v = (c.scales[None, :] * inner - c.zeros[None, :] * S[:, None]).astype(f)
    if c.bias is not None:
        v = (v + c.bias.astype(f)[None, :]).astype(f)
    return v.astype(np.float16)


# --------------------------------------------------------------------------------------------------------------
# rotation passes
# --------------------------------------------------------------------------------------------------------------
def make_pass_case(p, nblk, shared, M, *, xmax, seed):
    """Factors with fp16 entries k/64, k in [-64, 64]; X integers in [-xmax, xmax] (row 0 all +xmax when M > 1)."""
    rng = np.random.default_rng(seed)
    F = (rng.integers(-64, 65, size=(1 if shared else nblk, p, p)) / 64.0).astype(np.float16)
    X = rng.integers(-xmax, xmax + 1, size=(M, p * nblk)).astype(np.float16)
    if M > 1:
        X[0] = xmax
    return X, F


def check_pass(X, F):
    """Block-diagonal pass (rot.cu, rot_small.cu, rot_fewtok.cu, the DENSE wgmma pass): out_i = sum_j F_ij x_j with
    F_ij a multiple of 1/64, |F_ij| <= 1, x integers: every partial sum is a multiple of 1/64 and at most p max|x|,
    exact in fp32 when p max|x| 64 <= 2^24; the output stays below the fp16 maximum when p max|x| < 65504."""
    F64 = F.astype(np.float64)
    if not np.array_equal(F64 * 64, np.round(F64 * 64)) or np.abs(F64).max() > 1:
        raise BudgetError('factor entries must be k/64 with |k| <= 64')
    x = X.astype(np.float64)
    if not np.array_equal(x, np.round(x)):
        raise BudgetError('activations must be integers')
    p = F.shape[-1]
    bound = p * np.abs(x).max()
    if not bound < FP16_MAX:
        raise BudgetError(f'pass output bound {bound} reaches the fp16 maximum')
    return dict(acc=_fits(bound, 1 / 64, 'pass accumulator'))


def pass_f32(X, F, p, nblk, strided, order, seed=0):
    """The pass in fp32 with the block's inner index summed in `order`."""
    rng = np.random.default_rng(seed)
    f = np.float32
    M, n = X.shape
    Fb = np.broadcast_to(F.astype(f), (nblk, p, p))
    T = X.astype(f).reshape(M, p, nblk).transpose(0, 2, 1) if strided else X.astype(f).reshape(M, nblk, p)
    out = np.zeros((M, nblk, p), f)
    for idx in _k_orders(p, order, rng):
        for j in (idx if order == 'reversed' else [idx]):
            j = np.atleast_1d(j)
            out = (out + np.einsum('bij,mbj->mbi', Fb[:, :, j], T[:, :, j]).astype(f)).astype(f)
    out = out.transpose(0, 2, 1).reshape(M, n) if strided else out.reshape(M, n)
    return out.astype(np.float16)
