"""Exactly representable cases for whole incoherence sides of the packed forward.  TEST INFRASTRUCTURE ONLY.

quip_qlinear_forward (csrc/api.cu) runs a K side, the packed GEMM and an N side.  A side is two block-diagonal passes;
the K side first gathers and scales its input, the N side last scatters and adds the bias.  A pass (p, nblk, strided)
multiplies block b, whose element j sits at layout position j * nblk + b (strided) or b * p + j (contiguous):
out[pos(b, i)] = sum_j F[b][i][j] in[pos(b, j)].  The kernels that run a side, and where they round to fp16:

  two-pass routes   x1 = fp16(x[idx] * s[idx])                 quip_gather (gather_kernel, gather_fewtok_kernel),
                                                                the fused load of pass_fewtok_kernel, or the stage-in
                                                                of side_fused_kernel
                    t  = fp16(pass0(x1))                        quip_rot_pass / pass_fewtok_kernel, or side_fused_kernel
                    x2 = fp16(pass1(t))                         (its shared-memory tile holds fp16 words)
                    y[j] = fp16(fp16(w[idx[j]]) + bias[j])      w = pass1 output: quip_gather (fma with scale 1), the
                                                                fused scatter of pass_fewtok_kernel, or the stage-out of
                                                                side_fused_kernel -- the bias is added after rounding
  side_fewtok       t  = pass0(x1) in fp32, not rounded          rot_side_fewtok.cu: one launch for both passes
                    x2 = fp16(pass1(t)); bias as above

The gather multiplies by s in fp32 and rounds once; with s a power of two and integer x that is exact.  The bias is
added in fp32 to the rounded pass output and the sum rounded again: the reference repeats both roundings (fp64 -> fp32
-> fp16), so this step needs no budget.  When the layer
folds 1/s into its first V pass (meta[2] = 1) the kernels see no scale at all.

Exactness premise (as oracle/exact.py): every fp32 sum a kernel forms -- mma.sync / wgmma accumulators, fmaf chains,
shuffle and shared-memory reductions, in any order -- holds an integer multiple of a power-of-two granularity g and is
at most 2^24 g in magnitude, so it is exact.  Then the only roundings left are the fp16 ones listed above, and each
route returns its oracle bit for bit.  The budgets are proved on the case's own data: for a pass, g is the granularity
of the factors times that of the input, and every partial sum of output i is at most sum_j |F_ij| |in_j|.  An fp16
rounding of a multiple of g is still a multiple of g, so the second pass is budgeted from the first pass's
granularity whether or not t is rounded.  The GEMM sees x2 = 2^-a X with X integer: that is oracle/exact.check_mma's
case with scales 2^-(e + a), exact under the same budget.

Two families of layers get a side's output out of the forward:

  A  dense factors behind a transparent GEMM: asymmetric grid with zeros = 0, scales 2^-e, codes 1 at the column(s)
     a row selects and 0 elsewhere, every x2 column selected by some row.  z = fp16(2^-e sum of the selected x2), so y
     checks the K side, the GEMM hand-off (the row sums of x2 included) and the N side.
  B  integer sides behind a real asymmetric GEMM: V factors in {-1, 0, 1} with a few nonzeros per row, s = 2^k >= 1, so
     x2 stays integer; codes, zero points and scales random as in exact.make_gemm_case.  A wrong row sum of x2 (the
     side_fused_kernel xsum or quip_rowsum) changes y.  The symmetric variant skips the row sums.
"""
from dataclasses import dataclass, field, replace

import numpy as np

from . import exact as ex
from .exact import BudgetError, FP16_MAX, _fits
from .butterfly import butterfly_factors

BIAS_GRAN = ex.BIAS_GRAN


@dataclass
class Pass:
    p: int
    nblk: int
    strided: bool
    F: np.ndarray               # (1 or nblk, p, p) fp16 dyadic

    @property
    def shared(self):
        return self.F.shape[0] == 1 and self.nblk > 1


@dataclass
class LayerCase:
    family: str                 # 'A' or 'B'
    bits: int
    X: np.ndarray               # (M, K) fp16 integers
    inv_scale: object           # (K,) float32 powers of two, or None
    folded: bool                # the layer keeps inv_scale folded into its first V pass: the kernels never apply it
    v_idx: object               # (K,) int32 layout[l] = x[v_idx[l]], or None (identity)
    vp: list                    # two Pass, applied in order
    codes: np.ndarray           # (N, K) uint8, in layout order
    e: np.ndarray               # (N,) int: scales 2^-e
    zint: np.ndarray            # (N,) float64: zeros = 2^-e zint
    symmetric: bool
    up: list                    # two Pass
    u_idx: object               # (N,) int32 y[j] = layout[u_idx[j]], or None
    bias: object                # (N,) fp16 k/8, or None
    meta: dict = field(default_factory=dict)

    @property
    def M(self):
        return self.X.shape[0]

    @property
    def K(self):
        return self.X.shape[1]

    @property
    def N(self):
        return self.codes.shape[0]

    @property
    def scales(self):
        return np.ldexp(1.0, -self.e).astype(np.float32)

    @property
    def zeros(self):
        return (np.ldexp(1.0, -self.e) * self.zint).astype(np.float32)

    def kernel_scale(self):
        return None if (self.inv_scale is None or self.folded) else self.inv_scale


# --------------------------------------------------------------------------------------------------------------
# pass geometry (QuantLinear._side) and the route of each side (api.cu quip_qlinear_forward)
# --------------------------------------------------------------------------------------------------------------
def side_geometry(n, side):
    """[(p, nblk, strided)] of the two passes QuantLinear builds for a side of n features ('v' or 'u')."""
    p1, p2 = butterfly_factors(n)
    layout_a = p2 >= p1
    col, row = (p1, p2, layout_a), (p2, p1, not layout_a)
    return [col, row] if side == 'v' else [row, col]


def _align16(v):
    return (v + 15) // 16 * 16


def side_fewtok_ok(passes, n, M):
    """rot_side_fewtok.cu side_fewtok_ok, with the shared-memory plan sf_plan."""
    a, b = passes
    if not 1 <= M <= 8 or a.strided == b.strided or a.nblk != b.p or b.nblk != a.p or a.p % 16 or b.p % 16:
        return False
    if a.p * a.nblk != n or n >= 65536 or n % 8:
        return False
    bpc = 4 if b.p <= 16 else 1
    rows = b.p if b.p <= 64 else (32 if b.p > 512 else 64)
    ndots, nout = bpc * b.p, bpc * rows
    total = sum(_align16(x) for x in (ndots * a.p * 2, nout * b.p * 2, ndots * M * 4, nout * 8,
                                  M * a.nblk * (a.p + 2) * 2, M * n * 2, n * 2))
    return total <= 224 * 1024


def side_fused_ok(passes, n):
    """rot_side.cu side_fused_ok (QuantLinear derives fragment-order factors for p in {32, 64} and n <= 4096)."""
    col = [q for q in passes if q.strided]
    row = [q for q in passes if not q.strided]
    if len(col) != 1 or n > 4096 or any(q.p not in (32, 64) for q in passes):
        return False
    col, row = col[0], row[0]
    return col.p == row.nblk and col.nblk == row.p and (col.p, row.p) in ((64, 64), (32, 64), (64, 32))


DEFAULTS = dict(side_fused=1, side_fewtok=0, fewtok=1, fewtok_max_m=32, gemv=1)


def oracle_route(side_route):
    """side_fused_kernel keeps the two-pass rounding points (fp16 words in shared memory)."""
    return 'side_fewtok' if side_route == 'side_fewtok' else 'two_pass'


def plan(c, cfg):
    """The kernels quip_qlinear_forward launches for case c under quip_config values cfg (DEFAULTS updated):
    dict(v=..., u=..., launches=n).  Sides: 'side_fewtok', 'side_fused', 'two_pass'."""
    q = dict(DEFAULTS, **cfg)
    M, K, N = c.M, c.K, c.N
    fmax = q['fewtok_max_m']
    n = 0
    if q['fewtok'] and q['side_fewtok'] and side_fewtok_ok(c.vp, K, M):
        v, n = 'side_fewtok', n + 1
    elif q['side_fused'] and M > fmax and side_fused_ok(c.vp, K):
        v, n = 'side_fused', n + 1
    else:
        fuse_in = q['fewtok'] and M <= fmax and M <= 32 and c.vp[0].p <= 128 and c.vp[0].p % 16 == 0
        n += 2 + int((c.v_idx is not None or c.kernel_scale() is not None) and not fuse_in)
        v = 'two_pass'
    need_xsum = not c.symmetric and M > 32
    if need_xsum and v != 'side_fused':
        n += 1                                            # quip_rowsum
    n += 1                                                # the split-K kernel (gemv = 0) or the wgmma GEMM
    if q['fewtok'] and q['side_fewtok'] and side_fewtok_ok(c.up, N, M):
        u, n = 'side_fewtok', n + 1
    elif q['side_fused'] and M > fmax and side_fused_ok(c.up, N):
        u, n = 'side_fused', n + 1
    else:
        tail = c.u_idx is not None or c.bias is not None
        fuse_out = tail and q['fewtok'] and M <= fmax and M <= 32 and c.up[1].p % 16 == 0
        n += 2 + int(tail and not fuse_out)
        u = 'two_pass'
    return dict(v=v, u=u, launches=n)


# --------------------------------------------------------------------------------------------------------------
# float64 reference (torch, on any device)
# --------------------------------------------------------------------------------------------------------------
def _t(a, device):
    import torch
    return torch.from_numpy(np.ascontiguousarray(a)).to(device)


def r16(v):
    """fp16 round to nearest even of an fp32-exact float64 tensor (exact in two steps: fp64 -> fp32 loses nothing)."""
    import torch
    return v.to(torch.float32).to(torch.float16).to(torch.float64)


def apply_pass(W, ps):
    """One block-diagonal pass of W (M, n) float64 tensor, exact in float64 (the values stay far below 2^53)."""
    import torch
    M, n = W.shape
    F = _t(ps.F, W.device).double().expand(ps.nblk, ps.p, ps.p)
    if ps.strided:
        out = torch.einsum('bij,mjb->mib', F, W.reshape(M, ps.p, ps.nblk))
    else:
        out = torch.einsum('bij,mbj->mbi', F, W.reshape(M, ps.nblk, ps.p))
    return out.reshape(M, n)


def side_in(c, device):
    """x1: the K side's gathered and scaled input."""
    x = _t(c.X, device).double()
    s = c.kernel_scale()
    if s is not None:
        x = r16(x * _t(s, device).double()[None, :])
    if c.v_idx is not None:
        x = x[:, _t(c.v_idx, device).long()]
    return x


def two_passes(x, passes, route):
    t = apply_pass(x, passes[0])
    if route != 'side_fewtok':
        t = r16(t)
    return r16(apply_pass(t, passes[1]))


def dequant(c, device):
    import torch
    sc = torch.ldexp(torch.ones(c.N, dtype=torch.float64, device=device), -_t(c.e, device).double())
    return sc[:, None] * (_t(c.codes, device).double() - _t(c.zint, device).double()[:, None])


def side_out(c, w):
    if c.u_idx is not None:
        w = w[:, _t(c.u_idx, w.device).long()]
    if c.bias is not None:
        w = r16(w + _t(c.bias, w.device).double()[None, :])
    return w


def forward(c, v_route='two_pass', u_route='two_pass', device='cpu'):
    """fp16 y (M, N) as a numpy array, the result of the routes given for the two sides; also x2 and z (float64)."""
    x2 = two_passes(side_in(c, device), c.vp, v_route)
    z = r16(x2 @ dequant(c, device).T)
    y = side_out(c, two_passes(z, c.up, u_route))
    return y.cpu().numpy().astype(np.float16), x2, z


# --------------------------------------------------------------------------------------------------------------
# budgets
# --------------------------------------------------------------------------------------------------------------
def granularity(v):
    """The largest power of two g <= 1 of which every entry of v (float64 tensor or array) is an integer multiple."""
    import torch
    v = torch.as_tensor(np.asarray(v, np.float64)) if not isinstance(v, torch.Tensor) else v
    v = v[v != 0]
    for a in range(0, 60):
        if bool(torch.all(torch.frac(v * 2.0 ** a) == 0)):
            return 2.0 ** -a
    raise BudgetError('values are not dyadic')


def check_pass_budget(W, ps, gran_in, what):
    """Every partial sum of the pass on W is exact in fp32 and every output stays below the fp16 maximum."""
    F = ps.F.astype(np.float64)
    gf = granularity(F)
    bound = apply_pass(W.abs(), replace(ps, F=np.abs(F)))
    b = float(bound.max())
    if not b < FP16_MAX:
        raise BudgetError(f'{what}: output bound {b:.6g} reaches the fp16 maximum')
    return _fits(b, gf * gran_in, f'{what} accumulator')


def check_case(c, v_route='two_pass', u_route='two_pass', device='cpu'):
    """Prove the exactness premise of case c on the given side routes (or raise BudgetError); returns the bits used."""
    import torch
    x = c.X.astype(np.float64)
    if not np.array_equal(x, np.round(x)):
        raise BudgetError('activations must be integers')
    out = {}
    x1 = side_in(c, device)
    s = c.kernel_scale()
    if s is not None:
        xs = _t(c.X, device).double() * _t(s, device).double()[None, :]
        if not torch.equal(r16(xs), xs):
            raise BudgetError('x * s is not exact in fp16')
    g = granularity(x1)
    out['v0'] = check_pass_budget(x1, c.vp[0], g, 'V pass 0')
    t = apply_pass(x1, c.vp[0])
    g = g * granularity(c.vp[0].F.astype(np.float64))
    out['v1'] = check_pass_budget(t if v_route == 'side_fewtok' else r16(t), c.vp[1], g, 'V pass 1')
    _, x2, z = forward(c, v_route, u_route, device)
    a = -int(np.log2(granularity(x2)))
    gc = ex.GemmCase(c.bits, c.codes, c.e + a, c.zint, (x2 * 2.0 ** a).cpu().numpy(), None, c.symmetric)
    out.update({f'gemm_{k}': v for k, v in ex.check_mma(gc).items()})
    g = granularity(z)
    out['u0'] = check_pass_budget(z, c.up[0], g, 'U pass 0')
    t = apply_pass(z, c.up[0])
    g = g * granularity(c.up[0].F.astype(np.float64))
    out['u1'] = check_pass_budget(t if u_route == 'side_fewtok' else r16(t), c.up[1], g, 'U pass 1')
    w = side_out(c, two_passes(z, c.up, u_route))
    if not float(w.abs().max()) < FP16_MAX:
        raise BudgetError('output reaches the fp16 maximum')
    return out


# --------------------------------------------------------------------------------------------------------------
# fp32 simulation of the routes, summation order given (CPU, numpy)
# --------------------------------------------------------------------------------------------------------------
def pass_f32(X32, ps, order, rng):
    """The pass in fp32 (no final rounding), the block's inner index summed in `order`."""
    f = np.float32
    M, n = X32.shape
    Fb = np.broadcast_to(ps.F.astype(f), (ps.nblk, ps.p, ps.p))
    T = X32.reshape(M, ps.p, ps.nblk).transpose(0, 2, 1) if ps.strided else X32.reshape(M, ps.nblk, ps.p)
    out = np.zeros((M, ps.nblk, ps.p), f)
    for idx in ex._k_orders(ps.p, order, rng):
        for j in (idx if order == 'reversed' else [idx]):
            j = np.atleast_1d(j)
            out = (out + np.einsum('bij,mbj->mbi', Fb[:, :, j], T[:, :, j]).astype(f)).astype(f)
    return out.transpose(0, 2, 1).reshape(M, n) if ps.strided else out.reshape(M, n)


def simulate_f32(c, v_route, u_route, order, seed=0):
    """The route's arithmetic in fp32: gather, passes (t rounded or not), the mma GEMM epilogue, scatter and bias."""
    rng = np.random.default_rng(seed)
    f = np.float32
    x = c.X.astype(f)
    s = c.kernel_scale()
    if s is not None:
        x = (x * s.astype(f)[None, :]).astype(np.float16).astype(f)
    if c.v_idx is not None:
        x = x[:, c.v_idx]

    def side(x, passes, route):
        t = pass_f32(x, passes[0], order, rng)
        if route != 'side_fewtok':
            t = t.astype(np.float16).astype(f)
        return pass_f32(t, passes[1], order, rng).astype(np.float16)

    x2 = side(x, c.vp, v_route)
    gc = ex.GemmCase(c.bits, c.codes, c.e, c.zint, x2, None, c.symmetric)
    z = ex.gemm_f32_mma(gc, order, seed)
    w = side(z.astype(f), c.up, u_route)
    if c.u_idx is not None:
        w = w[:, c.u_idx]
    if c.bias is not None:
        w = (w.astype(f) + c.bias.astype(f)[None, :]).astype(np.float16)
    return w


# --------------------------------------------------------------------------------------------------------------
# case construction
# --------------------------------------------------------------------------------------------------------------
def _activations(rng, M, K, xmax):
    X = rng.integers(-xmax, xmax + 1, size=(M, K)).astype(np.float64)
    if M >= 2:
        X[M - 1] = 0.0                                  # the adversarial rows sit last: inside a partial last tile
        X[M - 2] = xmax
    return X.astype(np.float16)


def _dense(rng, nf, p, den):
    return (rng.integers(-den, den + 1, size=(nf, p, p)) / den).astype(np.float16)


def _sparse(rng, nf, p, nnz):
    F = np.zeros((nf, p, p))
    for b in range(nf):
        for i in range(p):
            F[b, i, rng.choice(p, nnz, replace=False)] = rng.choice([-1.0, 1.0], nnz)
    return F.astype(np.float16)


def make_passes(rng, n, side, kind, *, shared=False, geometry=None):
    """Two passes for a side of n features: kind ('dense', den) -> entries k/den; ('sparse', nnz) -> +-1 at nnz
    random positions per row.  geometry overrides side_geometry(n, side)."""
    out = []
    for (p, nblk, strided) in (geometry or side_geometry(n, side)):
        nf = 1 if shared else nblk
        F = _dense(rng, nf, p, kind[1]) if kind[0] == 'dense' else _sparse(rng, nf, p, kind[1])
        out.append(Pass(p, nblk, bool(strided), F))
    return out


def _abs_pass(W, ps):
    """|F| applied to |W| (float64 tensors): a bound of every partial sum of the pass."""
    return apply_pass(W.abs(), replace(ps, F=np.abs(ps.F.astype(np.float64))))


def _selection_codes(rng, N, K, bits):
    """Code 1 at the column(s) a row selects, 0 elsewhere; every column is selected by some row, every row selects."""
    codes = np.zeros((N, K), np.uint8)
    cols = rng.permutation(K)
    if K >= N:
        codes[rng.permutation(np.arange(K) % N), cols] = 1      # K / N columns per row
    else:
        codes[np.arange(N), cols[np.arange(N) % K]] = 1
    return codes


def make_case(family, K, N, M, *, bits=2, seed, v_kind=None, u_kind=None, xmax=None, perm=True, scale='apply',
              bias=True, shared=False, symmetric=False, v_geometry=None, device='cpu'):
    """One layer case.  scale: 'apply' (the kernels apply inv_scale), 'folded' (meta[2] = 1: they must not), None."""
    rng = np.random.default_rng(seed)
    if family == 'A':
        v_kind, u_kind, xmax = v_kind or ('dense', 2), u_kind or ('dense', 16), xmax or 2
        sexp = rng.integers(0, 3, size=K)                       # 1/s = 2^-k, k in 0..2
    else:
        v_kind, u_kind, xmax = v_kind or ('sparse', 2), u_kind or ('sparse', 2), xmax or 8
        sexp = -rng.integers(0, 2, size=K)                      # 1/s = 2^k >= 1: x2 stays integer
    X = _activations(rng, M, K, xmax)
    inv_scale = None if scale is None else np.ldexp(1.0, -sexp).astype(np.float32)
    v_idx = rng.permutation(K).astype(np.int32) if perm else None
    u_idx = rng.permutation(N).astype(np.int32) if perm else None
    vp = make_passes(rng, K, 'v', v_kind, shared=shared, geometry=v_geometry)
    up = make_passes(rng, N, 'u', u_kind, shared=shared)
    if family == 'A':
        codes = _selection_codes(rng, N, K, bits)
        e = rng.integers(0, 3, size=N)
        zint = np.zeros(N)
    else:
        codes = rng.integers(0, 1 << bits, size=(N, K), dtype=np.uint8)
        cbar = ((1 << bits) - 1) / 2.0
        zint = np.full(N, cbar) if symmetric else rng.integers(0, 1 << bits, size=N).astype(np.float64)
        e = rng.integers(0, 6, size=N)
    b = (rng.integers(-64, 65, size=N) * BIAS_GRAN).astype(np.float16) if bias else None
    if family == 'A':
        # scales 2^-e, e from three consecutive exponents: the smallest that keep the U side's outputs below 2^14
        xb = _t(X, device).double()
        if v_idx is not None:
            xb = xb[:, _t(v_idx, device).long()]
        for ps in vp:
            xb = _abs_pass(xb, ps)
        zb = xb @ _t(codes, device).double().T
        for ps in up:
            zb = _abs_pass(zb, ps)
        e = e + max(0, int(np.ceil(np.log2(max(float(zb.max()) / 2.0 ** 14, 1.0)))))
    c = LayerCase(family, bits, X, inv_scale, scale == 'folded', v_idx, vp, codes, e, zint, bool(symmetric), up, u_idx,
                  b, dict(K=K, N=N, M=M, seed=seed))
    if family == 'B':
        # scales: the smallest six consecutive exponents that keep every z below the fp16 maximum
        x2 = two_passes(side_in(c, device), c.vp, 'two_pass')
        worst = ((1 << bits) - 1) * float(x2.abs().sum(1).max()) + 1.0
        e_lo = max(0, int(np.ceil(np.log2(max(worst / (0.5 * FP16_MAX), 1.0)))))
        c.e = e_lo + c.e
    return c


A_LADDER = [dict(xmax=2, v_kind=('dense', 2), u_kind=('dense', 16)), dict(xmax=2, v_kind=('dense', 2), u_kind=('dense', 8)),
            dict(xmax=1, v_kind=('dense', 2), u_kind=('dense', 8)), dict(xmax=1, v_kind=('dense', 1), u_kind=('dense', 4))]
B_LADDER = [dict(xmax=8), dict(xmax=4), dict(xmax=2), dict(xmax=1)]


def fit_case(family, K, N, M, routes=(('two_pass', 'two_pass'),), device='cpu', **kw):
    """make_case with the first parameters of the family's ladder (richest first) that pass the budgets of the routes
    listed."""
    for step in (A_LADDER if family == 'A' else B_LADDER):
        c = make_case(family, K, N, M, device=device, **dict(kw, **step))
        try:
            for r in routes:
                check_case(c, *r, device=device)
            return c
        except BudgetError:
            if step is (A_LADDER if family == 'A' else B_LADDER)[-1]:
                raise
