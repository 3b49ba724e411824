"""Whole packed forwards (K side, GEMM, N side) on exactly representable layers, compared bit for bit with the float64
oracle of the route each side takes (oracle/exact_side.py).  Every route of quip_qlinear_forward's incoherence sides:
the one-kernel side_fused_kernel (with and without the row sums, partial last tiles), pass_fewtok_kernel with its fused
gather and scatter (one, two and four token groups), the one-launch side_fewtok_kernel (its row tiles at 11008), and the
unfused quip_gather + quip_rot_pass + quip_rowsum sequence.  The launch count of each call is checked against the route
the oracle assumed.  For up to 32 tokens the GEMM runs on the fp32 split-K kernel (gemv = 0): the int8 whole-K kernel
quantizes its tokens, which these activations do not survive exactly."""
import ctypes as C

import numpy as np
import pytest
import torch

from exact_util import assert_fp16_bits_equal
from oracle import exact_side as es

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
SHAPES = [(4096, 4096), (4096, 11008), (11008, 4096), (2048, 2048), (8192, 1024), (768, 2048)]
FEW_M = [1, 2, 3, 5, 8]
MID_M = [9, 15, 16, 17, 24, 31, 32]
MANY_M = [33, 47, 300, 2048]
HAND_64x32 = [(64, 32, True), (32, 64, False)]            # V side of 2048: strided 64-wide blocks first, then 32-wide
# per-case variants: gather permutations, inv_scale applied / folded / absent, bias, shared factors, bits
VARIANTS = [dict(perm=True, scale='apply', bias=True, shared=False, bits=2),
            dict(perm=False, scale='folded', bias=False, shared=True, bits=3),
            dict(perm=True, scale=None, bias=True, shared=True, bits=4),
            dict(perm=True, scale='folded', bias=False, shared=False, bits=2)]


def many_ms(K, N):
    return MANY_M if max(K, N) <= 4096 else MANY_M[:3]


def budget_routes(M):
    """Side routes a case of M tokens is budgeted for: the one-launch side (intermediate in fp32) exists for M <= 8.
    Budgets are per side, so these two also cover the mixed routes (one side in one launch, the other in two)."""
    return [('two_pass', 'two_pass')] + ([('side_fewtok', 'side_fewtok')] if M <= 8 else [])


def a_case(K, N, M, v_geometry=None, device='cpu'):
    var = VARIANTS[(K + N + M) % len(VARIANTS)]
    return es.fit_case('A', K, N, M, routes=budget_routes(M), seed=K * 7 + N * 3 + M, v_geometry=v_geometry,
                       device=device, **var)


def b_case(K, N, M, symmetric, v_geometry=None, device='cpu'):
    var = dict(VARIANTS[(K + M) % len(VARIANTS)], shared=False)
    return es.fit_case('B', K, N, M, routes=budget_routes(M), seed=K + N + M + int(symmetric), symmetric=symmetric,
                       v_geometry=v_geometry, device=device, **var)


def route_cfgs(M):
    """The quip_config settings each token count is run under (gemv = 0 throughout)."""
    if M <= 8:
        return [dict(gemv=0), dict(gemv=0, side_fewtok=1), dict(gemv=0, fewtok=0)]
    if M <= 32:
        return [dict(gemv=0), dict(gemv=0, fewtok_max_m=8)]
    return [dict(), dict(side_fused=0)]


# ---- the layer, its buffers overwritten with the case ----
def build_layer(c):
    from quip_b200 import quant as Q
    ql = Q.QuantLinear(c.bits, c.K, c.N, bias=c.bias is not None, incoh='blocked', rescale=c.inv_scale is not None)
    ql = ql.to(DEV)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).to(DEV)
    for side, passes, idx, n in (('v', c.vp, c.v_idx, c.K), ('u', c.up, c.u_idx, c.N)):
        for i, ps in enumerate(passes):
            setattr(ql, f'{side}_f{i}', t(ps.F).half().contiguous())
        getattr(ql, f'{side}_idx').copy_(t(np.arange(n) if idx is None else idx).int())
        ql.meta[3 if side == 'v' else 4] = int(idx is None)
    if c.inv_scale is not None:
        ql.inv_scale.copy_(t(c.inv_scale).float())
    ql.meta[2] = int(c.folded)
    ql._install(t(c.codes), t(c.scales).reshape(-1, 1), t(c.zeros).reshape(-1, 1),
                None if c.bias is None else t(c.bias))
    assert int(ql.meta[1]) == int(c.symmetric)
    ql._desc = None
    d = ql._descriptor()
    for sd, passes in ((d.V, c.vp), (d.U, c.up)):
        for i, ps in enumerate(passes):
            q = sd.passes[i]
            assert (q.p, q.nblk) == (ps.p, ps.nblk), (q.p, q.nblk, ps)
            q.strided = int(ps.strided)                   # a hand-built side: only the strided flags may differ
            assert q.shared == int(ps.shared)
    return ql


def run_forward(ql, X, cfg):
    """y (M, N) through quip_qlinear_forward under quip_config cfg, with a workspace filled with NaN (except the
    zeroed split-K counters) so that no stale row sum or intermediate can stand in for one a kernel failed to write;
    returns (y, launches)."""
    from quip_b200 import _lib
    lib = _lib.load()
    x = torch.from_numpy(X).to(DEV)
    M = X.shape[0]
    need = C.c_size_t()
    _lib.check(lib.quip_qlinear_workspace_bytes(ql._desc_ref, M, C.byref(need)))
    ws = torch.full((need.value,), 0xFF, dtype=torch.uint8, device=DEV)
    ws[:_lib.WS_HEADER_BYTES] = 0
    y = torch.full((M, ql.outfeatures), float('nan'), dtype=torch.float16, device=DEV)
    stream = C.c_void_p(torch.cuda.current_stream().cuda_stream)
    try:
        for k, v in cfg.items():
            _lib.check(lib.quip_config(k.encode(), v))
        before = lib.quip_launch_count()
        _lib.check(lib.quip_qlinear_forward(ql._desc_ref, x.data_ptr(), y.data_ptr(), M, ws.data_ptr(), ws.numel(),
                                            stream))
        launches = lib.quip_launch_count() - before
    finally:
        for k, v in es.DEFAULTS.items():
            lib.quip_config(k.encode(), v)
    torch.cuda.synchronize()
    assert int(ws[:_lib.WS_HEADER_BYTES].max()) == 0, 'split-K counters must be left zeroed'
    return y.cpu().numpy(), launches


def check_routes(c, what):
    ql = build_layer(c)
    want = {}
    for cfg in route_cfgs(c.M):
        p = es.plan(c, cfg)
        key = (es.oracle_route(p['v']), es.oracle_route(p['u']))
        if key not in want:
            want[key] = es.forward(c, *key, device=DEV)[0]
        y, launches = run_forward(ql, c.X, cfg)
        tag = f'{what} M={c.M} {cfg or "defaults"} sides={p["v"]}/{p["u"]}'
        assert_fp16_bits_equal(y, want[key], tag)
        assert launches == p['launches'], (tag, launches, p['launches'])


# ---- family A: dense factors behind a transparent GEMM ----
@pytest.mark.parametrize('K,N', SHAPES)
def test_few_token_sides_bit_exact(K, N):
    """1..8 tokens: fused gather / scatter in pass_fewtok, the one-launch side, and the many-token kernels (fewtok=0)."""
    for M in FEW_M:
        c = a_case(K, N, M, device=DEV)
        check_routes(c, f'A K={K} N={N}')


@pytest.mark.parametrize('K,N', SHAPES)
def test_batched_decode_sides_bit_exact(K, N):
    """9..32 tokens: pass_fewtok with two and four token groups, and (fewtok_max_m=8) side_fused without row sums."""
    for M in MID_M:
        c = a_case(K, N, M, device=DEV)
        check_routes(c, f'A K={K} N={N}')


@pytest.mark.parametrize('K,N', SHAPES)
def test_many_token_sides_bit_exact(K, N):
    """33+ tokens: side_fused with its row sums (partial last 16-token tiles), and the unfused gather / pass / rowsum."""
    for M in many_ms(K, N):
        c = a_case(K, N, M, device=DEV)
        check_routes(c, f'A K={K} N={N}')


# ---- family B: integer sides behind a real asymmetric (or symmetric) GEMM: the row sums of x2 matter ----
B_SHAPES = [(4096, 4096), (2048, 2048), (768, 2048), (4096, 11008)]
B_MS = [5, 17, 33, 47, 300]
HAND_MS = [1, 5, 17, 33, 300]


@pytest.mark.parametrize('symmetric', [False, True])
@pytest.mark.parametrize('K,N', B_SHAPES)
def test_integer_sides_real_gemm_bit_exact(K, N, symmetric):
    for M in B_MS:
        c = b_case(K, N, M, symmetric, device=DEV)
        check_routes(c, f'B K={K} N={N} sym={symmetric}')


# ---- the (64, 32) side_fused instantiation: QuantLinear never builds it (see hand_built_cases) ----
@pytest.mark.parametrize('family', ['A', 'B'])
def test_hand_built_64x32_side_bit_exact(family):
    for M in HAND_MS:
        c = a_case(2048, 2048, M, HAND_64x32, DEV) if family == 'A' else b_case(2048, 2048, M, False, HAND_64x32, DEV)
        if M > 32:
            assert es.plan(c, {})['v'] == 'side_fused'
        check_routes(c, f'{family} hand-built 64x32 V side')


def side_cases():
    """Every case of this file with the side routes it is budgeted for (for the CPU budget test)."""
    for (K, N) in SHAPES:
        for M in FEW_M + MID_M + many_ms(K, N):
            yield a_case(K, N, M), budget_routes(M)
    for (K, N) in B_SHAPES:
        for symmetric in (False, True):
            for M in B_MS:
                yield b_case(K, N, M, symmetric), budget_routes(M)
    for M in HAND_MS:
        yield a_case(2048, 2048, M, HAND_64x32), budget_routes(M)
        yield b_case(2048, 2048, M, False, HAND_64x32), budget_routes(M)
