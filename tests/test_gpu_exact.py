"""The few-token packed kernels (quip_qgemm path 1) and the block-diagonal passes (quip_rot_pass) on exactly
representable inputs, compared bit for bit with fp16(exact result) (oracle/exact.py; the wgmma GEMM is in
tests/test_gpu_exact_tc.py).  Each case's exactness premise is proved first by the budget check of its datapath."""
import pytest
import torch

from exact_util import assert_fp16_bits_equal, fit_xmax
from oracle import exact as ex
from test_gpu_kernels import PASS_CASES

pytestmark = pytest.mark.gpu

DEFAULTS = dict(gemv=1, sk_ksplit=0, gv_int=1, gv_rbc=0, gv_persist=1, gv_tma=1, gv_stream=32)


def _configured(cfg, fn):
    from quip_b200 import _lib
    lib = _lib.load()
    try:
        for k, v in cfg.items():
            _lib.check(lib.quip_config(k.encode(), v))
        return fn()
    finally:
        for k, v in DEFAULTS.items():
            lib.quip_config(k.encode(), v)


def _run_exact(c, what, path=1):
    from gpu_util import run_qgemm
    z, _ = run_qgemm(c.codes, c.scales, c.zeros, c.bits, c.X, path=path, bias=c.bias, symmetric=c.symmetric)
    assert_fp16_bits_equal(z, ex.to_fp16(ex.gemm_exact(c)), what)


# ---- fp16 whole-K kernel (qgemv_kernel): 6-8 tokens, every bits value (gv_int = 0 sends 2-/4-bit there too) ----
GV16_SHAPES = [(176, 11008), (4096, 4096)]


def gv16_case(bits, N, K, M, symmetric):
    return fit_xmax(lambda x: ex.make_gemm_case(bits, N, K, M, symmetric=symmetric, bias=True, xmax=x,
                                                seed=bits * 31 + N + K + M + int(symmetric)), ex.check_gv16)


@pytest.mark.parametrize('bits', [2, 3, 4])
@pytest.mark.parametrize('M', [6, 7, 8])
@pytest.mark.parametrize('gv_rbc', [0, 1])
def test_qgemv_fp16_bit_exact(bits, M, gv_rbc):
    def run():
        for (N, K) in GV16_SHAPES:
            for symmetric in (False, True):
                c = gv16_case(bits, N, K, M, symmetric)
                _run_exact(c, f'qgemv fp16 bits={bits} M={M} N={N} K={K} sym={symmetric} gv_rbc={gv_rbc}')
    _configured(dict(gv_int=0, gv_rbc=gv_rbc), run)


# ---- int8 whole-K kernels: every variant of test_qgemv_whole_k_kernels ----
I8_CFGS = [dict(gv_int=1, gv_rbc=0), dict(gv_int=1, gv_rbc=2), dict(gv_int=1, gv_tma=0, gv_rbc=1, gv_persist=0),
           dict(gv_int=1, gv_tma=0, gv_rbc=2), dict(gv_int=1, gv_stream=1)]


def i8_shapes(cfg):
    return [(2400, 11008), (4096, 4096)] if cfg.get('gv_stream') else [(176, 11008), (272, 1024), (4096, 4096)]


def i8_case(bits, N, K, M):
    """Every token's amax is 2^5 or 2^6 (so x 2^22/amax is an exact integer); the last token is all zero."""
    def make(x):
        c = ex.make_gemm_case(bits, N, K, M, symmetric=False, bias=True, xmax=x, seed=bits * 17 + N + K + M,
                              rows=(), pow2_amax=(5, 6))
        if M > 1:
            c.X[M - 1] = 0
        return c
    return fit_xmax(make, ex.check_i8, top=16)


@pytest.mark.parametrize('bits', [2, 4])
@pytest.mark.parametrize('M', [1, 2, 3, 5])
@pytest.mark.parametrize('cfg', I8_CFGS, ids=lambda d: '-'.join(f'{k}{v}' for k, v in d.items()))
def test_qgemv_int8_bit_exact(bits, M, cfg):
    def run():
        for (N, K) in i8_shapes(cfg):
            c = i8_case(bits, N, K, M)
            _run_exact(c, f'qgemv int8 {cfg} bits={bits} M={M} N={N} K={K}')
    _configured(cfg, run)


# ---- split-K mma.sync kernel (qgemm_skinny_kernel) ----
SK_K = 33 * 128                    # 33 super-blocks: the last K split is shorter than the others
SK_SHAPES = [(176, SK_K), (4096, SK_K)]


def sk_case(bits, N, K, M, symmetric):
    return ex.make_gemm_case(bits, N, K, M, symmetric=symmetric, bias=not symmetric, xmax=ex.gemm_xmax(bits, K, symmetric),
                             seed=bits * 7 + N + M + int(symmetric))


@pytest.mark.parametrize('bits', [2, 3, 4])
@pytest.mark.parametrize('M', [1, 9, 17, 32])
def test_skinny_split_k_bit_exact(bits, M):
    # one split, two, the heuristic (4 at N = 176, 2 at N = 4096); one split stages all 33 x 128 k of up to 16
    # tokens (32 do not fit shared memory, and the kernel refuses them)
    for ksplit in ((1, 2, 0) if M <= 16 else (2, 0)):
        def run():
            for (N, K) in SK_SHAPES:
                for symmetric in (False, True):
                    c = sk_case(bits, N, K, M, symmetric)
                    ex.check_mma(c)
                    _run_exact(c, f'skinny bits={bits} M={M} N={N} K={K} sym={symmetric} sk_ksplit={ksplit}')
        _configured(dict(gemv=0, sk_ksplit=ksplit), run)


def chunk_case():
    """100 tokens = three 32-token chunks through the split-K kernel + 4 through the int8 whole-K kernel."""
    return ex.make_gemm_case(2, 256, 1024, 100, symmetric=False, bias=True, xmax=16, seed=100,
                             rows=('max', 'zero'), pow2_amax=(5, 6))


def test_path1_chunk_loop_bit_exact():
    c = chunk_case()
    ex.check_mma(c)
    ex.check_i8(c)
    _run_exact(c, 'path 1 at 100 tokens')


# ---- block-diagonal passes ----
PASS_XMAX = 32


def pass_ms(p):
    return [1, 7, 37, 300] + ([2048] if p > 64 else [])


def pass_impls(p):
    """0: the routing of the forward (few-token kernel up to 32 tokens); 1: the generic CUDA-core kernel;
    2: tensor cores only (small-block kernels; wgmma DENSE pass above 32 tokens for p > 64); 3: mma.sync big-block."""
    return [0, 1, 2] if p <= 64 else [0, 1, 2, 3]


def _pass_exact_dev(X, F, p, nblk, strided):
    x = torch.from_numpy(X).cuda().double()
    Fb = torch.from_numpy(F).cuda().double().expand(nblk, p, p)
    M = X.shape[0]
    if strided:
        out = torch.einsum('bij,mjb->mib', Fb, x.reshape(M, p, nblk))
    else:
        out = torch.einsum('bij,mbj->mbi', Fb, x.reshape(M, nblk, p))
    return out.reshape(M, -1).float().half().cpu().numpy()        # exact in fp32: one rounding


@pytest.mark.parametrize('p,nblk,strided,shared', PASS_CASES)
def test_rot_pass_bit_exact(p, nblk, strided, shared):
    from gpu_util import run_pass
    for M in pass_ms(p):
        X, F = ex.make_pass_case(p, nblk, shared, M, xmax=PASS_XMAX, seed=p * 1000 + nblk + M)
        ex.check_pass(X, F)
        want = _pass_exact_dev(X, F, p, nblk, strided)
        for impl in pass_impls(p):
            got = run_pass(X, F, p, nblk, strided, impl=impl)
            assert_fp16_bits_equal(got, want, f'rot_pass p={p} nblk={nblk} strided={strided} shared={shared} '
                                              f'M={M} impl={impl}')


def exact_cases():
    """Every packed case of this file, for the host-side budget test: (case, budget checks)."""
    for bits in (2, 3, 4):
        for M in (6, 7, 8):
            for (N, K) in GV16_SHAPES:
                for symmetric in (False, True):
                    yield gv16_case(bits, N, K, M, symmetric), (ex.check_gv16,)
        for M in (1, 9, 17, 32):
            for (N, K) in SK_SHAPES:
                for symmetric in (False, True):
                    yield sk_case(bits, N, K, M, symmetric), (ex.check_mma,)
    for bits in (2, 4):
        for M in (1, 2, 3, 5):
            for (N, K) in sorted({s for cfg in I8_CFGS for s in i8_shapes(cfg)}):
                yield i8_case(bits, N, K, M), (ex.check_i8,)
    yield chunk_case(), (ex.check_mma, ex.check_i8)


def pass_cases():
    for (p, nblk, strided, shared) in PASS_CASES:
        for M in pass_ms(p):
            yield ex.make_pass_case(p, nblk, shared, M, xmax=PASS_XMAX, seed=p * 1000 + nblk + M)
