"""The quantizer kernels on exactly representable inputs (oracle/exact_quant.py), compared bit for bit with float64
references: quip_ldlq_block and quip_greedy_block alone, LDLQ / LDLQ-RG rounding with greedy passes end to end (the
blocked host loop plus the kernels), and quip_hessian_accumulate.  Each case's budget is proved before it runs."""
import ctypes as C
import functools

import numpy as np
import pytest
import torch

from oracle import exact_quant as eq

pytestmark = pytest.mark.gpu

CNTS = [1, 2, 5, 64, 81, 127, 128]      # 81..128 need more than 48 KiB of shared memory (the opt-in attribute)
MS = [1, 63, 64, 65, 1000]              # around the 64-row CTA
PAD = 7                                 # ld = m + PAD: the padding rows carry a NaN sentinel


def _stream():
    return C.c_void_p(torch.cuda.current_stream().cuda_stream)


def assert_equal_f32(got, want, what, col_block=None):
    """torch.equal on float32; on a mismatch report the count, the first (row, column) and, end to end, its block."""
    want = torch.as_tensor(want).to(got.device, torch.float32)
    assert got.dtype == torch.float32 and got.shape == want.shape, (what, got.dtype, got.shape, want.shape)
    if torch.equal(got, want):
        return
    bad = (got != want).nonzero()
    r, c = (int(v) for v in bad[0])
    blk = ''
    if col_block:
        d, b = got.shape[1], col_block
        i2 = d - ((d - 1 - c) // b) * b
        blk = f', in the column block [{max(0, i2 - b)}, {i2})'
    raise AssertionError(f'{what}: {len(bad)} of {got.numel()} elements differ; first at (row, column) = ({r}, {c}){blk}: '
                         f'got {float(got[r, c])!r} want {float(want[r, c])!r}')


def _padded_t(a, ld, dev='cuda'):
    """(m, n) row-major numpy -> (n, ld) float32 on the device, column j at [j * ld + r], NaN in rows [m, ld)."""
    out = torch.full((a.shape[1], ld), float('nan'), dtype=torch.float32)
    out[:, :a.shape[0]] = torch.from_numpy(np.ascontiguousarray(a.T)).float()
    return out.to(dev)


def _check_padded(t, want, m, what):
    assert_equal_f32(t[:, :m].T.contiguous(), want, what)
    assert bool(torch.isnan(t[:, m:]).all()), f'{what}: a padding row [m, ld) was written'


# ---- quip_ldlq_block alone ----
def ldlq_block_case(m, cnt, bits):
    return eq.make_ldlq_block_case(m, cnt, bits, seed=m * 131 + cnt * 7 + bits)


@pytest.mark.parametrize('bits', [2, 3, 4, 8])
@pytest.mark.parametrize('cnt', CNTS)
def test_ldlq_block_kernel_bit_exact(bits, cnt):
    from quip_b200 import _lib
    lib = _lib.load()
    for m in MS:
        c = ldlq_block_case(m, cnt, bits)
        want_q, want_e, _ = eq.ldlq_block_exact(c)       # raises BudgetError unless the case is exact
        ld = m + PAD
        baseT, wT = _padded_t(c.base, ld), _padded_t(c.w, ld)
        Lb = torch.from_numpy(c.Lb).float().cuda()
        qT = torch.full((cnt, ld), float('nan'), device='cuda')
        errT = torch.full((cnt, ld), float('nan'), device='cuda')
        _lib.check(lib.quip_ldlq_block(_lib.ptr(baseT), _lib.ptr(wT), _lib.ptr(Lb), _lib.ptr(qT), _lib.ptr(errT),
                                       m, ld, cnt, bits, _stream()))
        torch.cuda.synchronize()
        what = f'ldlq_block m={m} cnt={cnt} bits={bits}'
        _check_padded(qT, want_q, m, what + ' q')
        _check_padded(errT, want_e, m, what + ' err')


# ---- quip_greedy_block alone ----
def greedy_block_case(m, cnt):
    return eq.make_greedy_block_case(m, cnt, seed=m * 17 + cnt)


@pytest.mark.parametrize('cnt', CNTS)
def test_greedy_block_kernel_bit_exact(cnt):
    from quip_b200 import _lib
    lib = _lib.load()
    for m in MS:
        c = greedy_block_case(m, cnt)
        want_wr, want_s, st = eq.greedy_block_exact(c)
        assert st['ties'] > 0
        ld = m + PAD
        preT, wrT, sT = _padded_t(c.pre, ld), _padded_t(c.wr, ld), _padded_t(c.s, ld)
        Hb = torch.from_numpy(c.Hb).float().cuda()
        _lib.check(lib.quip_greedy_block(_lib.ptr(preT), _lib.ptr(Hb), _lib.ptr(wrT), _lib.ptr(sT), m, ld, cnt, _stream()))
        torch.cuda.synchronize()
        what = f'greedy_block m={m} cnt={cnt}'
        _check_padded(wrT, want_wr, m, what + ' wr')
        _check_padded(sT, want_s, m, what + ' s')


# ---- end to end: quantize.ldlq_round / ldlq_rg_round with the kernels ----
E2E_CASES = [(70, 96, 2), (1000, 96, 4), (70, 200, 3), (1000, 200, 2), (70, 1416, 2), (1000, 1416, 3)]   # 1416 = 11 * 128 + 8


@functools.lru_cache(maxsize=None)
def e2e_case(m, d, bits):
    return eq.make_ldlq_case(m, d, bits, seed=d + m)


@functools.lru_cache(maxsize=None)
def e2e_exact(m, d, bits, passes):
    return eq.ldlq_exact(e2e_case(m, d, bits), passes)[0]


@pytest.mark.parametrize('m,d,bits', E2E_CASES)
def test_device_cholesky_returns_the_dyadic_factor(m, d, bits):
    """The premise of the end-to-end test: the factor of H = C C^T is C, and cuSOLVER returns it bit for bit."""
    c = e2e_case(m, d, bits)
    H = torch.from_numpy(c.H).float().cuda()
    assert_equal_f32(torch.linalg.cholesky(H), c.C, f'cholesky d={d}')


@pytest.mark.parametrize('m,d,bits', E2E_CASES)
@pytest.mark.parametrize('rg', [False, True], ids=['ldlq', 'ldlq_rg'])
def test_ldlq_round_on_the_device_bit_exact(m, d, bits, rg):
    from quip_b200 import quantize as qz
    c = e2e_case(m, d, bits)
    w, H = c.scrambled() if rg else (c.w, c.H)
    w, H = torch.from_numpy(w).float().cuda(), torch.from_numpy(H).float().cuda()
    fn = qz.ldlq_rg_round if rg else qz.ldlq_round
    for passes in (0, 1, 2):
        want = e2e_exact(m, d, bits, passes)
        if rg:
            want = want[:, c.perm]
        for block in (128, 32):
            got = fn(w, H, bits, passes, block=block)
            assert_equal_f32(got, want, f'{fn.__name__} m={m} d={d} bits={bits} passes={passes} block={block}',
                             col_block=None if rg else block)


# ---- quip_hessian_accumulate ----
HK = [8, 120, 128, 136, 200, 1416]
HT = [1, 31, 32, 33, 255, 256, 257, 513, 4096]


def hessian_batches(T, K):
    """(activations, dtype) per add_batch call: two fp16 (the kernel), one fp32 (the float64 addmm), one fp16."""
    x = [eq.make_hessian_case(T, K, seed=T * 7 + K + i) for i in range(5)]
    return [(np.stack([x[0], x[1]]), torch.float16), (x[2], torch.float16), (x[3], torch.float32), (x[4], torch.float16)]


@pytest.mark.parametrize('K', HK)
def test_hessian_accumulator_bit_exact(K):
    from quip_b200 import quantize as qz
    for T in HT:
        batches = hessian_batches(T, K)
        for x, dt in batches:
            if dt == torch.float16:
                eq.check_hessian(x.reshape(-1, K))
        acc = qz.HessianAccumulator(K, device='cuda')
        nb = 0
        for x, dt in batches:
            acc.add_batch(torch.from_numpy(x).to('cuda', dt))
            nb += x.shape[0] if x.ndim == 3 else 1
        want = torch.from_numpy(eq.hessian_exact([x for x, _ in batches])).cuda()
        got = acc.result()
        assert acc.batches == nb
        what = f'HessianAccumulator K={K} T={T}'
        if not torch.equal(acc.H, want):
            assert_equal_f32(acc.H.float(), want.float(), what + ' float64 H')
            raise AssertionError(f'{what}: float64 H differs below fp32 precision')
        assert_equal_f32(got, (want / nb).float(), what + ' result()')


PREFILL_T = [1, 33, 256, 513]


def _lower_tiles(K):
    tile = np.arange(K) // 128
    return tile[:, None] > tile[None, :]


def prefilled_case(T, K):
    """X and a dyadic H0 with NaN in the lower block triangle (tiles ti > tj of 128 x 128)."""
    rng = np.random.default_rng(T + K)
    H0 = rng.integers(-(1 << 20), 1 << 20, size=(K, K)) / 256.0
    H0[_lower_tiles(K)] = np.nan
    return eq.make_hessian_case(T, K, seed=T * 3 + K), H0


@pytest.mark.parametrize('K', HK)
def test_hessian_kernel_adds_onto_the_upper_block_triangle(K):
    """Called directly on a pre-filled H: tiles ti <= tj (diagonal tiles in full) become H0 + X^T X exactly; the lower
    block triangle, a NaN sentinel, is not touched."""
    from quip_b200 import _lib
    lib = _lib.load()
    nt = -(-K // 128)
    lower = _lower_tiles(K)
    for T in PREFILL_T:
        X, H0 = prefilled_case(T, K)
        eq.check_hessian(X, H0)
        H = torch.from_numpy(H0).cuda()
        x = torch.from_numpy(X).cuda()
        _lib.check(lib.quip_hessian_accumulate(_lib.ptr(x), _lib.ptr(H), T, K, _stream()))
        torch.cuda.synchronize()
        want = H0 + eq.hessian_exact([X])
        low = torch.from_numpy(lower).cuda()
        what = f'hessian kernel K={K} T={T} ({nt} x {nt} tiles)'
        assert bool(torch.isnan(H[low]).all()), f'{what}: the lower block triangle was written'
        got = torch.where(low, 0.0, H)
        ref = torch.from_numpy(np.where(lower, 0.0, want)).cuda()
        if not torch.equal(got, ref):
            bad = (got != ref).nonzero()
            i, j = (int(v) for v in bad[0])
            raise AssertionError(f'{what}: {len(bad)} elements differ; first at ({i}, {j}), tile ({i // 128}, {j // 128}): '
                                 f'got {float(got[i, j])!r} want {float(ref[i, j])!r}')


def cases():
    """Every case of this file, for the host-side budget test: (name, thunk that runs its budget check)."""
    for bits in (2, 3, 4, 8):
        for cnt in CNTS:
            for m in MS:
                yield f'ldlq_block m={m} cnt={cnt} bits={bits}', lambda m=m, cnt=cnt, bits=bits: eq.ldlq_block_exact(ldlq_block_case(m, cnt, bits))
    for cnt in CNTS:
        for m in MS:
            yield f'greedy_block m={m} cnt={cnt}', lambda m=m, cnt=cnt: eq.greedy_block_exact(greedy_block_case(m, cnt))
    for (m, d, bits) in E2E_CASES:
        yield f'ldlq m={m} d={d} bits={bits}', lambda m=m, d=d, bits=bits: e2e_exact(m, d, bits, 2)
    for K in HK:
        for T in HT:
            for x, dt in hessian_batches(T, K):
                if dt == torch.float16:
                    yield f'hessian T={T} K={K}', lambda x=x, K=K: eq.check_hessian(x.reshape(-1, K))
        for T in PREFILL_T:
            yield f'hessian prefilled T={T} K={K}', lambda T=T, K=K: eq.check_hessian(*prefilled_case(T, K))
