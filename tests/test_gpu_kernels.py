"""CUDA kernels vs the CPU oracle, through the C ABI.  Everything except the wgmma GEMM (which has
its own file so a protocol bug there cannot poison this process's CUDA context)."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN
from oracle import butterfly as obf
from oracle import forward as ofw
from oracle import packing as opk
from oracle import qmath

pytestmark = pytest.mark.gpu

f16, f32 = np.float16, np.float32


def _rel(a, b):
    return ofw.rel_err(a, b)


@pytest.mark.parametrize('bits', [2, 3, 4])
@pytest.mark.parametrize('shape', [(16, 128), (48, 384), (4096, 4096), (176, 11008)])
def test_gpu_packer_bit_exact(bits, shape):
    from quip_b200 import quant as Q
    rng = np.random.default_rng(bits + shape[0])
    codes = rng.integers(0, 1 << bits, size=shape, dtype=np.uint8)
    q = Q.pack_codes(torch.from_numpy(codes).cuda(), bits)
    want = opk.native_pack(codes, bits)
    np.testing.assert_array_equal(q.cpu().numpy(), want)
    back = Q.unpack_codes(q, *shape, bits)
    np.testing.assert_array_equal(back.cpu().numpy(), codes)


def test_reference_layouts_decode_on_gpu():
    from quip_b200 import quant as Q
    z = np.load(os.path.join(GOLDEN, 'packing_ref.npz'))
    for bits in (3, 4):
        codes = z[f'codes{bits}']
        N, K = codes.shape
        got = Q.convert_ref_qweight(torch.from_numpy(z[f'qweight{bits}']).cuda(), K, N, bits)
        np.testing.assert_array_equal(got.cpu().numpy(), codes)
    rng = np.random.default_rng(0)
    codes = rng.integers(0, 4, size=(32, 256), dtype=np.uint8)
    got = Q.convert_ref_qweight(torch.from_numpy(opk.ref_pack2(codes)).cuda(), 256, 32, 2)
    np.testing.assert_array_equal(got.cpu().numpy(), codes)


@pytest.mark.parametrize('M,n', [(1, 128), (5, 384), (64, 11008)])
def test_gather_scale_bias(M, n):
    from gpu_util import run_gather
    rng = np.random.default_rng(n)
    X = rng.standard_normal((M, n)).astype(f16)
    idx = rng.permutation(n)
    scale = (0.5 + rng.random(n)).astype(f32)
    bias = rng.standard_normal(n).astype(f16)
    got = run_gather(X, idx, scale, bias)
    want = (X.astype(np.float64)[:, idx] * scale[idx][None, :] + bias.astype(np.float64)[None, :])
    # the kernel contracts scale and bias with one fp32 FMA before the fp16 rounding: <= 1 ulp from this
    np.testing.assert_allclose(got.astype(np.float64), want, rtol=1.5e-3, atol=1e-6)
    np.testing.assert_array_equal(run_gather(X, idx), X[:, idx])
    np.testing.assert_array_equal(run_gather(X, None, scale), (X.astype(f32) * scale[None, :]).astype(f16))


PASS_CASES = [
    # p, nblk, strided, shared
    (16, 16, False, False), (16, 16, True, False), (24, 16, True, False), (16, 24, False, False),
    (40, 16, False, False), (16, 40, True, False), (8, 16, True, False), (16, 8, False, False),
    (64, 64, False, False), (64, 64, True, False), (64, 32, True, False), (32, 64, False, False),
    (48, 16, False, False), (16, 48, True, False), (64, 64, True, True), (64, 64, False, True),
    (688, 16, False, False), (16, 688, True, False), (224, 32, False, False), (96, 32, False, False),
    (128, 64, False, True), (43, 16, False, False), (16, 43, True, False), (7, 9, True, False),
]


@pytest.mark.parametrize('p,nblk,strided,shared', PASS_CASES)
@pytest.mark.parametrize('M', [1, 37, 300])
def test_rot_pass_vs_oracle(p, nblk, strided, shared, M):
    from gpu_util import run_pass
    n = p * nblk
    rng = np.random.default_rng(p * 1000 + nblk + M)
    X = rng.standard_normal((M, n)).astype(f16)
    F = (rng.standard_normal((1 if shared else nblk, p, p)) / np.sqrt(p)).astype(f16)
    want = obf.apply_pass(X.astype(np.float64), F.astype(np.float64), p, nblk, strided)
    got = run_pass(X, F, p, nblk, strided, impl=0)
    assert got.shape == want.shape
    assert _rel(got, want) < 4e-4, (p, nblk, strided, shared, M)
    # the tensor-core kernels and the generic CUDA-core kernel agree (same fp16 output rounding)
    simple = run_pass(X, F, p, nblk, strided, impl=1)
    assert _rel(simple, want) < 4e-4
    assert _rel(got, simple) < 3e-4


def _qgemm_case(bits, N, K, M, symmetric, seed):
    rng = np.random.default_rng(seed)
    codes = rng.integers(0, 1 << bits, size=(N, K), dtype=np.uint8)
    scales = (0.01 + 0.02 * rng.random((N, 1))).astype(f32)
    cbar = ((1 << bits) - 1) / 2
    if symmetric:
        zeros = (scales * f32(cbar)).astype(f32)
    else:
        zeros = (scales * rng.integers(0, 1 << bits, size=(N, 1)).astype(f32)).astype(f32)
    X = (rng.standard_normal((M, K)) * (1 + 3 * rng.random(K))[None, :]).astype(f16)
    bias = rng.standard_normal(N).astype(f16)
    Qm = scales.astype(np.float64) * codes.astype(np.float64) - zeros.astype(np.float64)
    want = X.astype(np.float64) @ Qm.T + bias.astype(np.float64)[None, :]
    return codes, scales, zeros, X, bias, want


@pytest.mark.parametrize('bits', [2, 3, 4])
@pytest.mark.parametrize('M', [1, 3, 8, 9, 16, 17, 32])
@pytest.mark.parametrize('symmetric', [True, False])
def test_qgemm_skinny_vs_oracle(bits, M, symmetric):
    from gpu_util import run_qgemm
    for (N, K) in [(64, 128), (48, 384), (256, 1024), (4096, 4096)]:
        codes, scales, zeros, X, bias, want = _qgemm_case(bits, N, K, M, symmetric, bits * 100 + M)
        z, xsum = run_qgemm(codes, scales, zeros, bits, X, path=1, bias=bias, symmetric=symmetric)
        np.testing.assert_allclose(xsum, X.astype(np.float64).sum(1), rtol=1e-4, atol=1e-2)
        assert not np.isnan(z.astype(f32)).any()
        assert _rel(z, want) < 3e-4, (bits, M, symmetric, N, K, _rel(z, want))


@pytest.mark.parametrize('bits', [2, 3, 4])
@pytest.mark.parametrize('M', [1, 2, 4, 5, 6, 8])
@pytest.mark.parametrize('cfg', [dict(gv_int=1, gv_rbc=0), dict(gv_int=1, gv_rbc=2), dict(gv_int=0, gv_rbc=1),
                                 dict(gv_int=1, gv_tma=0, gv_rbc=1, gv_persist=0), dict(gv_int=1, gv_tma=0, gv_rbc=2),
                                 dict(gv_int=1, gv_stream=1)])
def test_qgemv_whole_k_kernels(bits, M, cfg):
    """The few-token kernels (int8 tensor path for <= 5 tokens, offset-free fp16 path above): odd numbers of k
    super-blocks, ragged row tiles, a token with a huge outlier (the int8 path scales per token by amax) and an
    all-zero token."""
    from gpu_util import run_qgemm
    from quip_b200 import _lib
    lib = _lib.load()
    try:
        for k, v in cfg.items():
            lib.quip_config(k.encode(), v)
        shapes = [(2400, 11008), (4096, 4096)] if cfg.get('gv_stream') else [(176, 11008), (272, 1024), (4096, 4096)]
        for (N, K) in shapes:
            codes, scales, zeros, X, bias, want = _qgemm_case(bits, N, K, M, False, bits * 10 + M)
            X = X.copy()
            X[0, 7] = f16(3000.0)                      # outlier: amax/sigma ~ 1000
            if M > 1:
                X[M - 1, :] = 0
            Qm = scales.astype(np.float64) * codes.astype(np.float64) - zeros.astype(np.float64)
            want = X.astype(np.float64) @ Qm.T + bias.astype(np.float64)[None, :]
            z, _ = run_qgemm(codes, scales, zeros, bits, X, path=1, bias=bias, symmetric=False)
            assert not np.isnan(z.astype(f32)).any()
            assert _rel(z, want) < 3e-4, (bits, M, cfg, N, K, _rel(z, want))
            if M > 1:
                np.testing.assert_allclose(z[M - 1].astype(f32), bias.astype(f32), atol=2e-3)
    finally:
        for k, v in dict(gv_int=1, gv_rbc=0, gv_persist=1, gv_tma=1, gv_stream=32).items():
            lib.quip_config(k.encode(), v)


def test_qgemm_skinny_large_M_loops():
    from gpu_util import run_qgemm
    codes, scales, zeros, X, bias, want = _qgemm_case(2, 256, 512, 100, False, 5)
    z, _ = run_qgemm(codes, scales, zeros, 2, X, path=1, bias=bias, symmetric=False)
    assert _rel(z, want) < 3e-4


@pytest.mark.parametrize('bits', [2, 3, 4])
@pytest.mark.parametrize('N,K', [(256, 1024), (4096, 4096), (200, 96), (11008, 4096)])
def test_vecquant_matmul_on_the_reference_layout(bits, N, K):
    """quip_vecquant_matmul (the stand-in for quant_cuda.vecquant3matmul / vecquant4matmul, quant.py:229-230): one fp32
    token against the reference's own packed layout, accumulated in place."""
    import ctypes as C
    from quip_b200 import _lib
    lib = _lib.load()
    rng = np.random.default_rng(bits * 7 + N)
    codes = rng.integers(0, 1 << bits, size=(N, K), dtype=np.uint8)
    ref = {2: opk.ref_pack2, 3: opk.ref_pack3, 4: opk.ref_pack4}[bits](codes)
    scales = (0.01 + 0.02 * rng.random(N)).astype(f32)
    zeros = (scales * rng.integers(0, 1 << bits, size=N)).astype(f32)
    x = rng.standard_normal(K).astype(f32)
    y0 = rng.standard_normal(N).astype(f32)
    want = y0.astype(np.float64) + (scales.astype(np.float64)[:, None] * codes - zeros.astype(np.float64)[:, None]) @ x.astype(np.float64)
    t = lambda a: torch.from_numpy(np.ascontiguousarray(a)).cuda()
    mat, vec, mul, sc, ze = t(ref.astype(np.int32)), t(x), t(y0), t(scales), t(zeros)
    _lib.check(lib.quip_vecquant_matmul(_lib.ptr(vec), _lib.ptr(mat), _lib.ptr(mul), _lib.ptr(sc), _lib.ptr(ze), K, N, bits,
                                        C.c_void_p(torch.cuda.current_stream().cuda_stream)))
    torch.cuda.synchronize()
    assert _rel(mul.cpu().numpy(), want) < 1e-5


def test_reference_quant3linear_module_runs_and_converts():
    """A Quant3Linear state_dict as the reference's pack() writes it (golden packing_ref.npz) loads into the same-named module
    here, runs one token through the vecquant stand-in, and converts to the native QuantLinear with the same result."""
    from quip_b200 import quant as Q
    z = np.load(os.path.join(GOLDEN, 'packing_ref.npz'))
    codes = z['codes3']
    N, K = codes.shape
    m = Q.Quant3Linear(K, N)
    sd = dict(qweight=torch.from_numpy(z['qweight3']), scales=torch.from_numpy(z['scales3']),
              zeros=torch.from_numpy(z['stored_zeros3']), bias=torch.linspace(-1, 1, N))
    m.load_state_dict(sd)
    m = m.cuda()
    rng = np.random.default_rng(3)
    x = torch.from_numpy(rng.standard_normal(K).astype(f32)).cuda()
    W = z['scales3'].astype(np.float64) * codes - z['stored_zeros3'].astype(np.float64)
    want = W @ x.cpu().numpy().astype(np.float64) + np.linspace(-1, 1, N)
    y = m(x.reshape(1, 1, K))
    assert y.shape == (1, 1, N) and _rel(y.reshape(-1).cpu().numpy(), want) < 1e-5
    with pytest.raises(ValueError, match='single token'):
        m(torch.zeros(2, K, device='cuda'))
    # K = 1024 and N = 16 suit the native layout too
    y2 = m.to_native()(x.half().reshape(1, K)).float().reshape(-1).cpu().numpy()
    assert _rel(y2, want) < 2e-3
