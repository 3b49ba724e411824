"""The GPU quantiser (SURVEY section 8f ranks 1-2): LDLQ / LDLQ-RG rounding with the column loop in csrc/ldlq.cu, Hessian
accumulation and the whole quantize_linear flow on the device -- against the LIVE REFERENCE's outputs under tests/golden
(oracle/gen_golden_ldlq.py, gen_golden_quantflow.py) and against the torch loop of quip_b200/quantize.py.

float32 sums are taken in a different (fixed) order than the reference's GEMV, so a rounding decision can flip where
w + feedback lands within ~1e-6 of a half-integer, and the flip then propagates along its row: codes are required to be
identical on >= 99.8 % of the positions and the proxy loss tr((Q-W) H (Q-W)^T) to agree within 0.1 %."""
import os

import numpy as np
import pytest
import torch

from conftest import GOLDEN

pytestmark = pytest.mark.gpu


def _loss(q, w, H):
    d = (q - w).double()
    return float(torch.trace(d @ H.double() @ d.T))


def test_ldlq_kernels_reproduce_the_reference_codes():
    from quip_b200 import quantize as qz
    z = np.load(os.path.join(GOLDEN, 'ldlq.npz'))
    for case in z['cases']:
        key, nbits, npasses = str(case).split(':')
        ci, meth = key.split('_')
        w, H = torch.from_numpy(z[f'{ci}_w']).cuda(), torch.from_numpy(z[f'{ci}_H']).cuda()
        fn = qz.ldlq_round if meth == 'ldlq' else qz.ldlq_rg_round
        want = torch.from_numpy(z[f'{key}_out']).cuda()
        for block in (128, 32):
            got = fn(w, H, int(nbits), int(npasses), block=block)
            assert got.shape == want.shape and float(got.min()) >= 0 and float(got.max()) <= 2 ** int(nbits) - 1
            assert torch.equal(got, torch.round(got))
            same = float((got == want).float().mean())
            assert same > 0.998, (case, block, same)
            assert abs(_loss(got, w, H) / _loss(want, w, H) - 1) < 1e-3, (case, block)
        assert torch.equal(fn(w, H, int(nbits), int(npasses)), fn(w, H, int(nbits), int(npasses)))      # deterministic


@pytest.mark.parametrize('m,d,bits,passes', [(512, 1024, 2, 0), (300, 640, 4, 0), (4096, 4096, 2, 0), (256, 384, 2, 2), (1000, 1408, 3, 1),
                                              (1000, 1416, 3, 1)])
def test_ldlq_kernels_agree_with_the_torch_loop(m, d, bits, passes):
    """Ragged row counts (not a multiple of the 64-row CTA), a last block shorter than 128 columns, greedy passes."""
    from quip_b200 import quantize as qz
    g = torch.Generator(device='cuda').manual_seed(m + d)
    X = torch.randn(2 * d, d, device='cuda', generator=g) * (1 + 3 * torch.rand(d, device='cuda', generator=g))
    H = (X.T @ X) / (2 * d)
    H = H + 0.01 * torch.diagonal(H).mean() * torch.eye(d, device='cuda')
    w = torch.rand(m, d, device='cuda', generator=g) * (2 ** bits - 1)
    got = qz.ldlq_round(w, H, bits, passes)
    want = qz.ldlq_round(w, H, bits, passes, kernels=False)
    same = float((got == want).float().mean())
    assert same > 0.998, same
    assert abs(_loss(got, w, H) / _loss(want, w, H) - 1) < 1e-3
    near = torch.clamp(torch.round(w), 0, 2 ** bits - 1)
    assert _loss(got, w, H) < 0.8 * _loss(near, w, H)


@pytest.mark.parametrize('name', ['plain_a', 'rescale_a'])
def test_quantize_linear_on_the_gpu_reproduces_reference_layers(name):
    """Raw fp16 weight + calibration activations -> Hessian (device) -> preprocessing -> LDLQ kernels -> codes / grid / 1/s,
    against the reference's own quantised layer (tests/golden/quantflow_*.npz)."""
    from quip_b200 import quantize as qz
    z = np.load(os.path.join(GOLDEN, f'quantflow_{name}.npz'))
    W0, X = torch.from_numpy(z['W0']).cuda(), torch.from_numpy(z['X']).cuda()
    acc = qz.HessianAccumulator(W0.shape[1], device='cuda')
    acc.add_batch(X.unsqueeze(0))
    method = {'ldlqRG': 'ldlq_rg'}.get(str(z['method']), str(z['method']))
    parts = qz.quantize_linear(W0, acc.result(), bits=int(z['bits']), method=method, greedy_passes=int(z['npasses']),
                               qfn=str(z['qfn']), rescale=bool(int(z['rescale'])), incoh=None)
    same = np.mean(parts.codes.numpy() == z['codes'])
    assert same > 0.99, same
    if int(z['rescale']):
        np.testing.assert_allclose(parts.scaleWH.numpy(), z['scaleWH'], rtol=1e-4)


def test_ldlq_rg_with_greedy_passes_on_the_projected_layer():
    """quantflow_incoh_rg.npz: the weight and Hessian as the reference's preproc left them (rescaled, projected by its own
    random U / V, damped) -> symmetric 2-bit grid of 2.4 rms (vector_balance.py:521-530) -> LDLQ-RG with two greedy passes."""
    from quip_b200 import quantize as qz
    z = np.load(os.path.join(GOLDEN, 'quantflow_incoh_rg.npz'))
    w, H = torch.from_numpy(z['w_pre']).cuda(), torch.from_numpy(z['H_pre']).cuda()
    bits, maxq = int(z['bits']), float(2 ** int(z['bits']) - 1)
    scale = 2.4 * w.square().mean().sqrt() + 1e-16                              # fp16 arithmetic, as the reference (SURVEY A7)
    t = torch.clamp(((w / scale) + 1) / 2 * maxq, 0, maxq).float()
    codes = qz.ldlq_rg_round(t, H, bits, int(z['npasses']))
    want = torch.from_numpy(z['codes']).cuda().float()
    assert float((codes == want).float().mean()) > 0.995
    assert abs(_loss(codes, t, H) / _loss(want, t, H) - 1) < 2e-3


@pytest.mark.parametrize('K,tokens', [(256, 300), (200, 77), (4096, 2048), (1416, 513)])
def test_hessian_accumulator_on_the_device(K, tokens):
    """quip_hessian_accumulate (tensor-core X^T X with a float64 carry) against the reference's float64 GEMM (method.py:98-123),
    several batches, ragged tiles (K not a multiple of 128), token counts that are not a multiple of the 32-token stage."""
    from quip_b200 import quantize as qz
    g = torch.Generator(device='cuda').manual_seed(K)
    xs = [(torch.randn(2, tokens, K, device='cuda', generator=g) * (1 + 3 * torch.rand(K, device='cuda', generator=g))).half()
          for _ in range(3)]
    ref = torch.zeros(K, K, dtype=torch.float64, device='cuda')
    for x in xs:
        f = x.reshape(-1, K).double()
        ref += f.T @ f
    ref = (ref / 6).float()
    acc = qz.HessianAccumulator(K, device='cuda')
    for x in xs:
        acc.add_batch(x)
    got = acc.result()
    assert acc.batches == 6
    assert torch.equal(got, got.T)
    err = float((got - ref).norm() / ref.norm())
    assert err < 2e-6, err
    assert float(((got - ref).abs() / ref.abs().clamp_min(1e-3 * float(ref.abs().max()))).max()) < 1e-4
    acc2 = qz.HessianAccumulator(K, device='cuda')          # fp32 activations take the float64 GEMM: same result
    for x in xs:
        acc2.add_batch(x.float())
    assert float((acc2.result() - ref).norm() / ref.norm()) < 1e-6
