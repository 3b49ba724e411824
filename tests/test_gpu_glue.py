"""Glue kernels of csrc/glue.cu (quip_rmsnorm / quip_rope / quip_silu_mul) against the torch restatement of the HF Llama
modules (oracle/glue.py, pinned bit-for-bit to transformers' LlamaRMSNorm / apply_rotary_pos_emb / SiLU*up on the CPU in
tests/test_fused_layer.py), at the Llama-2-7B shapes bench.py runs them at.  These are the cases of
tests/quick_glue_check.py; the wider shape sweep is in tests/test_gpu_staged.py."""
import pytest
import torch

pytestmark = pytest.mark.gpu

S, D, INTER, NH, HD = 2048, 4096, 11008, 32, 128


def _rnd(gen, *shape, scale=1.0):
    return (torch.randn(*shape, device='cuda', generator=gen) * scale).half()


def test_rope_kernel_is_bit_exact_at_7b_shapes():
    from oracle.glue import TorchGlue
    from quip_b200.fused import CudaGlue
    g = torch.Generator(device='cuda').manual_seed(0)
    q, k = _rnd(g, 1, S, NH * HD), _rnd(g, 1, S, NH * HD)
    ang = torch.rand(S, HD // 2, device='cuda', generator=g) * 100
    cos, sin = torch.cat((ang.cos(), ang.cos()), -1).half(), torch.cat((ang.sin(), ang.sin()), -1).half()
    q0, k0 = q.clone(), k.clone()
    TorchGlue().rope_(q0, k0, cos, sin, HD)
    CudaGlue().rope_(q, k, cos, sin, HD)
    assert torch.equal(q, q0) and torch.equal(k, k0)


def test_silu_mul_kernel_is_bit_exact_at_7b_shapes():
    from oracle.glue import TorchGlue
    from quip_b200.fused import CudaGlue
    g = torch.Generator(device='cuda').manual_seed(1)
    a, b = _rnd(g, 1, S, INTER, scale=3.0), _rnd(g, 1, S, INTER)
    assert torch.equal(CudaGlue().silu_mul(a, b), TorchGlue().silu_mul(a, b))


def test_rmsnorm_kernel_at_7b_shapes():
    """Only the summation order of the fp32 mean of squares differs from the HF module: a result moves by one fp16 ulp in
    about 2 of 100 000 positions (measured 1.8e-5); the fused residual sum is exact."""
    from oracle.glue import TorchGlue
    from quip_b200.fused import CudaGlue
    g = torch.Generator(device='cuda').manual_seed(2)
    x, r, w = _rnd(g, 1, S, D, scale=2.0), _rnd(g, 1, S, D), _rnd(g, D)
    for eps in (1e-5, 1e-6):
        want, got = TorchGlue().rmsnorm(x, w, eps), CudaGlue().rmsnorm(x, w, eps)
        assert float((want != got).float().mean()) < 1e-3
        assert float((want.float() - got.float()).abs().max()) <= float(want.float().abs().max()) * 2 ** -9
        s0, y0 = TorchGlue().rmsnorm(x, w, eps, residual=r)
        s1, y1 = CudaGlue().rmsnorm(x, w, eps, residual=r)
        assert torch.equal(s0, s1)
        assert float((y0 != y1).float().mean()) < 1e-3
        assert float((y0.float() - y1.float()).abs().max()) <= float(y0.float().abs().max()) * 2 ** -9
