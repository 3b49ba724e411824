"""Glue kernels (csrc/glue.cu), the fused Llama stack / decode step, and batched-decode token counts (9..32) through the
few-token passes.  Written in round 1 after its GPU budget was spent ("staged"); part of the default `-m gpu` run.

Covered: quip_rmsnorm / quip_rope / quip_silu_mul through quip_b200.fused.CudaGlue against the torch restatement
oracle/glue.py (itself pinned bit-for-bit against the HF modules on the CPU, tests/test_fused_layer.py); the fused Llama stack
(QUIP_FUSED_LAYER=1) against the HF decoder layers on a packed model; pass_fewtok_kernel<2>, <4>.
"""
import os

import pytest
import torch

pytestmark = pytest.mark.gpu


def _rand(shape, seed, scale=1.0):
    return (torch.randn(*shape, generator=torch.Generator().manual_seed(seed)) * scale).half().cuda()


@pytest.mark.parametrize('rows,d', [(1, 128), (7, 4096), (2048, 4096), (33, 8192), (5, 2048), (3, 11008), (2, 32768)])
def test_rmsnorm_kernel(rows, d):
    from oracle.glue import TorchGlue
    from quip_b200.fused import CudaGlue
    x, r, w = _rand((1, rows, d), 1, 2.0), _rand((1, rows, d), 2), _rand((d,), 3)
    for eps in (1e-5, 1e-6):
        want = TorchGlue().rmsnorm(x, w, eps)
        got = CudaGlue().rmsnorm(x, w, eps)
        # only the summation order of the fp32 mean differs: a result may move by one fp16 ulp, rarely
        diff = (got.float() - want.float()).abs()
        assert float(diff.max()) <= float(want.float().abs().max()) * 2 ** -9
        assert float((diff > 0).float().mean()) < 5e-3
        s_want, y_want = TorchGlue().rmsnorm(x, w, eps, residual=r)
        s_got, y_got = CudaGlue().rmsnorm(x, w, eps, residual=r)
        assert torch.equal(s_got, s_want)
        assert float(((y_got.float() - y_want.float()).abs() > 0).float().mean()) < 5e-3


@pytest.mark.parametrize('rows,nq,nkv,hd', [(1, 4, 4, 16), (2048, 32, 32, 128), (37, 64, 8, 128), (5, 4, 2, 64), (3, 2, 1, 32)])
def test_rope_kernel_is_bit_exact(rows, nq, nkv, hd):
    from oracle.glue import TorchGlue
    from quip_b200.fused import CudaGlue
    q, k = _rand((1, rows, nq * hd), 4), _rand((1, rows, nkv * hd), 5)
    ang = torch.rand(rows, hd // 2, generator=torch.Generator().manual_seed(6)) * 100
    cos = torch.cat((ang.cos(), ang.cos()), -1).half().cuda()
    sin = torch.cat((ang.sin(), ang.sin()), -1).half().cuda()
    q0, k0 = q.clone(), k.clone()
    TorchGlue().rope_(q0, k0, cos, sin, hd)
    CudaGlue().rope_(q, k, cos, sin, hd)
    assert torch.equal(q, q0) and torch.equal(k, k0)


@pytest.mark.parametrize('n', [8, 4096, 2048 * 11008, 1000 * 8])
def test_silu_mul_kernel(n):
    from oracle.glue import TorchGlue
    from quip_b200.fused import CudaGlue
    g, u = _rand((n,), 7, 3.0), _rand((n,), 8)
    g[:4] = torch.tensor([-70000.0, 70000.0, 0.0, -20.0]).half().cuda()[:4]          # -inf, +inf, 0, deep tail
    want, got = TorchGlue().silu_mul(g, u), CudaGlue().silu_mul(g, u)
    ok = torch.isfinite(want)
    assert torch.equal(torch.isfinite(got), ok)
    diff = (got[ok].float() - want[ok].float()).abs()
    # expf / division are the same libdevice routines torch's silu kernel compiles to; allow an ulp anyway
    assert float((diff > 0).float().mean()) < 1e-3
    assert float(diff.max()) <= float(want[ok].float().abs().max()) * 2 ** -9


def test_glue_argument_errors():
    from quip_b200.fused import CudaGlue
    ops = CudaGlue()
    with pytest.raises(RuntimeError, match='multiple of 8'):
        ops.rmsnorm(_rand((1, 2, 12), 1), _rand((12,), 2), 1e-5)
    with pytest.raises(ValueError, match='contiguous fp16'):
        ops.silu_mul(_rand((4, 16), 1).t(), _rand((16, 4), 2))
    with pytest.raises(ValueError, match='one row'):
        ops.rope_(_rand((1, 4, 64), 1), _rand((1, 4, 64), 2), _rand((3, 16), 3), _rand((3, 16), 4), 16)


@pytest.mark.parametrize('kv_heads', [4, 2])
def test_fused_stack_matches_hf_layers_on_a_packed_model(kv_heads, monkeypatch):
    from transformers import LlamaConfig
    from quip_b200 import evalloop, fused
    from quip_b200.synth import build_synthetic_model
    cfg = LlamaConfig(hidden_size=256, intermediate_size=512, num_hidden_layers=3, num_attention_heads=4,
                      num_key_value_heads=kv_heads, vocab_size=320, max_position_embeddings=128)
    model = build_synthetic_model(cfg, torch.device('cuda:0'), bits=2, incoh='blocked', rescale=True, seed=5, seqlen=64)
    ids = torch.randint(0, 320, (1, 64), generator=torch.Generator().manual_seed(3)).cuda()
    with torch.no_grad():
        h, kw = evalloop.layer_inputs(model, evalloop.LLAMA, ids)
        assert fused.supports(model, h, kw)
        ref = h
        for layer in model.model.layers:
            ref = evalloop._call_layer(layer, ref, kw)
        got = fused.llama_stack(list(model.model.layers), h.clone(), kw)
        err = float((got.float() - ref.float()).norm() / ref.float().norm())
        assert err < 2e-3, err
        monkeypatch.delenv('QUIP_FUSED_LAYER', raising=False)
        nll0 = float(evalloop.sample_nll(model, evalloop.LLAMA, ids))
        monkeypatch.setenv('QUIP_FUSED_LAYER', '1')
        nll1 = float(evalloop.sample_nll(model, evalloop.LLAMA, ids))
        assert abs(nll1 - nll0) / abs(nll0) < 1e-3
        stepper = evalloop.GraphedSampleNLL(model, evalloop.LLAMA, ids)          # the fused stack inside a CUDA graph
        assert abs(float(stepper(ids)) - nll1) / abs(nll1) < 1e-5


@pytest.mark.parametrize('kv_heads', [4, 2])
def test_fused_decode_step_matches_the_torch_glue_step(kv_heads, monkeypatch):
    from transformers import LlamaConfig
    from quip_b200.decode import GraphDecoder
    from quip_b200.synth import build_synthetic_model
    cfg = LlamaConfig(hidden_size=256, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=kv_heads, vocab_size=320, max_position_embeddings=128)
    model = build_synthetic_model(cfg, torch.device('cuda:0'), bits=2, incoh='blocked', rescale=True, seed=5, seqlen=64)
    ids = torch.randint(0, 320, (2, 12), generator=torch.Generator().manual_seed(3)).cuda()
    monkeypatch.delenv('QUIP_FUSED_LAYER', raising=False)
    plain = GraphDecoder(model, max_len=16, batch=2).capture()
    monkeypatch.setenv('QUIP_FUSED_LAYER', '1')
    fusedd = GraphDecoder(model, max_len=16, batch=2).capture()
    assert plain.ops is None and fusedd.ops is not None
    for i in range(ids.shape[1]):
        a, b = plain.step(ids[:, i]).float(), fusedd.step(ids[:, i]).float()
        assert float((a - b).norm() / a.norm()) < 2e-3, i


@pytest.mark.parametrize('K,N,bits,incoh', [(4096, 4096, 2, 'blocked'), (4096, 11008, 2, 'blocked'), (11008, 4096, 2, 'blocked'),
                                             (8192, 1024, 2, 'blocked'), (768, 3072, 4, None), (4096, 4096, 3, 'kron'),
                                             (2048, 8192, 4, 'noperm')])
def test_batched_decode_token_counts_through_the_few_token_passes(K, N, bits, incoh):
    """quip_config('fewtok_max_m', 32): 9..32 tokens run the few-token passes (pass_fewtok_kernel<2>, <4>: the factor
    fragments loaded once, two or four groups of 8 tokens) instead of the 16-token-tile side kernel.  Same results as the
    default route up to the accumulation order, and within the layer tolerance of the fp32 torch restatement."""
    from gpu_util import torch_reference_forward
    from quip_b200 import _lib
    from quip_b200 import quant as Q
    from quip_b200.synth import synth_layer_parts
    lib = _lib.load()
    tp = synth_layer_parts(K=K, N=N, bits=bits, incoh=incoh, rescale=incoh is not None, bias=(N in (1024, 3072)),
                           seed=K + N, qfn='a')
    ql = Q.QuantLinear(infeatures=K, outfeatures=N, **Q.spec_from_parts(tp)).cuda()
    ql.pack_parts(tp)
    x = (torch.randn(32, K, device='cuda') * (1 + 3 * torch.rand(K, device='cuda'))).half()
    want = torch_reference_forward(ql, x)
    try:
        for M in (8, 9, 15, 16, 17, 24, 31, 32):
            _lib.check(lib.quip_config(b'fewtok_max_m', 8))
            base = ql(x[:M]).float()
            _lib.check(lib.quip_config(b'fewtok_max_m', 32))
            y = ql(x[:M]).float()
            assert float((y - want[:M]).norm() / want[:M].norm()) < 1.5e-3, (M, 'vs torch')
            assert float((y - base).norm() / base.norm()) < 1e-3, (M, 'vs default route')
            if M == 8:
                assert torch.equal(y, base)                      # the limit does not touch the <= 8 token route
    finally:
        lib.quip_config(b'fewtok_max_m', 32)              # the library default
    assert lib.quip_config(b'fewtok_max_m', 33) != 0 and lib.quip_config(b'fewtok_max_m', 4) != 0


@pytest.mark.parametrize('rows,n', [(1, 128), (7, 11008), (2048, 11008), (3, 4096), (5, 28672)])
def test_silu_mul_gather_kernel(rows, n):
    """quip_silu_mul_gather: SiLU(gate[ig]) * up[iu] with the packed index ig | iu << 16, bit-identical to gathering first and
    calling quip_silu_mul."""
    from quip_b200.fused import CudaGlue
    g = torch.Generator().manual_seed(n + rows)
    gate, up = _rand((rows, n), 1, 3.0), _rand((rows, n), 2)
    ig, iu = torch.randperm(n, generator=g).cuda(), torch.randperm(n, generator=g).cuda()
    comb = ig | (iu << 16)
    idx = torch.where(comb >= 2 ** 31, comb - 2 ** 32, comb).to(torch.int32).contiguous()
    ops = CudaGlue()
    got = ops.silu_mul_gather(gate, up, idx)
    want = ops.silu_mul(gate[:, ig].contiguous(), up[:, iu].contiguous())
    assert torch.equal(got, want)


def test_layout_variants_are_pure_permutations():
    """QuantLinear.forward_layout: skipping the output gather returns y in U layout order (y_plain = y[..., u_idx]), skipping the
    input gather takes x already in V layout order -- bit-identical data, every token-count route."""
    from quip_b200 import quant as Q
    from quip_b200.synth import synth_layer_parts
    for (K, N) in [(4096, 11008), (11008, 4096), (4096, 4096)]:
        tp = synth_layer_parts(K=K, N=N, bits=2, incoh='blocked', rescale=True, bias=False, seed=K + N)
        ql = Q.QuantLinear(infeatures=K, outfeatures=N, **Q.spec_from_parts(tp)).cuda()
        ql.pack_parts(tp)
        assert ql.layout_variant_ok(True, True)
        x = (torch.randn(300, K, device='cuda') * (1 + 3 * torch.rand(K, device='cuda'))).half()
        vi, ui = ql.gather_index('v'), ql.gather_index('u')
        for M in (1, 8, 24, 300):
            y = ql(x[:M])
            y_layout = ql.forward_layout(x[:M], skip_out=True)
            assert torch.equal(y_layout[:, ui], y), (K, N, M, 'output gather')
            y_in = ql.forward_layout(x[:M][:, vi].contiguous(), skip_in=True)
            assert torch.equal(y_in, y), (K, N, M, 'input gather')
            assert torch.equal(ql.forward_layout(x[:M][:, vi].contiguous(), skip_in=True, skip_out=True)[:, ui], y)


def test_fused_stack_with_folded_gathers_is_bit_identical():
    """llama_stack(fold_gathers=True): gate / up in layout order, one silu_mul_gather, down without its input gather -- the same
    hidden states to the last bit as the stack with the separate gather kernels."""
    from transformers import LlamaConfig
    from quip_b200 import evalloop, fused
    from quip_b200.synth import build_synthetic_model
    cfg = LlamaConfig(hidden_size=4096, intermediate_size=11008, num_hidden_layers=1, num_attention_heads=32,
                      num_key_value_heads=32, vocab_size=320, max_position_embeddings=256)
    model = build_synthetic_model(cfg, torch.device('cuda:0'), bits=2, incoh='blocked', rescale=True, seed=5, seqlen=200)
    ids = torch.randint(0, 320, (1, 200), generator=torch.Generator().manual_seed(3)).cuda()
    with torch.no_grad():
        h, kw = evalloop.layer_inputs(model, evalloop.LLAMA, ids)
        layers = list(model.model.layers)
        assert fused.mlp_layout_plan(layers[0].mlp) is not None
        a = fused.llama_stack(layers, h.clone(), kw, fold_gathers=False)
        b = fused.llama_stack(layers, h.clone(), kw, fold_gathers=True)
    assert torch.equal(a, b)
