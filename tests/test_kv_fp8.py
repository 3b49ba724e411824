"""The e4m3 KV cache of generation (PromptDecoder / generate with kv_dtype=torch.float8_e4m3fn) on tiny fp32 HF models on
the CPU, where the step is the torch restatement of quip_decode_attention on an e4m3 cache, against oracle/kvfp8.py and an
fp32-cache decoder; and the argument checks of the C ABI on e4m3 caches."""
import ctypes as C

import pytest
import torch

from oracle import kvfp8
from quip_b200 import _lib
from quip_b200.decode import GraphDecoder, PromptDecoder, generate

from test_generate import KINDS, _model, _prompts

FP8 = torch.float8_e4m3fn


def _bytes(t):
    return t.view(torch.uint8)


def test_oracle_edge_cases():
    x = torch.tensor([[448.0, -3.0, 1.0, 0.0], [-448.0, 2.0, 0.5, 0.25]])
    q, s = kvfp8.quantize(x)
    assert s.tolist() == [1.0, 1.0]                                    # amax exactly 448: s = 1
    assert _bytes(q)[0, 0] == 0x7E and _bytes(q)[1, 0] == 0xFE         # +-448, the largest finite e4m3
    torch.testing.assert_close(kvfp8.dequantize(q, s), x, rtol=0, atol=0)
    q, s = kvfp8.quantize(torch.zeros(3, 64))
    assert torch.equal(s, torch.ones(3)) and not _bytes(q).any()
    # amax 448 (s = 1): 2^-8 and 3 * 2^-9 are e4m3 subnormals (steps of 2^-9 below 2^-6), 2^-11 rounds to zero (tie to even)
    q, s = kvfp8.quantize(torch.tensor([448.0, 2.0 ** -8, 3 * 2.0 ** -9, 2.0 ** -11, -(2.0 ** -9)]))
    assert _bytes(q).tolist() == [0x7E, 0x02, 0x03, 0x00, 0x81]
    g = torch.Generator().manual_seed(0)
    x = torch.randn(256, 128, generator=g) * torch.logspace(-6, 3, 256)[:, None]
    q, s = kvfp8.quantize(x)
    err = (kvfp8.dequantize(q, s) - x).abs()
    assert (err <= 2.0 ** -4 * x.abs().amax(-1, keepdim=True)).all()


def test_the_decoder_restatement_is_the_oracle():
    from quip_b200.decode import _e4m3_dequantize, _e4m3_quantize
    g = torch.Generator().manual_seed(1)
    x = torch.randn(4, 3, 9, 64, generator=g) * 10.0 ** torch.randint(-4, 4, (4, 3, 9, 1), generator=g)
    x[0, 0, 0] = 0.0
    q, s = _e4m3_quantize(x)
    q0, s0 = kvfp8.quantize(x)
    assert torch.equal(_bytes(q), _bytes(q0)) and torch.equal(s, s0)
    assert torch.equal(_e4m3_dequantize(q, s, torch.float32), kvfp8.dequantize(q0, s0))


def _pair(kind, max_len, batch, **kw):
    m = _model(kind)
    return m, PromptDecoder(m, max_len=max_len, batch=batch, kv_dtype=FP8, **kw), PromptDecoder(m, max_len=max_len,
                                                                                                batch=batch, **kw)


@pytest.mark.parametrize('kind', KINDS)
def test_prefill_stores_the_oracle_quantization_of_the_model_keys(kind):
    m, f8, ref = _pair(kind, 24, 3)
    prompts = _prompts(seed=3, lens=(7, 3, 10))
    with torch.no_grad():
        torch.testing.assert_close(f8.prefill(prompts), ref.prefill(prompts), rtol=0, atol=0)   # logits from the fp32 keys
    P = 10
    for cache, scales, src in ((f8.k_cache, f8.k_scale, ref.k_cache), (f8.v_cache, f8.v_scale, ref.v_cache)):
        q, s = kvfp8.quantize(src[:, :, :, :P])
        assert torch.equal(_bytes(cache[:, :, :, :P]), _bytes(q)) and torch.equal(scales[:, :, :, :P], s)
        assert not _bytes(cache[:, :, :, P:]).any() and not scales[:, :, :, P:].any()


@pytest.mark.parametrize('kind', KINDS)
def test_appends_and_logits_against_the_fp32_cache_decoder(kind):
    """Teacher-forced: both decoders take the same tokens.  A layer-0 key / value depends only on the token and its
    position, so every layer-0 slot the fp8 decoder appends is the oracle quantization of the fp32 decoder's slot.  The
    logits differ by the e4m3 rounding of the cache: relative norm error within one e4m3 step (2^-4)."""
    m, f8, ref = _pair(kind, 20, 3)
    prompts = _prompts(seed=4, lens=(5, 2, 8))
    ids = torch.randint(3, 199, (3, 7), generator=torch.Generator().manual_seed(5))
    worst = 0.0
    with torch.no_grad():
        errs = [float((f8.prefill(prompts) - ref.prefill(prompts)).norm())]
        for i in range(ids.shape[1]):
            a, b = f8.step(ids[:, i]), ref.step(ids[:, i])
            worst = max(worst, float((a - b).norm() / b.norm()))
    assert errs[0] == 0.0
    for b, p in enumerate(prompts):
        slots = torch.arange(p.numel(), p.numel() + ids.shape[1])
        for cache, scales, src in ((f8.k_cache, f8.k_scale, ref.k_cache), (f8.v_cache, f8.v_scale, ref.v_cache)):
            q, s = kvfp8.quantize(src[0, b, :, slots])
            assert torch.equal(_bytes(cache[0, b, :, slots]), _bytes(q)) and torch.equal(scales[0, b, :, slots], s)
    print(f'{kind}: fp8 vs fp32 cache logits, worst relative norm error {worst:.2e}')
    assert worst <= 2.0 ** -4, worst


@pytest.mark.parametrize('kind', ['llama_gqa', 'opt_post_ln'])
def test_generate_returns_the_tokens_of_the_fp8_decoder_stepped_by_hand(kind):
    m = _model(kind)
    prompts, n = _prompts(seed=6), 9
    out = generate(m, prompts, n, kv_dtype=FP8)
    dec = PromptDecoder(m, max_len=max(p.numel() for p in prompts) + n, batch=3, max_new=n, kv_dtype=FP8)
    with torch.no_grad():
        dec.prefill(prompts)
        for _ in range(n - 1):
            dec.step()
    for b in range(3):
        assert torch.equal(out[b], dec.generated[b])


def test_reset_zeroes_the_scales_and_starts_over():
    m = _model('llama_mha')
    dec = PromptDecoder(m, max_len=12, batch=2, max_new=4, kv_dtype=FP8)
    with torch.no_grad():
        dec.prefill(_prompts(seed=7, lens=(3, 6)))
        dec.step()
        dec.reset()
        assert not dec.k_scale.any() and not dec.v_scale.any() and not _bytes(dec.k_cache).any()
        fresh = PromptDecoder(m, max_len=12, batch=2, max_new=4, kv_dtype=FP8)
        for d in (dec, fresh):
            d.prefill(_prompts(seed=8, lens=(4, 2)))
            for _ in range(3):
                d.step()
    assert torch.equal(dec.generated, fresh.generated)


def test_fp8_decoder_holds_no_wide_cache_and_its_bytes_shrink():
    m = _model('llama_gqa')
    f8 = PromptDecoder(m, max_len=16, batch=3, kv_dtype=FP8)
    shape = (len(f8.layers), 3, f8.nkv, 16, f8.hd)
    wide = [k for k, t in vars(f8).items() if torch.is_tensor(t) and tuple(t.shape) == shape and t.dtype != FP8]
    assert not wide, wide
    assert f8.k_cache.dtype == f8.v_cache.dtype == FP8 and tuple(f8.k_cache.shape) == shape
    assert f8.k_scale.dtype == torch.float32 and tuple(f8.k_scale.shape) == shape[:-1]
    got = sum(t.numel() * t.element_size() for t in (f8.k_cache, f8.v_cache, f8.k_scale, f8.v_scale))
    fp16 = 2 * f8.k_cache.numel() * 2
    assert got * 2 * f8.hd == fp16 * (f8.hd + 4)


def test_kv_dtype_choices():
    m = _model('llama_mha')
    for dt in (None, torch.float16, torch.float32):
        dec = PromptDecoder(m, max_len=8, batch=1, kv_dtype=dt)
        assert dec.k_cache.dtype == torch.float32 and dec.k_scale is None
    for bad in (torch.bfloat16, torch.int8, torch.float8_e5m2, 'fp8'):
        with pytest.raises(ValueError, match='kv_dtype'):
            PromptDecoder(m, max_len=8, batch=1, kv_dtype=bad)
    with pytest.raises(ValueError, match='PromptDecoder takes float8_e4m3fn'):
        GraphDecoder(m, max_len=8, batch=1, kv_dtype=FP8)
    with pytest.raises(ValueError, match='kv_dtype'):
        generate(m, _prompts()[:1], 2, kv_dtype=torch.int8)


def test_e4m3_cache_descriptor_argument_errors_surface_as_messages():
    lib = _lib.load()
    buf, ws = 64, 1 << 20

    def call(B=2, nh=8, nkv=2, hd=128, max_len=256, q=buf, ks=buf, vs=buf, pos=buf, wsb=ws, out=buf, kc=buf):
        kv = _lib.QuipKvCache(k=kc, v=buf, k_scale=ks, v_scale=vs, format=_lib.QUIP_KV_E4M3, nkv=nkv, hd=hd,
                              max_len=max_len)
        return lib.quip_decode_attention(kv, q, buf, buf, pos, out, B, nh, 1.0, buf, wsb, None)
    assert call(hd=96) == 1 and b'quip_decode_attention: head_dim 96' in lib.quip_last_error()
    assert call(nh=6, nkv=4) == 1 and b'nh % nkv' in lib.quip_last_error()
    assert call(nh=32, nkv=2) == 1 and b'at most 8' in lib.quip_last_error()
    assert call(q=None) == 1 and b'null' in lib.quip_last_error()
    assert call(ks=None) == 1 and b'null' in lib.quip_last_error()
    assert call(vs=None) == 1 and b'null' in lib.quip_last_error()
    assert call(kc=72) == 1 and b'16-byte aligned' in lib.quip_last_error()
    assert call(vs=66) == 1 and b'4-byte aligned' in lib.quip_last_error()
    assert call(wsb=100) == 1 and b'workspace' in lib.quip_last_error()
    need = C.c_size_t(0)
    assert lib.quip_decode_attention_workspace_bytes(2, 8, 128, 256, C.byref(need)) == 0
    assert call(wsb=need.value - 1) == 1 and b'workspace' in lib.quip_last_error()
    assert call(B=0, wsb=0) == 0
    with pytest.raises(_lib.QuipError, match='head_dim'):
        _lib.check(call(hd=32))
    # the format is stated, never inferred from the scales
    fp16 = _lib.QuipKvCache(k=buf, v=buf, k_scale=buf, v_scale=buf, format=_lib.QUIP_KV_FP16, nkv=2, hd=128, max_len=256)
    assert lib.quip_decode_attention(fp16, buf, buf, buf, buf, buf, 2, 8, 1.0, buf, ws, None) == 1
    assert b'given for an fp16 cache' in lib.quip_last_error()
    fp16.format = 0
    assert lib.quip_decode_attention(fp16, buf, buf, buf, buf, buf, 2, 8, 1.0, buf, ws, None) == 1
    assert b'format 0' in lib.quip_last_error()
    assert lib.quip_decode_attention(None, buf, buf, buf, buf, buf, 2, 8, 1.0, buf, ws, None) == 1
    assert b'null cache descriptor' in lib.quip_last_error()

    def quant(src=buf, cache=buf, scales=buf, B=2, nkv=4, P=10, max_len=16, hd=64):
        return lib.quip_kv_quantize_fp8(src, cache, scales, B, nkv, P, max_len, hd, None)
    assert quant(hd=80) == 1 and b'quip_kv_quantize_fp8: head_dim 80' in lib.quip_last_error()
    assert quant(P=17) == 1 and b'P <= max_len' in lib.quip_last_error()
    assert quant(P=-1) == 1 and b'bad sizes' in lib.quip_last_error()
    assert quant(nkv=0) == 1 and b'bad sizes' in lib.quip_last_error()
    assert quant(cache=None) == 1 and b'null' in lib.quip_last_error()
    assert quant(scales=None) == 1 and b'null' in lib.quip_last_error()
    assert quant(src=72) == 1 and b'aligned' in lib.quip_last_error()
    assert quant(scales=66) == 1 and b'aligned' in lib.quip_last_error()
    assert quant(B=0) == 0 and quant(P=0) == 0                        # nothing to quantize


def test_fp8_wrappers_refuse_cpu_tensors_and_mismatched_scales():
    from quip_b200 import fused
    q = torch.zeros(1, 4, 64, dtype=torch.float16)
    kv = torch.zeros(1, 4, 64, dtype=torch.float16)
    cache = torch.zeros(1, 4, 16, 64, dtype=FP8)
    sc = torch.zeros(1, 4, 16)
    pos = torch.zeros(1, dtype=torch.long)
    with pytest.raises(RuntimeError, match='CUDA device only'):
        fused.decode_attention(q, kv, kv, cache, cache.clone(), pos, 0.125, k_scale=sc, v_scale=sc.clone())
    with pytest.raises(ValueError, match='need k_scale and v_scale'):
        fused.decode_attention(q, kv, kv, cache, cache.clone(), pos, 0.125)
    with pytest.raises(ValueError, match='do not agree'):
        fused.decode_attention(q, kv, kv, cache, cache.clone(), pos, 0.125, k_scale=sc, v_scale=torch.zeros(1, 4, 15))
    with pytest.raises(ValueError, match='fp32 scales'):
        fused.decode_attention(q, kv, kv, cache, cache.clone(), pos, 0.125, k_scale=sc, v_scale=sc.half())
    with pytest.raises(ValueError, match='float8_e4m3fn caches only'):
        fused.decode_attention(q, kv, kv, cache.half(), cache.half(), pos, 0.125, k_scale=sc, v_scale=sc.clone())
    src = torch.zeros(1, 4, 5, 64, dtype=torch.float16)
    with pytest.raises(RuntimeError, match='CUDA device only'):
        fused.kv_quantize(src, cache, sc)
    with pytest.raises(ValueError, match='do not agree'):
        fused.kv_quantize(src, cache, torch.zeros(1, 4, 17))
    with pytest.raises(ValueError, match='do not agree'):
        fused.kv_quantize(torch.zeros(1, 4, 17, 64, dtype=torch.float16), cache, sc)
