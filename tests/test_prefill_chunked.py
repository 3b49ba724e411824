"""Chunked prefill (PromptDecoder.prefill(chunk=C), generate(prefill_chunk_size=C)) on the tiny fp32 HF models of
test_generate on the CPU, where the chunk's attention is the torch restatement of csrc/attn_prefill.cu (per-row scatter
of the counted slots, SDPA under the causal mask)."""
import pytest
import torch

from oracle.glue import TorchGlue
from quip_b200 import _lib
from quip_b200.decode import PromptDecoder, SpecDecoder, generate
from test_generate import KINDS, _model, _prompts

SENTINEL = 7.25
LENS = (5, 11, 2)


def _hf_prompt(m, p):
    with torch.no_grad():
        return m(p[None], use_cache=True)


@pytest.mark.parametrize('C', [1, 3, 4, 16, 11])
@pytest.mark.parametrize('kind,glue', [(k, False) for k in KINDS] + [('llama_mha', True), ('llama_gqa', True)])
def test_chunked_prefill_leaves_hf_keys_values_and_logits_and_writes_nothing_past_a_prompt(kind, glue, C):
    """C = 11 is the longest prompt: one chunk.  glue: the Llama layer loop with the glue ops (torch restatement)."""
    m = _model(kind)
    prompts = _prompts(seed=3, lens=LENS)
    dec = PromptDecoder(m, max_len=20, batch=3, ops=TorchGlue() if glue else None)
    dec.k_cache.fill_(SENTINEL)
    dec.v_cache.fill_(SENTINEL)
    logits = dec.prefill(prompts, chunk=C)
    assert dec.positions.tolist() == list(LENS) and dec._pos_host == list(LENS)
    for b, p in enumerate(prompts):
        out = _hf_prompt(m, p)
        n = p.numel()
        for li in range(len(dec.layers)):
            kv = out.past_key_values.layers[li]
            torch.testing.assert_close(dec.k_cache[li, b, :, :n], kv.keys[0], rtol=1e-5, atol=1e-5)
            torch.testing.assert_close(dec.v_cache[li, b, :, :n], kv.values[0], rtol=1e-5, atol=1e-5)
            assert (dec.k_cache[li, b, :, n:] == SENTINEL).all() and (dec.v_cache[li, b, :, n:] == SENTINEL).all()
        torch.testing.assert_close(logits[b], out.logits[0, -1], rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize('kind', ['llama_gqa', 'opt_post_ln'])
def test_chunked_prefill_never_runs_the_hf_forward(kind, monkeypatch):
    m = _model(kind)
    prompts = _prompts(seed=4, lens=LENS)
    want = PromptDecoder(m, max_len=16, batch=3).prefill(prompts)

    def boom(*a, **k):
        raise AssertionError('the HF forward ran')
    monkeypatch.setattr(m.model, 'forward', boom)
    got = PromptDecoder(m, max_len=16, batch=3).prefill(prompts, chunk=4)
    torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-4)
    with pytest.raises(AssertionError, match='HF forward'):
        PromptDecoder(m, max_len=16, batch=3).prefill(prompts)


@pytest.mark.parametrize('kind', KINDS)
def test_generate_with_chunked_prefill_equals_generate(kind):
    m = _model(kind)
    prompts = _prompts(seed=5, lens=LENS)
    n = 12
    want = generate(m, prompts, n)
    for C in (1, 4, 64):
        got = generate(m, prompts, n, prefill_chunk_size=C)
        assert all(torch.equal(g, w) for g, w in zip(got, want)), C


@pytest.mark.parametrize('kind', ['llama_gqa', 'opt_pre_ln'])
def test_generate_with_chunked_prefill_equals_generate_with_eos_sampling_and_lookup(kind):
    m = _model(kind)
    prompts = _prompts(seed=2, lens=LENS)
    n = 40 - max(LENS) - 7
    free = generate(m, prompts, n)
    eos = int(free[0][3])
    for kw in (dict(eos_token_id=[eos]),
               dict(do_sample=True, seed=[11, 12, 13], top_k=20, temperature=0.9),
               dict(prompt_lookup_num_tokens=3),
               dict(prompt_lookup_num_tokens=2, do_sample=True, seed=[1, 2, 3], top_p=0.9)):
        want = generate(m, prompts, n, **kw)
        got = generate(m, prompts, n, prefill_chunk_size=3, **kw)
        assert all(torch.equal(g, w) for g, w in zip(got, want)), kw


def test_spec_decoder_chunked_prefill_keeps_the_history():
    m = _model('llama_mha')
    prompts = _prompts(seed=6, lens=LENS)
    a = SpecDecoder(m, max_len=24, batch=3, max_new=4, draft_tokens=2)
    b = SpecDecoder(m, max_len=24, batch=3, max_new=4, draft_tokens=2)
    a.prefill(prompts)
    b.prefill(prompts, chunk=4)
    for name in ('hist', 'n_gen', 'positions', 'generated', '_t'):
        assert torch.equal(getattr(a, name), getattr(b, name)), name


@pytest.mark.parametrize('kind', ['llama_mha', 'llama_gqa', 'opt_pre_ln'])
def test_e4m3_chunked_prefill_equals_teacher_forced_e4m3_decode(kind):
    """With an e4m3 cache a chunk attends over the quantized keys and values of the cache, its own included: what T = 1
    steps fed the prompt token by token compute.  The chunk's linears run at another row count, so an fp32 value may
    land on the other side of an e4m3 rounding boundary: nearly every byte equal, logits close."""
    m = _model(kind)
    prompts = _prompts(seed=8, lens=LENS)
    e4 = torch.float8_e4m3fn
    dec = PromptDecoder(m, max_len=16, batch=3, kv_dtype=e4)
    logits = dec.prefill(prompts, chunk=4)
    same = total = 0
    for b, p in enumerate(prompts):
        one = PromptDecoder(m, max_len=16, batch=1, kv_dtype=e4)
        with torch.no_grad():
            for t in p:
                want = one.step(t.reshape(1))
        n = p.numel()
        eq = dec.k_cache[:, b, :, :n].view(torch.uint8) == one.k_cache[:, 0, :, :n].view(torch.uint8)
        eq = torch.cat((eq.flatten(), (dec.v_cache[:, b, :, :n].view(torch.uint8) ==
                                       one.v_cache[:, 0, :, :n].view(torch.uint8)).flatten()))
        same, total = same + int(eq.sum()), total + eq.numel()
        torch.testing.assert_close(dec.k_scale[:, b, :, :n], one.k_scale[:, 0, :, :n], rtol=1e-5, atol=0)
        torch.testing.assert_close(dec.v_scale[:, b, :, :n], one.v_scale[:, 0, :, :n], rtol=1e-5, atol=0)
        torch.testing.assert_close(logits[b], want[0], rtol=2e-3, atol=2e-3)
    assert same >= 0.999 * total, (same, total)


def test_chunk_size_is_checked_before_any_work():
    m = _model('llama_mha')
    p = _prompts()[0]
    for bad in (0, -2, 2.5, True, '4', [4]):
        with pytest.raises(ValueError, match='chunk size'):
            generate(m, [p], 3, prefill_chunk_size=bad)
        with pytest.raises(ValueError, match='chunk size'):
            PromptDecoder(m, max_len=8, batch=1).prefill([p], chunk=bad)


def test_prefill_attention_and_append_argument_errors_surface_as_messages():
    lib = _lib.load()
    buf = 64

    def attn(fp8=False, B=2, T=4, nh=8, nkv=2, hd=128, max_len=256, q=buf, cnt=buf, ks=buf):
        if fp8:
            return lib.quip_prefill_attention_fp8(q, buf, buf, ks, buf, buf, cnt, buf, B, T, nh, nkv, hd, max_len, 1.0,
                                                  None)
        return lib.quip_prefill_attention(q, buf, buf, buf, cnt, buf, B, T, nh, nkv, hd, max_len, 1.0, None)

    def append(fp8=False, B=2, T=4, nkv=2, hd=128, max_len=256, kn=buf, cnt=buf, vs=buf):
        if fp8:
            return lib.quip_kv_append_fp8(kn, buf, buf, buf, buf, vs, buf, cnt, B, T, nkv, hd, max_len, None)
        return lib.quip_kv_append(kn, buf, buf, buf, buf, cnt, B, T, nkv, hd, max_len, None)
    for fp8 in (False, True):
        name = b'quip_prefill_attention' + (b'_fp8' if fp8 else b'')
        assert attn(fp8, hd=96) == 1 and b'head_dim 96' in lib.quip_last_error()
        assert name in lib.quip_last_error()
        assert attn(fp8, nh=32, nkv=2) == 1 and b'at most 8' in lib.quip_last_error()
        assert attn(fp8, nh=6, nkv=4) == 1 and b'nh % nkv' in lib.quip_last_error()
        assert attn(fp8, T=0) == 1 and b'tokens per row' in lib.quip_last_error()
        assert attn(fp8, T=257) == 1 and b'tokens per row' in lib.quip_last_error()
        assert attn(fp8, q=None) == 1 and b'null' in lib.quip_last_error()
        assert attn(fp8, cnt=None) == 1 and b'null' in lib.quip_last_error()
        assert attn(fp8, q=68) == 1 and b'aligned' in lib.quip_last_error()
        assert attn(fp8, B=0) == 0                                    # no rows: nothing to launch
        name = b'quip_kv_append' + (b'_fp8' if fp8 else b'')
        assert append(fp8, hd=96) == 1 and b'head_dim 96' in lib.quip_last_error()
        assert name in lib.quip_last_error()
        assert append(fp8, T=0) == 1 and b'tokens per row' in lib.quip_last_error()
        assert append(fp8, kn=None) == 1 and b'null' in lib.quip_last_error()
        assert append(fp8, cnt=None) == 1 and b'null' in lib.quip_last_error()
        assert append(fp8, B=0) == 0
    assert attn(True, ks=None) == 1 and b'null' in lib.quip_last_error()
    assert append(True, vs=None) == 1 and b'null' in lib.quip_last_error()
    with pytest.raises(_lib.QuipError, match='head_dim'):
        _lib.check(attn(hd=32))


def test_chunk_wrappers_refuse_cpu_tensors():
    from quip_b200 import fused
    q = torch.zeros(1, 3, 4, 64, dtype=torch.float16)
    kv = torch.zeros(1, 3, 4, 64, dtype=torch.float16)
    cache = torch.zeros(1, 4, 16, 64, dtype=torch.float16)
    pos, cnt = torch.zeros(1, dtype=torch.long), torch.full((1,), 3, dtype=torch.long)
    with pytest.raises(RuntimeError, match='CUDA device only'):
        fused.kv_append(kv, kv, cache, cache.clone(), pos, cnt)
    with pytest.raises(RuntimeError, match='CUDA device only'):
        fused.prefill_attention(q, cache, cache.clone(), pos, cnt, 0.125)
    with pytest.raises(ValueError, match='int64 positions and counts'):
        fused.prefill_attention(q, cache, cache.clone(), pos, cnt.int(), 0.125)
    with pytest.raises(ValueError, match='do not agree'):
        fused.kv_append(kv, kv, cache, cache.clone(), pos, torch.zeros(2, dtype=torch.long))
