"""Generation from prompts (quip_b200/decode.py: PromptDecoder, generate) on tiny fp32 HF models on the CPU, where the
step's attention is the torch restatement of csrc/attn_decode.cu (per-row scatter, SDPA under arange <= positions)."""
import pytest
import torch

from oracle.glue import TorchGlue
from quip_b200 import _lib
from quip_b200.decode import PromptDecoder, generate

KINDS = ['llama_mha', 'llama_gqa', 'opt_pre_ln', 'opt_post_ln']


def _model(kind):
    torch.manual_seed(0)
    if kind.startswith('opt'):
        from transformers import OPTConfig, OPTForCausalLM
        pre = kind == 'opt_pre_ln'
        cfg = OPTConfig(hidden_size=64, ffn_dim=128, num_hidden_layers=2, num_attention_heads=4, vocab_size=199,
                        max_position_embeddings=40, word_embed_proj_dim=64 if pre else 48, do_layer_norm_before=pre)
        return OPTForCausalLM(cfg).float().eval()
    from transformers import LlamaConfig, LlamaForCausalLM
    cfg = LlamaConfig(hidden_size=128, intermediate_size=352, num_hidden_layers=2, num_attention_heads=4,
                      num_key_value_heads=4 if kind == 'llama_mha' else 2, vocab_size=199, max_position_embeddings=64)
    return LlamaForCausalLM(cfg).float().eval()


def _prompts(seed=1, lens=(5, 11, 2)):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(3, 199, (n,), generator=g) for n in lens]


def _hf_greedy(m, p, n, eos=None):
    with torch.no_grad():
        r = m.generate(p[None], do_sample=False, max_new_tokens=n, eos_token_id=eos, pad_token_id=0)
    return r[0, p.numel():]


@pytest.mark.parametrize('kind', KINDS)
def test_generate_matches_hf_greedy_alone_and_in_a_ragged_batch(kind):
    m = _model(kind)
    prompts = _prompts()
    n = 14
    want = [_hf_greedy(m, p, n) for p in prompts]
    for p, w in zip(prompts, want):
        got, = generate(m, [p], n)
        assert torch.equal(got, w), (p.numel(), got, w)
    batched = generate(m, prompts, n)
    for b, (g, w) in enumerate(zip(batched, want)):
        assert torch.equal(g, w), (b, g, w)


@pytest.mark.parametrize('kind', ['llama_gqa', 'opt_pre_ln'])
def test_generate_cuts_after_the_first_eos(kind):
    m = _model(kind)
    prompts = _prompts(seed=2)
    n = 40 - max(p.numel() for p in prompts)                          # runs past the first EOS check (step 16)
    free = [_hf_greedy(m, p, n) for p in prompts]
    eos = int(free[0][3])                                             # a token row 0 produces: it must stop there
    got = generate(m, prompts, n, eos_token_id=[eos])
    for p, g in zip(prompts, got):
        w = _hf_greedy(m, p, n, eos=eos)
        assert torch.equal(g, w), (g, w)
    assert got[0].numel() <= 4 and int(got[0][-1]) == eos


@pytest.mark.parametrize('kind', KINDS)
def test_prefill_leaves_hf_keys_and_values_in_every_real_slot(kind):
    m = _model(kind)
    prompts = _prompts(seed=3, lens=(7, 3, 10))
    dec = PromptDecoder(m, max_len=24, batch=3)
    logits = dec.prefill(prompts)
    assert dec.positions.tolist() == [7, 3, 10]
    for b, p in enumerate(prompts):
        with torch.no_grad():
            out = m(p[None], use_cache=True)
        L = p.numel()
        for li in range(len(dec.layers)):
            torch.testing.assert_close(dec.k_cache[li, b, :, :L], out.past_key_values.layers[li].keys[0], rtol=1e-5, atol=1e-5)
            torch.testing.assert_close(dec.v_cache[li, b, :, :L], out.past_key_values.layers[li].values[0], rtol=1e-5, atol=1e-5)
        torch.testing.assert_close(logits[b], out.logits[0, -1], rtol=1e-4, atol=1e-4)


@pytest.mark.parametrize('nkv', [4, 2])
def test_prompt_decoder_steps_with_the_glue_ops_equal_hf_decode(nkv):
    """The fused-glue layer path (torch restatement of the glue kernels injected) with per-row positions."""
    m = _model('llama_mha' if nkv == 4 else 'llama_gqa')
    prompts = _prompts(seed=4, lens=(3, 8))
    ids = torch.randint(3, 199, (2, 6), generator=torch.Generator().manual_seed(5))
    dec = PromptDecoder(m, max_len=16, batch=2, ops=TorchGlue())
    dec.prefill(prompts)
    got = [dec.step(ids[:, i]).clone() for i in range(ids.shape[1])]
    for b, p in enumerate(prompts):
        with torch.no_grad():
            out = m(torch.cat((p, ids[b]))[None])
        want = out.logits[0, p.numel():]
        for i in range(ids.shape[1]):
            torch.testing.assert_close(got[i][b], want[i], rtol=2e-4, atol=2e-4)


def test_uniform_positions_agree_with_graph_decoder():
    from quip_b200.decode import GraphDecoder
    m = _model('llama_gqa')
    ids = torch.randint(3, 199, (3, 8), generator=torch.Generator().manual_seed(6))
    g, p = GraphDecoder(m, max_len=12, batch=3), PromptDecoder(m, max_len=12, batch=3)
    with torch.no_grad():
        for i in range(ids.shape[1]):
            torch.testing.assert_close(p.step(ids[:, i]), g.step(ids[:, i]), rtol=1e-5, atol=1e-5)


def test_generate_rejects_bad_requests_before_any_work():
    m = _model('llama_mha')
    p = _prompts()[0]
    with pytest.raises(ValueError, match='exceeds max_len'):
        generate(m, [p], 10, max_len=p.numel() + 9)
    with pytest.raises(ValueError, match='empty prompt'):
        generate(m, [p, torch.zeros(0, dtype=torch.long)], 4)
    with pytest.raises(ValueError, match='learned positions'):
        generate(_model('opt_pre_ln'), [p], 40)                       # 5 + 40 positions, the table has 40
    generate(_model('opt_pre_ln'), [p], 35)                           # exactly the table
    dec = PromptDecoder(m, max_len=8, batch=1, max_new=3)
    dec.prefill([p])
    dec.step()
    dec.step()
    with pytest.raises(ValueError, match='generated already'):
        dec.step()


def test_decode_attention_descriptor_argument_errors_surface_as_messages():
    lib = _lib.load()
    buf, ws = 64, 1 << 20

    def call(B=2, nh=8, nkv=2, hd=128, max_len=256, q=buf, pos=buf, wsb=ws, out=buf):
        kv = _lib.QuipKvCache(k=buf, v=buf, format=_lib.QUIP_KV_FP16, nkv=nkv, hd=hd, max_len=max_len)
        return lib.quip_decode_attention(kv, q, buf, buf, pos, out, B, nh, 1.0, buf, wsb, None)
    assert call(hd=96) == 1 and b'head_dim 96' in lib.quip_last_error()
    assert call(nh=6, nkv=4) == 1 and b'nh % nkv' in lib.quip_last_error()
    assert call(nh=32, nkv=2) == 1 and b'at most 8' in lib.quip_last_error()
    assert call(q=None) == 1 and b'null' in lib.quip_last_error()
    assert call(pos=None) == 1 and b'null' in lib.quip_last_error()
    assert call(out=68) == 1 and b'aligned' in lib.quip_last_error()
    assert call(wsb=100) == 1 and b'workspace' in lib.quip_last_error()
    with pytest.raises(_lib.QuipError, match='head_dim'):
        _lib.check(call(hd=32))
    import ctypes as C
    need = C.c_size_t(0)
    assert lib.quip_decode_attention_workspace_bytes(2, 8, 128, 256, C.byref(need)) == 0 and need.value > 0
    assert call(wsb=need.value - 1) == 1 and b'workspace' in lib.quip_last_error()
    assert lib.quip_decode_attention_workspace_bytes(2, 8, 80, 256, C.byref(need)) == 1
    assert call(B=0, wsb=0) == 0                                      # no rows: nothing to launch


def test_decode_attention_wrapper_refuses_cpu_tensors():
    from quip_b200 import fused
    q = torch.zeros(1, 4, 64, dtype=torch.float16)
    kv = torch.zeros(1, 4, 64, dtype=torch.float16)
    cache = torch.zeros(1, 4, 16, 64, dtype=torch.float16)
    with pytest.raises(RuntimeError, match='CUDA device only'):
        fused.decode_attention(q, kv, kv, cache, cache.clone(), torch.zeros(1, dtype=torch.long), 0.125)


def test_generate_one_token_is_the_prefill_argmax():
    m = _model('llama_gqa')
    prompts = _prompts()
    got = generate(m, prompts, 1)
    for p, g in zip(prompts, got):
        assert torch.equal(g, _hf_greedy(m, p, 1))


def _warm_up_keeps_state(dec):
    state = dec._capture_state()
    saved = [t.clone() for t in state]
    dec._warm_up(state, saved)                                        # capture()'s eager warm-up steps
    for t, t0 in zip(state, saved):
        assert torch.equal(t, t0)


@pytest.mark.parametrize('kind', ['llama_gqa', 'opt_pre_ln'])
def test_capture_warm_up_stays_in_range_from_any_state(kind):
    """The warm-up steps capture() runs index the rotary / position tables at the step's positions and the generated
    buffer at the step counter: from a fresh decoder with max_new = 1, after prefill (counter at max_new), and with a row's
    cache full, every index stays in range and the state is put back."""
    m = _model(kind)
    dec = PromptDecoder(m, max_len=6, batch=2, max_new=1)
    _warm_up_keeps_state(dec)
    dec.prefill(_prompts(seed=5, lens=(6, 2)))                        # row 0 at max_len, the counter at max_new
    _warm_up_keeps_state(dec)
    from quip_b200.decode import GraphDecoder
    g = GraphDecoder(m, max_len=4)
    ids = torch.randint(3, 199, (4,), generator=torch.Generator().manual_seed(2))
    with torch.no_grad():
        for i in range(3):
            g.step(ids[i:i + 1])
        _warm_up_keeps_state(g)                                       # position max_len - 1
        g.step(ids[3:])
        _warm_up_keeps_state(g)                                       # position max_len: the cache is full


def test_reset_starts_the_prompt_decoder_over():
    m = _model('llama_mha')
    prompts = _prompts(seed=6, lens=(4, 7))
    dec = PromptDecoder(m, max_len=12, batch=2, max_new=5)
    dec.prefill(_prompts(seed=7, lens=(3, 9)))
    for _ in range(3):
        dec.step()
    dec.reset()
    assert dec.positions.tolist() == [0, 0] and int(dec._t) == 0 and not dec.generated.any()
    fresh = PromptDecoder(m, max_len=12, batch=2, max_new=5)
    for d in (dec, fresh):
        d.prefill(prompts)
        for _ in range(4):
            d.step()
    assert torch.equal(dec.generated, fresh.generated)
    torch.testing.assert_close(dec.logits, fresh.logits, rtol=1e-6, atol=1e-6)
