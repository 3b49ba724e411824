"""Speculative generation on the CPU (quip_b200/decode.py: SpecDecoder, generate(prompt_lookup_num_tokens=...)): the
torch restatements of drafting and acceptance against oracle/speculative.py, speculative generation against plain
generation and HF greedy on the tiny fp32 models of test_generate.py, and the argument checks of the new C ABI."""
import functools

import numpy as np
import pytest
import torch

from oracle import speculative as oracle
from quip_b200 import _lib
from quip_b200.decode import SpecDecoder, _ngram_draft_torch, _spec_accept_torch, generate

KINDS = ['llama_mha', 'llama_gqa', 'opt_pre_ln', 'opt_post_ln']


def _model(kind):
    from test_generate import _model as model
    return model(kind)


def _draft(hist, pos, k, n_max, n_min=1):
    want = oracle.ngram_draft(np.array(hist), np.array(pos), k, n_min, n_max)
    got = _ngram_draft_torch(torch.tensor(hist), torch.tensor(pos), k, n_min, n_max)
    assert np.array_equal(got.numpy(), want)
    return want.tolist()


def test_draft_rule_on_named_cases():
    assert _draft([[1, 2, 3, 4]], [3], 3, 3) == [[4, 4, 4, 4]]                      # no match: the current token
    assert _draft([[5, 6, 7, 5]], [3], 4, 3) == [[5, 6, 7, 5, 6]]                   # match at position 0, then overlap
    assert _draft([[9, 9, 0, 0]], [1], 3, 3) == [[9, 9, 9, 9]]                      # continuation runs into the current token
    assert _draft([[1, 2, 1, 2, 1, 0]], [4], 5, 3) == [[1, 2, 1, 2, 1, 2]]          # period 2 < k
    assert _draft([[1, 2, 1, 2, 1, 0]], [4], 5, 1) == [[1, 2, 1, 2, 1, 2]]          # latest single-token match
    assert _draft([[1, 4, 2, 5, 4, 6, 1, 4]], [7], 2, 2) == [[4, 2, 5]]             # longest (1 4) beats the latest (4)
    assert _draft([[1, 4, 2, 5, 4, 6, 1, 4]], [7], 2, 1) == [[4, 6, 1]]             # n_max 1: the latest (4)
    assert _draft([[1, 4, 2, 5, 4, 6, 1, 4]], [7], 2, 2, n_min=3) == [[4, 4, 4]]    # shorter than n_min: no match
    assert _draft([[7, 8]], [0], 2, 3) == [[7, 7, 7]]                               # nothing before the current token
    assert _draft([[7, 8]], [2], 2, 3) == [[0, 0, 0]]                               # outside the history


@pytest.mark.parametrize('k,n_max', [(1, 1), (4, 3), (7, 2), (7, 6)])
def test_draft_torch_equals_the_oracle_on_random_histories(k, n_max):
    g = np.random.default_rng(k * 10 + n_max)
    for vocab in (2, 5, 50):
        hist = g.integers(0, vocab, (12, 40))
        hist[::3, :] = np.tile(g.integers(0, vocab, 3), 14)[:40]       # periodic rows
        pos = g.integers(0, 40, 12)
        pos[0] = 0
        _draft(hist.tolist(), pos.tolist(), k, n_max)


def test_accept_torch_equals_the_oracle():
    g = np.random.default_rng(3)
    B, T, max_new, max_len = 30, 5, 8, 30
    for trial in range(6):
        tokens = g.integers(0, 3, (B, T))
        targets = g.integers(0, 3, (B, T))
        targets[::4, :-1] = tokens[::4, 1:]                            # every draft right
        n_gen = g.integers(0, max_new + 2, B)                          # finished rows and max_new clamps
        positions = g.integers(0, max_len - 1, B)
        positions[-1] = max_len - 2                                    # history writes clipped at max_len
        state = [g.integers(0, 3, (B, max_new)), g.integers(0, 3, (B, max_len)), positions, n_gen, g.integers(0, 4, B)]
        want = [x.copy() for x in state]
        oracle.spec_accept(tokens, targets, *want, max_new)
        got = [torch.tensor(x) for x in state]
        _spec_accept_torch(torch.tensor(tokens), torch.tensor(targets), *got, max_new)
        for a, w in zip(got, want):
            assert np.array_equal(a.numpy(), w), trial
    # a finished row is left alone; a row one short takes exactly one token
    st = [np.zeros((2, 4), np.int64), np.zeros((2, 9), np.int64), np.array([3, 5]), np.array([4, 3]), np.zeros(2, np.int64)]
    oracle.spec_accept(np.array([[1, 2, 3], [1, 2, 3]]), np.array([[2, 3, 9], [2, 3, 9]]), *st, 4)
    assert st[2].tolist() == [3, 6] and st[3].tolist() == [4, 4] and st[4].tolist() == [0, 0] and st[0][1, 3] == 2


def _quoting_prompts(m, lens=(10, 14, 9), c=8, **kw):
    """Prompts that quote the model's own continuation, as a summary or a RAG answer quotes its source: the last c tokens
    of each prompt are replaced by what generate(m, prompt, c, **kw) continues it with, twice over.  The continuation of
    the result then largely repeats what it quotes, so prompt lookup finds drafts the model accepts on every kind,
    including the post-LN OPT, whose random-weight continuation follows the position far more than the tokens and has
    no cycles of its own within its 40 positions."""
    from test_generate import _prompts
    base = _prompts(seed=1, lens=lens)
    q = base
    for _ in range(2):
        q = [torch.cat((p[:p.numel() - c], y)) for p, y in zip(base, generate(m, q, c, **kw))]
    return q


@functools.lru_cache(maxsize=None)
def _plain(kind, n, kv_dtype=None):
    m = _model(kind)
    prompts = _quoting_prompts(m, kv_dtype=kv_dtype)
    return m, prompts, generate(m, prompts, n, kv_dtype=kv_dtype)


@pytest.mark.parametrize('n_max', [1, 3])
@pytest.mark.parametrize('k', [1, 3, 7])
@pytest.mark.parametrize('kind', KINDS)
def test_speculative_greedy_equals_plain_and_hf_greedy(kind, k, n_max):
    from test_generate import _hf_greedy
    m, prompts, plain = _plain(kind, 14)
    stats = {}
    got = generate(m, prompts, 14, prompt_lookup_num_tokens=k, max_matching_ngram_size=n_max, spec_stats=stats)
    assert sum(stats['accepted']) > 0
    for p, g, w in zip(prompts, got, plain):
        assert torch.equal(g, w), (g, w)
    if k == 3 and n_max == 3:
        for p, g in zip(prompts, got):
            assert torch.equal(g, _hf_greedy(m, p, 14))


@pytest.mark.parametrize('kind', ['llama_gqa', 'opt_pre_ln'])
def test_speculative_generation_cuts_after_the_first_eos(kind):
    from test_generate import _hf_greedy, _prompts
    m = _model(kind)
    prompts = _prompts(seed=2)
    n = 40 - max(p.numel() for p in prompts) - 4
    free = [_hf_greedy(m, p, n) for p in prompts]
    eos = int(free[0][3])
    stats = {}
    got = generate(m, prompts, n, eos_token_id=[eos], prompt_lookup_num_tokens=4, spec_stats=stats)
    assert sum(stats['accepted']) > 0
    for p, g in zip(prompts, got):
        assert torch.equal(g, _hf_greedy(m, p, n, eos=eos))
    assert got[0].numel() <= 4 and int(got[0][-1]) == eos


@pytest.mark.parametrize('kind', KINDS)
def test_speculative_sampling_equals_plain_sampling(kind):
    m = _model(kind)
    kw = dict(do_sample=True, temperature=0.5, top_k=3, top_p=0.9, seed=[11, 12, 13])
    prompts = _quoting_prompts(m, **kw)
    plain = generate(m, prompts, 20, **kw)
    for k in (2, 5):
        stats = {}
        got = generate(m, prompts, 20, prompt_lookup_num_tokens=k, spec_stats=stats, **kw)
        assert sum(stats['accepted']) > 0
        for g, w in zip(got, plain):
            assert torch.equal(g, w), (k, g, w)


@pytest.mark.parametrize('kind', ['llama_gqa', 'opt_post_ln'])
def test_speculative_e4m3_cache_equals_plain_e4m3_generation(kind):
    m, prompts, plain = _plain(kind, 14, kv_dtype=torch.float8_e4m3fn)
    for k in (1, 4):
        stats = {}
        got = generate(m, prompts, 14, kv_dtype=torch.float8_e4m3fn, prompt_lookup_num_tokens=k, spec_stats=stats)
        assert sum(stats['accepted']) > 0
        for g, w in zip(got, plain):
            assert torch.equal(g, w)


def test_spec_decoder_state_reset_warm_up_and_guards():
    from test_generate import _prompts, _warm_up_keeps_state
    m = _model('llama_gqa')
    prompts = _prompts(seed=6, lens=(4, 7))
    dec = SpecDecoder(m, max_len=20, batch=2, max_new=6, draft_tokens=3)
    _warm_up_keeps_state(dec)
    dec.prefill(prompts)
    assert dec.hist[0, :4].tolist() == prompts[0].tolist() and int(dec.hist[0, 4]) == int(dec.generated[0, 0])
    assert dec.n_gen.tolist() == [1, 1]
    _warm_up_keeps_state(dec)
    for _ in range(5):
        dec.step()
    assert dec.n_gen.tolist() == [6, 6]
    with pytest.raises(ValueError, match='generated already'):
        dec.step()
    _warm_up_keeps_state(dec)
    gen = dec.generated.clone()
    dec.reset()
    assert not dec.hist.any() and not dec.n_gen.any() and not dec.accepted.any() and not dec.positions.any()
    dec.prefill(prompts)
    for _ in range(5):
        dec.step()
    assert torch.equal(dec.generated, gen)
    with pytest.raises(ValueError, match='exceed the cache'):
        dec.prefill(_prompts(seed=6, lens=(12, 3)))                   # 12 + 6 + 3 > 20
    with pytest.raises(ValueError, match='draft_tokens'):
        SpecDecoder(m, max_len=20, batch=1, max_new=4, draft_tokens=8)


def test_generate_rejects_bad_speculation_settings():
    from test_generate import _prompts
    m = _model('llama_mha')
    p = _prompts()[0]
    for k in (0, 8, 2.5):
        with pytest.raises(ValueError, match='prompt_lookup_num_tokens'):
            generate(m, [p], 4, prompt_lookup_num_tokens=k)
    with pytest.raises(ValueError, match='max_matching_ngram_size'):
        generate(m, [p], 4, prompt_lookup_num_tokens=2, max_matching_ngram_size=0)
    with pytest.raises(ValueError, match='drafts exceeds max_len'):
        generate(m, [p], 10, max_len=p.numel() + 12, prompt_lookup_num_tokens=3)
    with pytest.raises(ValueError, match='learned positions'):
        generate(_model('opt_pre_ln'), [p], 33, prompt_lookup_num_tokens=3)   # 5 + 33 + 3 positions, the table has 40
    generate(_model('opt_pre_ln'), [p], 32, prompt_lookup_num_tokens=3)       # exactly the table


def test_spec_abi_argument_errors_surface_as_messages():
    import ctypes as C
    lib = _lib.load()
    buf, ws = 64, 1 << 20

    def ext(B=2, T=4, nh=8, nkv=2, hd=128, max_len=256, q=buf, wsb=ws, out=buf, fmt=_lib.QUIP_KV_FP16, ks=None):
        kv = _lib.QuipKvCache(k=buf, v=buf, k_scale=ks, v_scale=buf if ks else None, format=fmt, nkv=nkv, hd=hd,
                              max_len=max_len)
        return lib.quip_extend_attention(kv, q, buf, buf, buf, out, B, T, nh, 1.0, buf, wsb, None)
    assert ext(hd=96) == 1 and b'head_dim 96' in lib.quip_last_error()
    assert ext(T=9) == 1 and b'1 <= T <= 8' in lib.quip_last_error()
    assert ext(T=0) == 1 and b'1 <= T <= 8' in lib.quip_last_error()
    assert ext(nh=32, nkv=2) == 1 and b'at most 8' in lib.quip_last_error()
    assert ext(q=None) == 1 and b'null' in lib.quip_last_error()
    assert ext(out=68) == 1 and b'aligned' in lib.quip_last_error()
    need = C.c_size_t(0)
    assert lib.quip_extend_attention_workspace_bytes(2, 4, 8, 128, 256, C.byref(need)) == 0 and need.value > 0
    assert ext(wsb=need.value - 1) == 1 and b'workspace' in lib.quip_last_error()
    assert lib.quip_extend_attention_workspace_bytes(2, 9, 8, 128, 256, C.byref(need)) == 1
    assert ext(B=0, wsb=0) == 0
    assert ext(fmt=_lib.QUIP_KV_E4M3) == 1 and b'null' in lib.quip_last_error()
    assert lib.quip_ngram_draft(buf, buf, buf, 2, 16, 3, 0, 3, None) == 1 and b'n_min' in lib.quip_last_error()
    assert lib.quip_ngram_draft(None, buf, buf, 2, 16, 3, 1, 3, None) == 1 and b'null' in lib.quip_last_error()
    assert lib.quip_spec_accept(buf, buf, buf, buf, buf, buf, buf, 2, 4, 9, 8, 32, None) == 1
    assert b'max_new <= gen_cols' in lib.quip_last_error()
    assert lib.quip_sample_at(buf, buf, buf, buf, buf, buf, buf, 2, 0, 100, None) == 1 and b'T >= 1' in lib.quip_last_error()
    with pytest.raises(_lib.QuipError, match='T <= 8'):
        _lib.check(ext(T=12))


def test_new_wrappers_refuse_cpu_tensors():
    from quip_b200 import fused
    q = torch.zeros(1, 2, 4, 64, dtype=torch.float16)
    kv = torch.zeros(1, 2, 4, 64, dtype=torch.float16)
    cache = torch.zeros(1, 4, 16, 64, dtype=torch.float16)
    with pytest.raises(RuntimeError, match='CUDA device only'):
        fused.extend_attention(q, kv, kv, cache, cache.clone(), torch.zeros(1, dtype=torch.long), 0.125)
    h = torch.zeros(1, 8, dtype=torch.long)
    with pytest.raises(RuntimeError, match='CUDA device only'):
        fused.ngram_draft(h, torch.zeros(1, dtype=torch.long), torch.zeros(1, 3, dtype=torch.long), 1, 3)
