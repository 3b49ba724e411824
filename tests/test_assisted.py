"""Assisted generation on the CPU (quip_b200/decode.py: AssistedDecoder, generate(assistant_model=...)): the decoder's
rounds against the cache-free loop of oracle/assisted.py fed the models' full forwards, and assisted generation against
plain generation with every option it combines with, on the tiny fp32 models of test_generate.py."""
import copy
import functools

import numpy as np
import pytest
import torch

from oracle.assisted import assisted_generate
from quip_b200.constrain import TokenAutomaton
from quip_b200.decode import AssistedDecoder, _sample_torch, generate

KINDS = ['llama_mha', 'llama_gqa', 'opt_pre_ln', 'opt_post_ln']
ASSISTS = ['self', 'noisy', 'other']


def _model(kind):
    from test_generate import _model as model
    return model(kind)


def _prompts(**kw):
    from test_generate import _prompts as prompts
    return prompts(**kw)


@functools.lru_cache(maxsize=None)
def _pair(kind, assist):
    """(target, assistant): the target itself, a copy whose lm_head (untied from OPT's embedding) has noise added, or
    an unrelated tiny model of the other family with the same vocabulary.  The noise is sized so that the copy's drafts
    are often all right and often not: the pre-LN OPT's continuation mostly repeats its input, which small noise does
    not move."""
    m = _model(kind)
    if assist == 'self':
        return m, m
    if assist == 'noisy':
        a = copy.deepcopy(m)
        g = torch.Generator().manual_seed(1)
        w = a.lm_head.weight.detach()
        a.lm_head = torch.nn.Linear(w.shape[1], w.shape[0], bias=False)
        with torch.no_grad():
            a.lm_head.weight.copy_(w + torch.randn(w.shape, generator=g) * float(w.std()) *
                                   (0.5 if kind == 'opt_pre_ln' else 0.1))
        return m, a
    return m, _model('llama_mha' if kind.startswith('opt') else 'opt_pre_ln')


def _close(a, b):
    from test_gen_logprobs import _close as close
    return close(a, b)


def _full(m):
    def fn(seq):
        with torch.no_grad():
            return m(torch.tensor(seq)[None]).logits[0].numpy()
    return fn


def _greedy(z, t):
    return int(np.argmax(z))


def _run(m, a, prompts, n, k, sampling=None):
    """AssistedDecoder's tokens and, per row, the drafts accepted in each round the row was live."""
    dec = AssistedDecoder(m, a, max_len=max(p.numel() for p in prompts) + n + k, batch=len(prompts), max_new=n,
                          draft_tokens=k, sampling=sampling is not None)
    if sampling is not None:
        dec.set_sampling(*sampling)
    rounds = [[] for _ in prompts]
    with torch.no_grad():
        dec.prefill(prompts)
        for _ in range(n - 1):
            g0, a0 = dec.n_gen.clone(), dec.accepted.clone()
            dec.step()
            for b in range(len(prompts)):
                if int(g0[b]) < n:
                    rounds[b].append(int(dec.accepted[b] - a0[b]))
    return dec, rounds


@pytest.mark.parametrize('assist', ASSISTS)
@pytest.mark.parametrize('k', [1, 3, 7])
@pytest.mark.parametrize('kind', KINDS)
def test_assisted_decoder_equals_the_cache_free_oracle(kind, k, assist):
    m, a = _pair(kind, assist)
    prompts, n = _prompts(), 14
    dec, rounds = _run(m, a, prompts, n, k)
    for b, p in enumerate(prompts):
        want, want_rounds = assisted_generate(_full(m), _full(a), p.tolist(), n, k, _greedy)
        assert dec.generated[b].tolist() == want, (b, dec.generated[b].tolist(), want)
        assert rounds[b] == want_rounds, (b, rounds[b], want_rounds)
    if assist == 'self':                           # every draft is the target's own choice: all accepted, budget allowing
        for b in range(len(prompts)):
            g, full = 1, []
            for _ in rounds[b]:
                full.append(min(k, n - g - 1))
                g += full[-1] + 1
            assert rounds[b] == full, (b, rounds[b], full)
    if assist == 'noisy' and k > 1:               # both full and partial rounds (not cut by the budget)
        flat = [r for rs in rounds for r in rs[:-1]]
        assert k in flat and any(r < k for r in flat), rounds


@pytest.mark.parametrize('kind', ['llama_gqa', 'opt_post_ln'])
def test_sampled_assisted_decoder_equals_the_cache_free_oracle(kind):
    m, a = _pair(kind, 'noisy')
    prompts, n, k = _prompts(), 14, 3
    temp, top_k, top_p, seeds = [0.8, 1.2, 0.5], [0, 5, 20], [0.9, 1.0, 0.8], [7, 8, 9]
    dec, rounds = _run(m, a, prompts, n, k, sampling=(temp, top_k, top_p, seeds))
    for b, p in enumerate(prompts):
        t_b, k_b, p_b, s_b = (torch.tensor([x[b]]) for x in (temp, top_k, top_p, seeds))

        def select(z, t):
            return int(_sample_torch(torch.from_numpy(z)[None], t_b, k_b, p_b, s_b, t)[0])
        want, want_rounds = assisted_generate(_full(m), _full(a), p.tolist(), n, k, select)
        assert dec.generated[b].tolist() == want and rounds[b] == want_rounds, b
    assert sum(map(sum, rounds)) > 0


@pytest.mark.parametrize('assist', ASSISTS)
@pytest.mark.parametrize('kind', KINDS)
def test_assisted_greedy_equals_plain_and_hf_greedy(kind, assist):
    from test_generate import _hf_greedy
    m, a = _pair(kind, assist)
    prompts = _prompts()
    plain = generate(m, prompts, 14)
    for k in (1, 4):
        stats = {}
        got = generate(m, prompts, 14, assistant_model=a, num_assistant_tokens=k, spec_stats=stats)
        assert all(torch.equal(g, w) for g, w in zip(got, plain)), (k, got, plain)
        assert stats['steps'] == 13 and len(stats['accepted']) == len(prompts)
        if assist == 'self':
            assert min(stats['accepted']) > 0
    for p, w in zip(prompts, plain):
        assert torch.equal(w, _hf_greedy(m, p, 14))


@pytest.mark.parametrize('assist', ASSISTS)
@pytest.mark.parametrize('kind', ['llama_mha', 'opt_pre_ln'])
def test_assisted_sampling_equals_plain_sampling(kind, assist):
    m, a = _pair(kind, assist)
    prompts = _prompts()
    kw = dict(do_sample=True, temperature=0.7, top_k=20, top_p=0.9, seed=[11, 12, 13])
    plain = generate(m, prompts, 16, **kw)
    for k in (2, 5):
        got = generate(m, prompts, 16, assistant_model=a, num_assistant_tokens=k, **kw)
        assert all(torch.equal(g, w) for g, w in zip(got, plain)), (k, got, plain)


@pytest.mark.parametrize('assist', ASSISTS)
@pytest.mark.parametrize('kind', ['llama_gqa', 'opt_post_ln'])
def test_assisted_e4m3_and_chunked_prefill_equal_plain(kind, assist):
    m, a = _pair(kind, assist)
    prompts = _prompts(seed=3, lens=(7, 3, 10))
    for kw in (dict(kv_dtype=torch.float8_e4m3fn), dict(prefill_chunk_size=4),
               dict(kv_dtype=torch.float8_e4m3fn, prefill_chunk_size=3)):
        plain = generate(m, prompts, 12, **kw)
        got = generate(m, prompts, 12, assistant_model=a, num_assistant_tokens=3, **kw)
        assert all(torch.equal(g, w) for g, w in zip(got, plain)), kw


@pytest.mark.parametrize('assist', ASSISTS)
def test_assisted_shared_prefixes_and_return_sequences_equal_plain(assist):
    m, a = _pair('llama_mha', assist) if assist != 'other' else (_model('llama_mha'), _model('llama_gqa'))   # 70 + slots
    base = _prompts(seed=8, lens=(70,))[0]
    prompts = [base, torch.cat((base[:66], torch.tensor([3, 4])))]
    kw = dict(do_sample=True, seed=5, top_k=10)
    want = generate(m, prompts, 6, num_return_sequences=2, **kw)
    got = generate(m, prompts, 6, num_return_sequences=2, assistant_model=a, num_assistant_tokens=2, **kw)
    assert all(torch.equal(x, y) for x, y in zip(got, want))
    plain = generate(m, prompts, 8, prefill_chunk_size=512)
    for ch in (None, 16):
        shared = generate(m, prompts, 8, share_prompt_prefixes=True, prefill_chunk_size=ch, assistant_model=a,
                          num_assistant_tokens=3)
        assert all(torch.equal(x, y) for x, y in zip(shared, plain))


@pytest.mark.parametrize('sample', [False, True])
@pytest.mark.parametrize('assist', ASSISTS)
def test_assisted_processors_constraint_eos_budgets_and_logprobs_equal_plain(assist, sample):
    m, a = _pair('llama_gqa', assist)
    prompts = [torch.tensor([5, 6, 7, 8, 5, 6, 7, 8, 5, 6, 9])] + _prompts(seed=6)[1:]
    loop = TokenAutomaton({0: {5: 1, 6: 0, 9: 0}, 1: {6: 2, 7: 0}, 2: {7: 3, 8: 3}, 3: {8: 0, 5: 1}}, 0)
    plain0 = generate(m, prompts, 16)
    eos = int(plain0[1][5])                                           # greedy row 1 stops early
    kw = dict(token_constraint=[loop, None, None], eos_token_id=eos, repetition_penalty=1.2, no_repeat_ngram_size=3,
              bad_words_ids=[[int(plain0[2][2])]], min_new_tokens=[0, 2, 3])
    if sample:
        kw.update(do_sample=True, temperature=0.9, seed=[1, 2, 3])
    budgets = [16, 12, 9]
    lp_plain, lp_got = {}, {}
    plain = generate(m, prompts, budgets, logprobs=lp_plain, top_logprobs=3, **kw)
    got = generate(m, prompts, budgets, assistant_model=a, num_assistant_tokens=3, logprobs=lp_got, top_logprobs=3,
                   **kw)
    assert all(torch.equal(x, y) for x, y in zip(got, plain)), (got, plain)
    assert sample or got[1].numel() < budgets[1] and int(got[1][-1]) == eos
    assert all(g.numel() <= n for g, n in zip(got, budgets))
    for key in ('token', 'top_ids', 'top'):         # logprobs: the verify step's logits round otherwise than plain ones
        for x, y in zip(lp_got[key], lp_plain[key]):
            assert torch.equal(x, y) if key == 'top_ids' else _close(x, y), key


def test_assisted_decoder_warm_up_keeps_state_and_reset_clears_the_assistant():
    from test_generate import _warm_up_keeps_state
    m, a = _pair('llama_gqa', 'noisy')
    prompts = _prompts(seed=6, lens=(4, 7))
    dec = AssistedDecoder(m, a, max_len=20, batch=2, max_new=6, draft_tokens=3)
    assert dec.assistant.model is a and dec.assistant.max_len == 20
    _warm_up_keeps_state(dec)
    dec.prefill(prompts)
    assert dec.assistant.positions.tolist() == [4, 7] and dec.n_gen.tolist() == [1, 1]
    _warm_up_keeps_state(dec)
    for _ in range(5):
        dec.step()
    _warm_up_keeps_state(dec)
    gen = dec.generated.clone()
    dec.reset()
    ast = dec.assistant
    assert not ast.positions.any() and not ast.k_cache.any() and not ast.v_cache.any()
    assert not dec.hist.any() and not dec.n_gen.any() and not dec.accepted.any()
    dec.prefill(prompts)
    for _ in range(5):
        dec.step()
    assert torch.equal(dec.generated, gen)
    fp8 = AssistedDecoder(m, a, max_len=20, batch=2, max_new=6, draft_tokens=3, kv_dtype=torch.float8_e4m3fn)
    fp8.prefill(prompts)
    assert fp8.assistant.kv_dtype == torch.float8_e4m3fn and fp8.assistant.k_scale.any()
    _warm_up_keeps_state(fp8)
    fp8.reset()
    assert not fp8.assistant.k_scale.any() and not fp8.assistant.positions.any()


def test_generate_rejects_bad_assistant_settings_before_any_work(monkeypatch):
    from quip_b200 import decode
    m, a = _pair('llama_mha', 'noisy')
    p = _prompts()[0]
    opt = _model('opt_pre_ln')
    wide = copy.deepcopy(a)
    wide.lm_head = torch.nn.Linear(wide.lm_head.in_features, 200, bias=False)
    meta = copy.deepcopy(a).to('meta')

    def no_work(*args, **kw):
        raise AssertionError('a decoder was built')
    monkeypatch.setattr(decode.GraphDecoder, '__init__', no_work)
    cases = [(dict(num_assistant_tokens=3), 'needs assistant_model'),
             (dict(assistant_model=a, prompt_lookup_num_tokens=3), 'prompt_lookup_num_tokens'),
             (dict(assistant_model=a, num_beams=2), 'num_beams'),
             (dict(assistant_model=a, max_batch_size=2), 'max_batch_size'),
             (dict(assistant_model=torch.nn.Linear(2, 2)), 'Llama or OPT'),
             (dict(assistant_model=wide), 'vocabulary'),
             (dict(assistant_model=meta), 'same device|is on'),
             (dict(assistant_model=opt), 'learned positions of the assistant'),
             (dict(assistant_model=a, max_len=p.numel() + 10 + 3), 'drafts exceeds max_len')]
    for k in (0, 8, 2.5, True):
        cases.append((dict(assistant_model=a, num_assistant_tokens=k), r'num_assistant_tokens must be'))
    for kw, msg in cases:
        with pytest.raises(ValueError, match=msg):
            generate(m, [p], 10 if 'max_len' in kw else 36, **kw)
    with pytest.raises(ValueError, match='vocabulary'):
        AssistedDecoder(m, wide, max_len=20)
