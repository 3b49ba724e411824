"""Log-probabilities of generation (generate(..., logprobs={}, top_logprobs=n); the rule of include/quip_b200.h's
quip_token_topk_logprobs, restated in torch by decode._token_topk_logprobs_torch and in numpy by
oracle/topk_logprobs.py) on the CPU: the raw distribution against HF's output_logits and teacher forcing, against
score, across every generation path, on the tiny fp32 models of test_generate."""
import numpy as np
import pytest
import torch

import quip_b200.decode as D
from oracle.topk_logprobs import topk_row
from quip_b200 import fused
from quip_b200.decode import _token_topk_logprobs_torch, generate, score
from test_generate import KINDS, _model, _prompts

EOS = 7
TOL = 1e-5


def _hf_out(m, p, n, **kw):
    with torch.no_grad():
        r = m.generate(p[None], do_sample=False, max_new_tokens=n, pad_token_id=0, output_logits=True,
                       return_dict_in_generate=True, **kw)
    return r.sequences[0, p.numel():], torch.stack(r.logits)[:, 0].float()


def _teacher(m, p, o):
    """log_softmax of the HF forward over prompt + output, at the positions that predict o: (len(o), vocab)."""
    with torch.no_grad():
        x = m(torch.cat((p, o))[None]).logits[0, p.numel() - 1:p.numel() - 1 + o.numel()].float()
    return torch.log_softmax(x, -1)


def _close(a, b, tol=TOL):
    return a.shape == b.shape and float((a.double() - b.double()).abs().max()) <= tol


def _far_from_ties(x, n):
    """The n + 1 largest values of each row of x (len, vocab) are pairwise apart."""
    top = torch.topk(x, min(n + 1, x.shape[-1]), -1).values
    return bool(((top[:, :-1] - top[:, 1:]) > 1e-4).all())


@pytest.mark.parametrize('kind', KINDS)
def test_greedy_logprobs_equal_hf_output_logits(kind):
    m = _model(kind)
    prompts = _prompts(seed=3, lens=(5, 11, 2))
    free = generate(m, prompts, 14)
    eos = int(free[0][5])                                            # ends row 0 mid-run
    budgets = [14, 9, 12]
    for kw in (dict(), dict(repetition_penalty=1.6, bad_words_ids=[[11], [40, 41]])):
        lp = {}
        got = generate(m, prompts, budgets, eos_token_id=eos, logprobs=lp, top_logprobs=4, **kw)
        for b, p in enumerate(prompts):
            seq, logits = _hf_out(m, p, budgets[b], eos_token_id=eos, **kw)
            assert torch.equal(got[b], seq), (kw, b)
            ls = torch.log_softmax(logits, -1)                       # HF's output_logits: before its processors
            assert _close(lp['token'][b], ls.gather(-1, seq[:, None])[:, 0]), (kw, b)
            if _far_from_ties(logits, 4):
                want = torch.sort(logits, dim=-1, descending=True, stable=True).indices[:, :4]
                assert torch.equal(lp['top_ids'][b], want), (kw, b)
                assert _close(lp['top'][b], ls.gather(-1, want))
        if not kw:
            assert got[0].numel() <= 6 and int(got[0][-1]) == eos


def test_each_prompt_alone_equals_the_batch():
    m = _model('llama_gqa')
    prompts = _prompts(seed=4, lens=(9, 3, 14))
    lp = {}
    generate(m, prompts, 10, logprobs=lp, top_logprobs=3)
    for b, p in enumerate(prompts):
        one = {}
        generate(m, [p], 10, logprobs=one, top_logprobs=3)
        assert _close(lp['token'][b], one['token'][0]) and torch.equal(lp['top_ids'][b], one['top_ids'][0])


def test_greedy_rows_rank_their_token_first_bit_for_bit():
    m = _model('opt_pre_ln')
    prompts = _prompts(seed=5)
    lp = {}
    out = generate(m, prompts, 12, logprobs=lp, top_logprobs=5)
    for b, o in enumerate(out):
        assert torch.equal(lp['top_ids'][b][:, 0], o)
        assert torch.equal(lp['top'][b][:, 0].view(torch.int32), lp['token'][b].view(torch.int32))
        assert lp['top_ids'][b].dtype == torch.int64 and lp['top'][b].dtype == torch.float32
        assert lp['top'][b].shape == (o.numel(), 5) and lp['token'][b].shape == (o.numel(),)
        assert bool((lp['top'][b][:, :-1] >= lp['top'][b][:, 1:]).all())


@pytest.mark.parametrize('mode', ['sampled', 'spec', 'spec_sampled'])
def test_sampled_and_speculative_logprobs_equal_teacher_forcing(mode):
    m = _model('llama_mha')
    p0 = torch.tensor([5, 6, 7, 8, 5, 6, 7, 8, 5, 6, 7])               # repeats: the drafts get accepted
    prompts = [p0, _prompts(seed=6)[1]]
    kw = dict(eos_token_id=[EOS])
    if mode != 'spec':
        kw.update(do_sample=True, temperature=0.7, top_k=30, seed=[1, 2])
    if mode != 'sampled':
        kw.update(prompt_lookup_num_tokens=3)
    lp = {}
    out = generate(m, prompts, 16, logprobs=lp, top_logprobs=2, **kw)
    for b, (p, o) in enumerate(zip(prompts, out)):
        ls = _teacher(m, p, o)
        assert _close(lp['token'][b], ls.gather(-1, o[:, None])[:, 0]), (mode, b)
        assert _close(lp['top'][b], ls.gather(-1, lp['top_ids'][b]))
    again = {}
    out2 = generate(m, prompts, 16, logprobs=again, top_logprobs=2, **kw)
    assert all(torch.equal(x, y) for x, y in zip(out, out2))
    assert all(torch.equal(x, y) for x, y in zip(lp['token'], again['token']))


@pytest.mark.parametrize('kw', [dict(), dict(repetition_penalty=1.3, bad_words_ids=[[6, 9]]),
                                dict(do_sample=True, temperature=0.3, seed=[1, 2])])
def test_speculative_logprobs_equal_plain_logprobs(kw):
    m = _model('llama_mha')
    p = torch.tensor([5, 6, 7, 8, 5, 6, 7, 8, 5, 6, 7])
    prompts = [p, _prompts(seed=6)[1]]
    kw = dict(kw, eos_token_id=[EOS])
    plain, spec = {}, {}
    a = generate(m, prompts, [16, 11], logprobs=plain, top_logprobs=3, **kw)
    stats = {}
    b = generate(m, prompts, [16, 11], prompt_lookup_num_tokens=3, spec_stats=stats, logprobs=spec, top_logprobs=3,
                 **kw)
    assert sum(stats['accepted']) > 0 or kw.get('repetition_penalty') or kw.get('do_sample')
    for r, (x, y) in enumerate(zip(a, b)):
        k = min(x.numel(), y.numel())
        if kw.get('do_sample'):       # a sampled token near a draw boundary may follow the other step's rounding
            k = int((x[:k] != y[:k]).long().cumsum(0).eq(0).sum())
            assert k >= 1
        else:
            assert torch.equal(x, y)
        assert _close(plain['token'][r][:k], spec['token'][r][:k])
        assert torch.equal(plain['top_ids'][r][:k], spec['top_ids'][r][:k])


def test_sums_equal_score():
    m = _model('llama_gqa')
    prompts = _prompts(seed=7, lens=(6, 10, 3))
    lp = {}
    out = generate(m, prompts, 9, logprobs=lp)
    assert set(lp) == {'token'}
    got = score(m, [p.tolist() for p in prompts], [o.tolist() for o in out])
    for b, (s, greedy) in enumerate(got):
        assert abs(float(lp['token'][b].double().sum()) - s) <= 1e-4 and greedy


@pytest.mark.parametrize('kv', [None, torch.float8_e4m3fn])
def test_continuous_batching_equals_each_prompt_alone(kv):
    m = _model('opt_post_ln')
    prompts = _prompts(seed=7, lens=(5, 11, 2, 8, 3))
    budgets = [9, 5, 12, 7, 10]
    kw = dict(eos_token_id=EOS, kv_dtype=kv, prefill_chunk_size=7, repetition_penalty=[1.5, 1.0, 2.0, 1.2, 1.0])
    lp = {}
    got = generate(m, prompts, budgets, max_batch_size=2, logprobs=lp, top_logprobs=3, **kw)
    for b, p in enumerate(prompts):
        one, alone = {}, {k: (v[b] if isinstance(v, list) else v) for k, v in kw.items()}
        want, = generate(m, [p], budgets[b], logprobs=one, top_logprobs=3, **alone)
        assert torch.equal(got[b], want)
        assert _close(lp['token'][b], one['token'][0]) and torch.equal(lp['top_ids'][b], one['top_ids'][0])
        assert lp['token'][b].shape == (want.numel(),)


def test_return_sequences_and_shared_prefixes():
    m = _model('llama_mha')
    base = _prompts(seed=8, lens=(70,))[0]
    prompts = [base, torch.cat((base[:66], torch.tensor([3, 4])))]
    kw = dict(do_sample=True, seed=5, top_p=0.9)
    a, b = {}, {}
    got = generate(m, prompts, [6, 4, 5, 6], num_return_sequences=2, logprobs=a, top_logprobs=2, **kw)
    want = generate(m, [p for p in prompts for _ in range(2)], [6, 4, 5, 6], share_prompt_prefixes=True, logprobs=b,
                    top_logprobs=2, **kw)
    assert all(torch.equal(x, y) for x, y in zip(got, want))
    assert all(torch.equal(x, y) for x, y in zip(a['token'], b['token']))
    shared, plain = {}, {}
    generate(m, prompts, 6, share_prompt_prefixes=True, logprobs=shared)
    generate(m, prompts, 6, prefill_chunk_size=512, logprobs=plain)
    for x, y in zip(shared['token'], plain['token']):
        assert _close(x, y)


@pytest.mark.parametrize('chunk', [1, 7, 64])
def test_prefill_chunks(chunk):
    m = _model('llama_gqa')
    prompts = _prompts(seed=9, lens=(9, 3, 14))
    ref, lp = {}, {}
    want = generate(m, prompts, 8, logprobs=ref, top_logprobs=2)
    got = generate(m, prompts, 8, prefill_chunk_size=chunk, logprobs=lp, top_logprobs=2)
    assert all(torch.equal(x, y) for x, y in zip(got, want))
    for x, y in zip(lp['token'], ref['token']):
        assert _close(x, y)


def test_e4m3_runs_are_deterministic_and_equal_score():
    m = _model('llama_gqa')
    prompts = _prompts(seed=10)
    e4 = torch.float8_e4m3fn
    a, b = {}, {}
    out = generate(m, prompts, 10, kv_dtype=e4, prefill_chunk_size=4, logprobs=a, top_logprobs=3)
    generate(m, prompts, 10, kv_dtype=e4, prefill_chunk_size=4, logprobs=b, top_logprobs=3)
    assert all(torch.equal(x, y) for x, y in zip(a['token'], b['token']))
    assert all(torch.equal(x, y) for x, y in zip(a['top_ids'], b['top_ids']))
    got = score(m, [p.tolist() for p in prompts], [o.tolist() for o in out], kv_dtype=e4, prefill_chunk_size=4,
                share_prompt_prefixes=False)
    for b, (s, _) in enumerate(got):
        assert abs(float(a['token'][b].double().sum()) - s) <= 1e-4


@pytest.mark.parametrize('kw', [dict(), dict(do_sample=True, seed=3, temperature=1.3), dict(prompt_lookup_num_tokens=2),
                                dict(no_repeat_ngram_size=2, min_new_tokens=4, eos_token_id=EOS),
                                dict(max_batch_size=2, eos_token_id=EOS)])
def test_tokens_are_unchanged(kw):
    m = _model('llama_mha')
    prompts = _prompts(seed=11, lens=(4, 9, 6))
    off = generate(m, prompts, 12, **kw)
    on = generate(m, prompts, 12, logprobs={}, top_logprobs=20, **kw)
    assert all(torch.equal(x, y) for x, y in zip(off, on))


def test_the_default_call_launches_and_allocates_nothing(monkeypatch):
    def refuse(*a, **k):
        raise AssertionError('logprobs ran')
    monkeypatch.setattr(fused, 'token_topk_logprobs', refuse)
    monkeypatch.setattr(D, '_token_topk_logprobs_torch', refuse)
    made = []
    for name in ('PromptDecoder', 'SpecDecoder', 'ContinuousDecoder'):
        base = getattr(D, name)
        spy = type(name, (base,), {'__init__': lambda self, *a, _b=base, **k: (_b.__init__(self, *a, **k),
                                                                                 made.append(self))[0]})
        monkeypatch.setattr(D, name, spy)
    m = _model('llama_gqa')
    prompts = _prompts(seed=12)
    for kw in (dict(), dict(prompt_lookup_num_tokens=2), dict(max_batch_size=2), dict(repetition_penalty=1.4)):
        generate(m, prompts, 6, **kw)
        generate(m, prompts, 6, logprobs=None, top_logprobs=0, **kw)
    assert made and all(d.lp is None and d.top_ids is None and d.top_lp is None for d in made)


def test_argument_errors_are_raised_before_any_work(monkeypatch):
    def no_decoder(*a, **k):
        raise AssertionError('work started')
    for name in ('PromptDecoder', 'SpecDecoder', 'ContinuousDecoder', 'BeamDecoder'):
        monkeypatch.setattr(D, name, no_decoder)
    m = _model('llama_gqa')
    p = _prompts()
    cases = ((dict(top_logprobs=-1, logprobs={}), 'top_logprobs'), (dict(top_logprobs=21, logprobs={}), 'top_logprobs'),
             (dict(top_logprobs=2.0, logprobs={}), 'top_logprobs'), (dict(top_logprobs=True, logprobs={}), 'top_logprobs'),
             (dict(top_logprobs='3', logprobs={}), 'top_logprobs'), (dict(top_logprobs=3), 'logprobs dict'),
             (dict(logprobs=[]), 'dict'), (dict(logprobs=True), 'dict'),
             (dict(logprobs={}, num_beams=2), 'num_beams'), (dict(logprobs={}, top_logprobs=3, num_beams=4), 'num_beams'))
    for kw, msg in cases:
        with pytest.raises(ValueError, match=msg):
            generate(m, p, 5, **kw)


def test_decoder_and_wrapper_checks():
    m = _model('llama_mha')
    with pytest.raises(ValueError, match='logprobs'):
        D.PromptDecoder(m, max_len=8, batch=1, max_new=2, logprobs=21)
    with pytest.raises(ValueError, match='max_new'):
        D.PromptDecoder(m, max_len=8, batch=1, logprobs=0)
    B, V, G = 2, 50, 4
    x = torch.zeros(B, V, dtype=torch.float16)
    args = dict(tokens=torch.zeros(B, dtype=torch.long), cols=torch.zeros(1, dtype=torch.long),
                lp=torch.zeros(B, G), top_ids=torch.zeros(B, G, 3, dtype=torch.long), top_lp=torch.zeros(B, G, 3))
    with pytest.raises(RuntimeError, match='CUDA device only'):
        fused.token_topk_logprobs(x, **args)
    with pytest.raises(ValueError, match='fp16'):
        fused.token_topk_logprobs(x.float(), **args)
    with pytest.raises(ValueError, match='together'):
        fused.token_topk_logprobs(x, **{**args, 'top_lp': None})
    with pytest.raises(ValueError, match='n <= 20'):
        fused.token_topk_logprobs(x, **{**args, 'top_ids': torch.zeros(B, G, 21, dtype=torch.long),
                                        'top_lp': torch.zeros(B, G, 21)})
    with pytest.raises(ValueError, match='cols'):
        fused.token_topk_logprobs(x, **{**args, 'cols': torch.zeros(3, dtype=torch.long)})
    with pytest.raises(ValueError, match='T must'):
        fused.token_topk_logprobs(x, T=9, **args)
    with pytest.raises(ValueError, match='pass rows'):
        fused.token_topk_logprobs(torch.zeros(3, V, dtype=torch.float16), **{**args, 'tokens': torch.zeros(3).long()})
    with pytest.raises(ValueError, match='top_lp'):
        fused.token_topk_logprobs(x, **{**args, 'top_lp': torch.zeros(B, G, 3, dtype=torch.float16)})


def test_quip_token_topk_logprobs_argument_errors_surface_as_messages():
    from quip_b200 import _lib
    lib = _lib.load()
    buf = 64

    def call(R=2, T=1, V=50, ld=50, n=3, per_row=1, logits=buf, tokens=buf, top=buf):
        return lib.quip_token_topk_logprobs(logits, ld, R, T, V, None, tokens, buf, per_row, buf, top, top, n, 2, 4,
                                            None)
    assert call(V=2 ** 24 + 1, ld=2 ** 24 + 1) == 1 and b'V' in lib.quip_last_error()
    assert call(ld=10) == 1 and b'ld' in lib.quip_last_error()
    assert call(R=3, T=2) == 1 and call(R=9, T=9) == 1
    assert call(n=21) == 1 and call(per_row=2) == 1
    assert call(tokens=None) == 1 and b'null' in lib.quip_last_error()
    assert call(top=None) == 1 and b'null' in lib.quip_last_error()
    assert call(logits=65) == 1 and b'aligned' in lib.quip_last_error()
    assert call(R=0) == 0 and call(R=0, n=0, top=None) == 0


def _rows16(V, R, seed):
    """fp16 rows with ties (planted and natural), +-0, +-inf and a NaN row."""
    g = np.random.default_rng(seed)
    x = np.round(g.standard_normal((R, V)) * 4, 1).astype(np.float16)     # coarse values: many ties
    x[0, :5] = np.array([-0.0, 0.0, -0.0, 0.0, -0.0], dtype=np.float16)[:V]
    x[0, 5:] = -np.inf
    x[1, [3 % V, 9 % V, 17 % V]] = np.inf
    x[2, :] = 1.5
    x[3, 7 % V] = np.nan
    x[4, ::3] = -np.inf
    return x


@pytest.mark.parametrize('V', [1, 7, 50, 300])
def test_oracle_agrees_with_the_restatement(V):
    R, n = 6, 20
    x = _rows16(V, R, seed=V)
    tokens = torch.tensor([0, 3 % V, V - 1, 0, -1, V], dtype=torch.long)
    lp = torch.zeros(R, 1)
    ids, top = torch.zeros(R, 1, n, dtype=torch.long), torch.zeros(R, 1, n)
    _token_topk_logprobs_torch(torch.from_numpy(x), tokens, torch.zeros(1, dtype=torch.long), lp, ids, top)
    for r in range(R):
        want_ids, want = topk_row(x[r], n)
        assert np.array_equal(ids[r, 0].numpy(), want_ids), r
        assert np.allclose(top[r, 0].numpy(), want, atol=1e-5, equal_nan=True), r
    assert bool(torch.isnan(lp[3:]).all()) and not bool(torch.isnan(lp[[0, 2]]).any())    # row 1 holds +inf: NaN too
    k = min(n, V)
    assert bool((ids[:, 0, k:] == -1).all()) and bool(torch.isnan(top[:, 0, k:]).all())
    assert bool((ids[3] == -1).all())


def test_restatement_addressing_and_column_guards():
    V, B, G = 30, 4, 5
    g = torch.Generator().manual_seed(1)
    x = torch.randn(6, V, generator=g)
    tokens = torch.randint(0, V, (6,), generator=g)
    lp = torch.full((B, G), 7.0)
    ids, top = torch.full((B, G, 2), 9, dtype=torch.long), torch.full((B, G, 2), 7.0)
    rows = torch.tensor([2, 0, -1])                                   # T = 2: logits rows 4, 5 belong to no row
    cols = torch.tensor([3, 0, 4, 1])                                 # row 2 at 4, 5: 5 is past the buffers
    _token_topk_logprobs_torch(x, tokens, cols, lp, ids, top, T=2, rows=rows)
    ls = torch.log_softmax(x, -1)
    assert lp[2, 4] == ls[0, tokens[0]] and lp[0, 3] == ls[2, tokens[2]] and lp[0, 4] == ls[3, tokens[3]]
    written = {(2, 4), (0, 3), (0, 4)}
    for b in range(B):
        for c in range(G):
            if (b, c) not in written:
                assert lp[b, c] == 7.0 and bool((ids[b, c] == 9).all())
