"""Logits processors of generation (generate(..., repetition_penalty, no_repeat_ngram_size, min_new_tokens,
bad_words_ids); the rule of include/quip_b200.h's quip_logits_process, restated in torch by decode._process_torch and in
numpy by oracle/logits_process.py) on the CPU: the restatement against HF's own processors, and generation against HF's
generate on the tiny fp32 models of test_generate, one prompt at a time."""
import numpy as np
import pytest
import torch

import quip_b200.decode as D
from oracle.logits_process import process_row
from quip_b200.decode import PromptDecoder, _process_torch, _sample_torch, generate
from test_generate import KINDS, _model, _prompts

EOS = 7


def _hf_processors(pen, n, bad, eos, prompt_len, m):
    from transformers.generation.logits_process import (MinNewTokensLengthLogitsProcessor,
                                                        NoBadWordsLogitsProcessor, NoRepeatNGramLogitsProcessor,
                                                        RepetitionPenaltyLogitsProcessor)
    procs = []
    if pen != 1.0:
        procs.append(RepetitionPenaltyLogitsProcessor(pen))
    if n > 0:
        procs.append(NoRepeatNGramLogitsProcessor(n))
    if bad is not None:
        procs.append(NoBadWordsLogitsProcessor(bad, eos))
    if m > 0 and eos:
        procs.append(MinNewTokensLengthLogitsProcessor(prompt_len, m, eos))
    return procs


def _bits(x):
    return x.contiguous().view(torch.int32) if x.dtype == torch.float32 else x.contiguous().view(torch.int16)


def _same(a, b):
    """Bit for bit, every NaN counted equal to every NaN."""
    a, b = torch.as_tensor(a), torch.as_tensor(b)
    nan = torch.isnan(a) & torch.isnan(b)
    return bool(((_bits(a) == _bits(b)) | nan).all())


def _row(V, g):
    x = torch.randn(V, generator=g) * 3
    x[torch.randint(0, V, (6,), generator=g)] = 0.0
    x[torch.randint(0, V, (6,), generator=g)] = -0.0
    x[torch.randint(0, V, (3,), generator=g)] = float('inf')
    x[torch.randint(0, V, (3,), generator=g)] = float('-inf')
    x[torch.randint(0, V, (3,), generator=g)] = float('nan')
    return x


def _cases():
    """(history, prompt_len, penalty, n, min_new, bad, eos) covering duplicates, n > L, bad words longer than h."""
    g = torch.Generator().manual_seed(0)
    out = []
    for k in range(60):
        L = int(torch.randint(1, 40, (1,), generator=g))
        h = torch.randint(0, 12 if k % 2 else 50, (L,), generator=g).tolist()      # small alphabets repeat n-grams
        plen = int(torch.randint(1, L + 1, (1,), generator=g))
        pen = [1.0, 1.3, 0.7, 2.0][k % 4]
        n = [0, 1, 2, 3, 4, L + 1, L + 3][k % 7]
        m = [0, 3, 50][k % 3]
        bad = [None, [[h[-1]], [EOS], h[-2:] + [5], [3, 4], list(range(45, 45 + 16)), h[-3:] + [9]],
               [[EOS], [h[0]]]][k % 3]
        eos = [[EOS], [EOS, 11], [EOS, 11, 2]][k % 3]
        out.append((h, plen, pen, n, m, bad, eos))
    return out


def _restated(x, h, plen, pen, n, m, bad, eos):
    bad = bad or []
    pad = torch.zeros(len(bad), 16, dtype=torch.long)
    for j, w in enumerate(bad):
        pad[j, :len(w)] = torch.tensor(w)
    y = x.clone()[None]
    _process_torch(y, 1, torch.tensor([h]), torch.tensor([len(h) - 1]), torch.tensor([plen]),
                   torch.tensor([pen], dtype=torch.float32), torch.tensor([n], dtype=torch.int32),
                   torch.tensor([m], dtype=torch.int32), torch.tensor(eos), pad,
                   torch.tensor([len(w) for w in bad], dtype=torch.int32))
    return y[0]


def test_torch_restatement_equals_hf_processors_and_the_oracle():
    g = torch.Generator().manual_seed(1)
    V = 64
    for h, plen, pen, n, m, bad, eos in _cases():
        x = _row(V, g)
        want = x.clone()[None]
        for p in _hf_processors(pen, n, bad, eos, plen, m):
            want = p(torch.tensor([h]), want)
        got = _restated(x, h, plen, pen, n, m, bad, eos)
        assert _same(got, want[0]), (h, pen, n, m, bad)
        assert _same(got, torch.from_numpy(process_row(x.numpy(), h, plen, pen, n, m, eos, bad or [])))


def test_all_off_rows_are_untouched_and_out_of_range_ids_are_skipped():
    g = torch.Generator().manual_seed(2)
    x = _row(32, g)
    assert _same(_restated(x, [1, 2, 1, 2], 1, 1.0, 0, 0, None, [EOS]), x)
    y = _restated(x, [-5, 40, 3], 1, 2.0, 1, 0, None, [EOS])                # 3 penalised, then banned by n = 1
    assert torch.isinf(y[3]) and _same(y[:3], x[:3]) and _same(y[4:], x[4:])


def _hf(m, p, n, eos, **kw):
    with torch.no_grad():
        r = m.generate(p[None], do_sample=False, max_new_tokens=n, eos_token_id=eos, pad_token_id=0, **kw)
    return r[0, p.numel():]


SETTINGS = [dict(repetition_penalty=1.8), dict(no_repeat_ngram_size=2), dict(min_new_tokens=6),
            dict(bad_words_ids=[[EOS], [11], [40, 41], [3, 4, 5]]),
            dict(repetition_penalty=1.5, no_repeat_ngram_size=3, min_new_tokens=4, bad_words_ids=[[9], [20, 21]])]


@pytest.mark.parametrize('kind', KINDS)
def test_greedy_generate_equals_hf_for_each_prompt_alone(kind):
    m = _model(kind)
    prompts = _prompts(seed=3, lens=(5, 11, 2))
    n = 14
    free = generate(m, prompts, n)
    eos = int(free[0][5])                                             # ends row 0 mid-run without processors
    for kw in SETTINGS:
        want = [_hf(m, p, n, eos, **kw) for p in prompts]
        got = generate(m, prompts, n, eos_token_id=eos, **kw)
        for b, (g, w) in enumerate(zip(got, want)):
            assert torch.equal(g, w), (kw, b, g, w)


@pytest.mark.parametrize('chunk', [1, 7, 64])
def test_per_prompt_values_and_prefill_chunks(chunk):
    m = _model('llama_gqa')
    prompts = _prompts(seed=4, lens=(9, 3, 14))
    pens, ngs, mns = [1.0, 2.0, 1.4], [2, 0, 3], [0, 5, 2]
    got = generate(m, prompts, 12, eos_token_id=[EOS, 13], prefill_chunk_size=chunk, repetition_penalty=pens,
                   no_repeat_ngram_size=ngs, min_new_tokens=mns, bad_words_ids=[[13, 14], [30]])
    for b, p in enumerate(prompts):
        w = _hf(m, p, 12, [EOS, 13], repetition_penalty=pens[b], no_repeat_ngram_size=ngs[b], min_new_tokens=mns[b],
                bad_words_ids=[[13, 14], [30]])
        assert torch.equal(got[b], w), (b, got[b], w)


def test_min_new_tokens_delays_an_eos_that_ends_a_row_mid_run():
    m = _model('opt_pre_ln')
    p = _prompts(seed=2)[0]
    free, = generate(m, [p], 20)
    eos = int(free[2])
    early, = generate(m, [p], 20, eos_token_id=eos)
    late, = generate(m, [p], 20, eos_token_id=eos, min_new_tokens=8)
    assert early.numel() <= 3 and (late.numel() == 20 or late.numel() > 8)
    assert torch.equal(late, _hf(m, p, 20, eos, min_new_tokens=8))


def test_sampled_processing_is_reproducible_and_samples_the_processed_logits():
    m = _model('llama_mha')
    prompts = _prompts(seed=5, lens=(6, 4))
    kw = dict(do_sample=True, temperature=0.8, top_k=20, seed=[3, 9], repetition_penalty=1.6, no_repeat_ngram_size=2,
              bad_words_ids=[[5], [8, 9]])
    a, b = generate(m, prompts, 10, **kw), generate(m, prompts, 10, **kw)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    dec = PromptDecoder(m, max_len=20, batch=2, max_new=10, sampling=True, processing=True)
    dec.set_sampling(0.8, 20, 1.0, [3, 9])
    dec.set_processing(1.6, 2, 0, [[5], [8, 9]])
    logits = dec.prefill(prompts)                                      # processed in place before the selection
    steps = [(logits.clone(), 0)]
    for t in range(1, 10):
        steps.append((dec.step().clone(), t))
    for t, (x, s) in enumerate(steps):
        want = _sample_torch(x, dec.temperature, dec.top_k, dec.top_p, dec.seed, s)
        assert torch.equal(dec.generated[:, t], want), t
    assert all(torch.equal(dec.generated[r, :a[r].numel()], a[r]) for r in range(2))


@pytest.mark.parametrize('sample', [False, True])
def test_speculative_runs_equal_plain_runs(sample):
    m = _model('llama_gqa')
    p = torch.tensor([5, 6, 7, 8, 5, 6, 7, 8, 5, 6, 7])                   # repeats: the drafts get accepted
    prompts = [p, _prompts(seed=6)[1]]
    kw = dict(repetition_penalty=1.3, no_repeat_ngram_size=4, min_new_tokens=3, bad_words_ids=[[6, 9]],
              eos_token_id=[EOS])
    if sample:
        kw.update(do_sample=True, temperature=0.9, seed=[1, 2])
    plain = generate(m, prompts, 16, **kw)
    stats = {}
    spec = generate(m, prompts, 16, prompt_lookup_num_tokens=3, spec_stats=stats, **kw)
    assert all(torch.equal(x, y) for x, y in zip(plain, spec)), (plain, spec)


@pytest.mark.parametrize('kv', [None, torch.float8_e4m3fn])
def test_continuous_batching_equals_each_prompt_alone(kv):
    m = _model('opt_post_ln')
    prompts = _prompts(seed=7, lens=(5, 11, 2, 8, 3))
    kw = dict(repetition_penalty=[1.5, 1.0, 2.0, 1.2, 1.0], no_repeat_ngram_size=[2, 3, 0, 1, 2],
              min_new_tokens=[0, 4, 2, 0, 6], bad_words_ids=[[4, 5], [17]], eos_token_id=EOS, kv_dtype=kv,
              prefill_chunk_size=7)
    got = generate(m, prompts, [9, 5, 12, 7, 10], max_batch_size=2, **kw)
    for b, p in enumerate(prompts):
        one = {k: (v[b] if isinstance(v, list) and k != 'bad_words_ids' else v) for k, v in kw.items()}
        want, = generate(m, [p], [9, 5, 12, 7, 10][b], **one)
        assert torch.equal(got[b], want), (b, got[b], want)


def test_return_sequences_and_shared_prefixes():
    m = _model('llama_mha')
    base = _prompts(seed=8, lens=(70,))[0]
    prompts = [base, torch.cat((base[:66], torch.tensor([3, 4])))]
    kw = dict(do_sample=True, seed=5, repetition_penalty=[1.2, 1.9, 1.5, 1.1], no_repeat_ngram_size=2,
              bad_words_ids=[[10]])
    got = generate(m, prompts, 6, num_return_sequences=2, **kw)
    want = generate(m, [p for p in prompts for _ in range(2)], 6, share_prompt_prefixes=True, **kw)
    assert all(torch.equal(x, y) for x, y in zip(got, want))
    kw.pop('do_sample'), kw.pop('seed')
    kw['repetition_penalty'] = [1.2, 1.9]
    shared = generate(m, prompts, 6, share_prompt_prefixes=True, **kw)
    plain = generate(m, prompts, 6, prefill_chunk_size=512, **kw)
    assert all(torch.equal(x, y) for x, y in zip(shared, plain))


def test_e4m3_processing_is_deterministic():
    m = _model('llama_gqa')
    prompts = _prompts(seed=9)
    kw = dict(kv_dtype=torch.float8_e4m3fn, repetition_penalty=1.7, no_repeat_ngram_size=2, bad_words_ids=[[3]],
              prefill_chunk_size=4)
    a, b = generate(m, prompts, 10, **kw), generate(m, prompts, 10, **kw)
    assert all(torch.equal(x, y) for x, y in zip(a, b))


def test_explicit_defaults_take_todays_path(monkeypatch):
    m = _model('llama_mha')
    prompts = _prompts(seed=10)
    made = []

    class Spy(PromptDecoder):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            made.append(self)
    monkeypatch.setattr(D, 'PromptDecoder', Spy)
    want = generate(m, prompts, 8)
    got = generate(m, prompts, 8, repetition_penalty=1.0, no_repeat_ngram_size=0, min_new_tokens=0, bad_words_ids=None)
    assert all(torch.equal(x, y) for x, y in zip(got, want))
    assert len(made) == 2 and not any(d.processing or hasattr(d, 'hist') or hasattr(d, 'penalty') for d in made)


def test_argument_errors_are_raised_before_any_work(monkeypatch):
    def no_decoder(*a, **k):
        raise AssertionError('work started')
    for name in ('PromptDecoder', 'SpecDecoder', 'ContinuousDecoder', 'BeamDecoder'):
        monkeypatch.setattr(D, name, no_decoder)
    m = _model('llama_gqa')
    p = _prompts()
    cases = ((dict(repetition_penalty=0.0), 'repetition_penalty'), (dict(repetition_penalty=float('inf')), 'finite'),
             (dict(repetition_penalty=[1.0, 2.0]), 'repetition_penalty'), (dict(no_repeat_ngram_size=-1), '>= 0'),
             (dict(no_repeat_ngram_size=1.5), 'integer'), (dict(min_new_tokens=True), 'integer'),
             (dict(min_new_tokens=3), 'eos_token_id'), (dict(bad_words_ids=[]), 'non-empty'),
             (dict(bad_words_ids=[[]]), '1 .. 16'), (dict(bad_words_ids=[list(range(17))]), '1 .. 16'),
             (dict(bad_words_ids=[[199]]), r'\[0, 199\)'), (dict(bad_words_ids=[[-1]]), r'\[0, 199\)'),
             (dict(bad_words_ids=[[1]] * 257), 'at most 256'), (dict(bad_words_ids=[3]), 'list of 1'),
             (dict(repetition_penalty=1.2, eos_token_id=list(range(9))), 'at most 8'),
             (dict(no_repeat_ngram_size=2, num_beams=2), 'num_beams'),
             (dict(bad_words_ids=[[3]], num_beams=3), 'num_beams'))
    for kw, msg in cases:
        with pytest.raises(ValueError, match=msg):
            generate(m, p, 5, **kw)
    with pytest.raises(ValueError, match='processing=True'):
        PromptDecoder(m, max_len=8, batch=1, max_new=2).set_processing(1.5)
    with pytest.raises(ValueError, match='max_new'):
        PromptDecoder(m, max_len=8, batch=1, processing=True)


def test_logits_process_wrapper_checks_and_refuses_cpu_tensors():
    from quip_b200 import fused
    B, V = 2, 50
    z = lambda *s, dt=torch.long: torch.zeros(s, dtype=dt)
    args = dict(hist=z(B, 8), last=z(B), prompt_len=z(B), penalty=z(B, dt=torch.float32), ngram=z(B, dt=torch.int32),
                min_new=z(B, dt=torch.int32), eos=z(1), bad=z(1, 16), bad_len=z(1, dt=torch.int32))
    x = torch.zeros(B, V, dtype=torch.float16)
    with pytest.raises(RuntimeError, match='CUDA device only'):
        fused.logits_process(x, 1, **args)
    with pytest.raises(ValueError, match='fp16'):
        fused.logits_process(x.float(), 1, **args)
    with pytest.raises(ValueError, match='penalty'):
        fused.logits_process(x, 1, **{**args, 'penalty': z(B)})
    with pytest.raises(ValueError, match='at most 8'):
        fused.logits_process(x, 1, **{**args, 'eos': z(9)})
    with pytest.raises(ValueError, match='bad'):
        fused.logits_process(x, 1, **{**args, 'bad': z(1, 8)})
    with pytest.raises(ValueError, match='drafts'):
        fused.logits_process(x, 2, **args)
    with pytest.raises(ValueError, match='pass rows'):
        fused.logits_process(torch.zeros(3, V, dtype=torch.float16), 1, **args)


def test_quip_logits_process_argument_errors_surface_as_messages():
    from quip_b200 import _lib
    lib = _lib.load()
    buf = 64

    def call(R=2, T=1, V=50, ld=50, n_eos=1, n_bad=1, logits=buf, hist=buf, tokens=None):
        return lib.quip_logits_process(logits, ld, R, T, V, None, hist, buf, tokens, buf, buf, buf, buf, buf, n_eos,
                                       buf, buf, n_bad, 2, 8, None)
    assert call(V=2 ** 18 + 1, ld=2 ** 18 + 1) == 1 and b'V' in lib.quip_last_error()
    assert call(ld=10) == 1 and b'ld' in lib.quip_last_error()
    assert call(R=3, T=2) == 1
    assert call(n_eos=9) == 1 and b'at most' in lib.quip_last_error()
    assert call(n_bad=257) == 1 and b'at most' in lib.quip_last_error()
    assert call(hist=None) == 1 and b'null' in lib.quip_last_error()
    assert call(T=2, R=2) == 1 and b'null' in lib.quip_last_error()               # drafts needed at T > 1
    assert call(logits=65) == 1 and b'aligned' in lib.quip_last_error()
    assert call(R=0) == 0                                                         # no rows: nothing to launch


def test_oracle_agrees_on_fp16_rows():
    g = np.random.default_rng(3)
    x = (g.standard_normal(40) * 4).astype(np.float16)
    x[[1, 2]] = [np.float16(-0.0), np.float16(np.inf)]
    y = process_row(x, [1, 2, 3, 1, 2], 2, 1.7, 0, 0, [EOS], [[2]])
    assert y.dtype == np.float16 and np.isnan(y[2]) and y[1] == 0 and not np.signbit(y[1])
    f = np.float32(x[3])
    assert y[3] == np.float16(f * np.float32(1.7) if f < 0 else f / np.float32(1.7))
