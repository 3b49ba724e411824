"""Constrained generation by token automata (generate(..., token_constraint=...); the rule of include/quip_b200.h's
quip_constrain_mask / quip_constrain_advance, restated in torch by decode._constrain_torch / _constrain_advance_torch
and in numpy by oracle/constrain.py) on the CPU: the restatement against HF's PrefixConstrainedLogitsProcessor, and
generation against HF's generate(prefix_allowed_tokens_fn=...) on the tiny fp32 models of test_generate, one prompt at
a time."""
import numpy as np
import pytest
import torch

import quip_b200.decode as D
from oracle import constrain as O
from quip_b200.constrain import TokenAutomaton, pack_automata
from quip_b200.decode import (PromptDecoder, _constrain_advance_torch, _constrain_torch, _sample_torch,
                              _token_logprobs_torch, generate)
from test_generate import KINDS, _model, _prompts

EOS = 7
V = 199


def _same(a, b):
    """Bit for bit, every NaN counted equal to every NaN."""
    a, b = torch.as_tensor(a), torch.as_tensor(b)
    bits = (lambda x: x.contiguous().view(torch.int32)) if a.dtype == torch.float32 else \
        (lambda x: x.contiguous().view(torch.int16))
    nan = torch.isnan(a) & torch.isnan(b)
    return a.dtype == b.dtype and bool(((bits(a) == bits(b)) | nan).all())


def _row(n, g):
    x = torch.randn(n, generator=g) * 3
    for val, k in ((0.0, 6), (-0.0, 6), (float('inf'), 3), (float('-inf'), 3), (float('nan'), 3)):
        x[torch.randint(0, n, (k,), generator=g)] = val
    x[[0, n - 1]] = torch.tensor([-0.0, float('inf')])
    return x


def _random_automaton(g, n_states, vocab, eos=None):
    """A random cyclic automaton: states allowing 1, a few, or every token (ids 0 and vocab - 1 included)."""
    trans = {}
    for s in range(n_states):
        k = [1, 3, vocab, 12, 2][s % 5]
        ids = torch.randperm(vocab, generator=g)[:k].tolist()
        if s % 5 == 3:
            ids[:2] = [0, vocab - 1]
        trans[s] = {v: int(torch.randint(0, n_states, (1,), generator=g)) for v in ids}
    if eos is not None:
        trans[n_states - 1][eos] = 0
    return TokenAutomaton(trans, 0)


def test_torch_restatement_equals_hf_processor_and_the_oracle():
    from transformers.generation.logits_process import PrefixConstrainedLogitsProcessor
    g = torch.Generator().manual_seed(0)
    a = _random_automaton(g, 10, V)
    offsets, ids, nxt, (start,) = pack_automata([None, a][1:], V)
    for s in range(10):
        x = _row(V, g)
        want = PrefixConstrainedLogitsProcessor(lambda b, _: a.allowed(s), 1)(torch.zeros(1, 3, dtype=torch.long),
                                                                              x.clone()[None])[0]
        got = _constrain_torch(x.clone()[None], 1, torch.tensor([start + s], dtype=torch.int32), offsets, ids, nxt)[0]
        assert _same(got, want), s
        assert _same(got, torch.from_numpy(O.mask_row(x.numpy(), offsets.numpy(), ids.numpy(), nxt.numpy(), s)))
    allowed_all = next(s for s in range(10) if len(a.allowed(s)) == V)
    x = _row(V, g)
    y = _constrain_torch(x.clone()[None], 1, torch.tensor([allowed_all], dtype=torch.int32), offsets, ids, nxt)[0]
    want = x.clone()
    want[want == 0] = 0                                                        # -0 -> +0, everything else kept
    assert not torch.signbit(y[0]) and _same(y, want)


def test_draft_walks_and_unconstrained_rows():
    g = torch.Generator().manual_seed(1)
    a, b = _random_automaton(g, 8, V), _random_automaton(g, 5, V)
    offsets, ids, nxt, starts = pack_automata([a, None, b, a], V)
    B, T = 4, 5
    state = torch.tensor(starts, dtype=torch.int32)
    state[3] = offsets.numel() + 2                                             # out of range: untouched
    tokens = torch.randint(0, V, (B, T), generator=g)
    for r in (0, 2):                                                           # drafts along allowed arcs, then one not
        auto, s = (a, a.start) if r == 0 else (b, b.start)
        for j in range(1, 3):
            tokens[r, j] = auto.allowed(s)[0]
            s = auto.walk(s, [tokens[r, j]])
    x = torch.stack([_row(V, g) for _ in range(B * T)])
    got = _constrain_torch(x.clone(), T, state, offsets, ids, nxt, tokens=tokens)
    for r in range(B * T):
        row, i = divmod(r, T)
        want = O.mask_row(x[r].numpy(), offsets.numpy(), ids.numpy(), nxt.numpy(), int(state[row]),
                          tokens[row, 1:i + 1].tolist())
        assert _same(got[r], torch.from_numpy(want)), r
        if row in (1, 3):
            assert _same(got[r], x[r])
        else:
            auto = a if row == 0 else b
            allowed = auto.allowed(auto.walk(auto.start, tokens[row, 1:i + 1].tolist()))
            assert torch.equal(torch.isfinite(got[r]).nonzero()[:, 0], torch.isfinite(x[r]).nonzero()[:, 0][
                torch.isin(torch.isfinite(x[r]).nonzero()[:, 0], torch.tensor(allowed))])
    counts = torch.tensor([2, 5, 9, -1])
    st = _constrain_advance_torch(state.clone(), tokens, offsets, ids, nxt, counts=counts)
    want = O.advance(state.numpy(), tokens.numpy(), offsets.numpy(), ids.numpy(), nxt.numpy(), counts=counts.numpy())
    assert st.tolist() == want.tolist() and st[3] == state[3]
    assert int(st[0]) == starts[0] + a._index[a.walk(a.start, tokens[0, :2].tolist())]


def test_automaton_validation_and_helpers():
    with pytest.raises(ValueError, match='no token'):
        TokenAutomaton({0: {1: 1}, 1: {}}, 0)
    with pytest.raises(ValueError, match='not a state'):
        TokenAutomaton({0: {1: 5}}, 0)
    with pytest.raises(ValueError, match='start'):
        TokenAutomaton({0: {1: 0}}, 3)
    with pytest.raises(ValueError, match='integers'):
        TokenAutomaton({0: {-1: 0}}, 0)
    a = TokenAutomaton.from_sequences([[3, 4], [3, 5, 6], [9]], eos=[EOS, 8])
    assert a.allowed(a.start) == [3, 9] and a.allowed(a.walk(a.start, [3])) == [4, 5]
    assert a.allowed(a.walk(a.start, [3, 4])) == [EOS, 8]
    sink = a.walk(a.start, [9, EOS])
    assert a.allowed(sink) == [EOS, 8] and a.walk(sink, [EOS, 100]) == sink        # unchanged on a miss
    fn = a.hf_prefix_allowed_tokens_fn(2)
    assert fn(0, torch.tensor([50, 60, 3, 5])) == [6]
    with pytest.raises(ValueError, match='EOS'):
        TokenAutomaton.from_sequences([[3, EOS]], EOS)
    offsets, ids, nxt, starts = pack_automata([a, None, a], V)
    assert starts == [0, -1, 0] and offsets.numel() == len(a.states) + 1 and ids.numel() == nxt.numel()
    with pytest.raises(ValueError, match='vocabulary'):
        pack_automata([a], 8)


def _hf(m, p, n, eos, a, **kw):
    with torch.no_grad():
        r = m.generate(p[None], do_sample=False, max_new_tokens=n, eos_token_id=eos, pad_token_id=0,
                       prefix_allowed_tokens_fn=a.hf_prefix_allowed_tokens_fn(p.numel()), **kw)
    return r[0, p.numel():]


LABELS = [[10, 11, 12], [10, 20], [30], [40, 41, 42, 43]]
PROCESSORS = [dict(repetition_penalty=1.8), dict(no_repeat_ngram_size=2), dict(min_new_tokens=6),
              dict(bad_words_ids=[[11], [40, 41], [3, 4, 5]])]


@pytest.mark.parametrize('kind', KINDS)
def test_greedy_generate_equals_hf_for_each_prompt_alone(kind):
    m = _model(kind)
    prompts = _prompts(seed=3, lens=(5, 11, 2))
    g = torch.Generator().manual_seed(4)
    labels = TokenAutomaton.from_sequences(LABELS, EOS)
    cyclic = _random_automaton(g, 6, V, eos=EOS)
    runs = [(labels, 8, {}), (cyclic, 14, {})] + [(cyclic, 14, kw) for kw in PROCESSORS]
    runs.append((TokenAutomaton.from_sequences([[30]], EOS), 9, dict(min_new_tokens=5)))   # EOS-only state banned
    for a, n, kw in runs:
        got = generate(m, prompts, n, eos_token_id=EOS, token_constraint=a, **kw)
        for b, p in enumerate(prompts):
            w = _hf(m, p, n, EOS, a, **kw)
            assert torch.equal(got[b], w), (kind, kw, b, got[b], w)


def test_min_new_tokens_over_an_eos_only_state_keeps_the_state():
    m = _model('llama_mha')
    p = _prompts(seed=2)[0]
    a = TokenAutomaton.from_sequences([[30]], EOS)
    out, = generate(m, [p], 9, eos_token_id=EOS, token_constraint=a, min_new_tokens=5)
    assert out[0] == 30 and out[-1] == EOS and out.numel() == 6                # all-banned rows pick id 0
    assert a.walk(a.start, out[:-1].tolist()) == a.walk(a.start, [30])


def test_per_prompt_automata_and_unconstrained_rows_in_one_batch():
    m = _model('opt_pre_ln')
    prompts = _prompts(seed=5, lens=(6, 3, 9))
    g = torch.Generator().manual_seed(6)
    auts = [_random_automaton(g, 4, V), None, TokenAutomaton.from_sequences(LABELS, EOS)]
    got = generate(m, prompts, 10, eos_token_id=EOS, token_constraint=auts)
    free = generate(m, prompts, 10, eos_token_id=EOS)
    assert torch.equal(got[1], free[1])
    for b in (0, 2):
        assert torch.equal(got[b], _hf(m, prompts[b], 10, EOS, auts[b]))


def _obeys(a, toks):
    s = a.start
    for t in toks:
        if t not in a.allowed(s):
            return False
        s = a.walk(s, [t])
    return True


def test_sampled_rows_sample_the_masked_logits_and_obey_the_automaton():
    m = _model('llama_gqa')
    prompts = _prompts(seed=7, lens=(4, 8))
    g = torch.Generator().manual_seed(8)
    a = _random_automaton(g, 5, V)
    kw = dict(do_sample=True, temperature=0.9, top_k=20, seed=[3, 9], token_constraint=a)
    x, y = generate(m, prompts, 10, **kw), generate(m, prompts, 10, **kw)
    assert all(torch.equal(u, v) for u, v in zip(x, y)) and all(_obeys(a, o.tolist()) for o in x)
    dec = PromptDecoder(m, max_len=20, batch=2, max_new=10, sampling=True, constraint=True)
    dec.set_sampling(0.9, 20, 1.0, [3, 9])
    dec.set_constraint(*pack_automata([a, a], V))
    steps = [(dec.prefill(prompts).clone(), 0)]                                 # masked in place before the selection
    for t in range(1, 10):
        steps.append((dec.step().clone(), t))
    for t, (lg, s) in enumerate(steps):
        assert torch.equal(dec.generated[:, t], _sample_torch(lg, dec.temperature, dec.top_k, dec.top_p, dec.seed, s))
    assert all(torch.equal(dec.generated[r], x[r]) for r in range(2))


@pytest.mark.parametrize('sample', [False, True])
def test_speculative_batched_and_shared_runs_equal_plain_runs(sample):
    m = _model('llama_gqa')
    rep = torch.tensor([5, 6, 7, 8, 5, 6, 7, 8, 5, 6, 9])
    prompts = [rep, _prompts(seed=6)[1], _prompts(seed=6)[2]]
    g = torch.Generator().manual_seed(9)
    loop = TokenAutomaton({0: {5: 1, 6: 0, 9: 0}, 1: {6: 2, 7: 0}, 2: {7: 3, 8: 3}, 3: {8: 0, 5: 1}}, 0)
    auts = [loop, _random_automaton(g, 5, V), None]
    kw = dict(token_constraint=auts, eos_token_id=EOS, repetition_penalty=1.2)
    if sample:
        kw.update(do_sample=True, temperature=0.9, seed=[1, 2, 3])
    plain = generate(m, prompts, 16, **kw)
    stats = {}
    spec = generate(m, prompts, 16, prompt_lookup_num_tokens=3, spec_stats=stats, **kw)
    assert all(torch.equal(x, y) for x, y in zip(plain, spec)), (plain, spec)
    assert stats['accepted'][0] > 0
    cont = generate(m, prompts, 16, max_batch_size=2, prefill_chunk_size=4, **kw)
    assert all(torch.equal(x, y) for x, y in zip(plain, cont))
    for b, p in enumerate(prompts):                                             # each prompt as if alone
        one = {k: (v[b:b + 1] if isinstance(v, list) else v) for k, v in kw.items()}
        want, = generate(m, [p], 16, max_batch_size=1, **one)
        assert torch.equal(want, plain[b])


def test_return_sequences_and_shared_prefixes():
    m = _model('llama_mha')
    base = _prompts(seed=8, lens=(70,))[0]
    prompts = [base, torch.cat((base[:66], torch.tensor([3, 4])))]
    g = torch.Generator().manual_seed(10)
    auts = [_random_automaton(g, 4, V), None, TokenAutomaton.from_sequences(LABELS, EOS), _random_automaton(g, 3, V)]
    kw = dict(do_sample=True, seed=5, token_constraint=auts, eos_token_id=EOS)
    got = generate(m, prompts, 6, num_return_sequences=2, **kw)
    want = generate(m, [p for p in prompts for _ in range(2)], 6, share_prompt_prefixes=True, **kw)
    assert all(torch.equal(x, y) for x, y in zip(got, want))
    kw = dict(token_constraint=auts[2:], eos_token_id=EOS)
    shared = generate(m, prompts, 6, share_prompt_prefixes=True, **kw)
    plain = generate(m, prompts, 6, prefill_chunk_size=512, **kw)
    assert all(torch.equal(x, y) for x, y in zip(shared, plain))


@pytest.mark.parametrize('mode', ['plain', 'spec', 'continuous'])
def test_logprobs_stay_raw(mode):
    m = _model('opt_post_ln')
    prompts = _prompts(seed=11, lens=(5, 9))
    a = TokenAutomaton.from_sequences(LABELS, EOS)
    kw = dict(prompt_lookup_num_tokens=2) if mode == 'spec' else dict(max_batch_size=1) if mode == 'continuous' else {}
    lp = {}
    out = generate(m, prompts, 6, eos_token_id=EOS, token_constraint=a, logprobs=lp, top_logprobs=3, **kw)
    plain = generate(m, prompts, 6, eos_token_id=EOS, token_constraint=a, **kw)
    assert all(torch.equal(x, y) for x, y in zip(out, plain))
    for p, o, t in zip(prompts, out, lp['token']):
        with torch.no_grad():
            logits = m(torch.cat((p, o))[None]).logits[0, p.numel() - 1:-1]
        want, _ = _token_logprobs_torch(logits, o)
        assert torch.allclose(t, want, atol=1e-4), (t, want)
        assert torch.isfinite(t).all()


def test_kv_e4m3_and_prefill_chunks():
    m = _model('llama_gqa')
    prompts = _prompts(seed=12, lens=(9, 3, 14))
    a = TokenAutomaton.from_sequences(LABELS, EOS)
    for kw in (dict(prefill_chunk_size=4), dict(kv_dtype=torch.float8_e4m3fn, prefill_chunk_size=5)):
        out = generate(m, prompts, 6, eos_token_id=EOS, token_constraint=a, **kw)
        assert all(_obeys(a, o.tolist()) and o[-1] == EOS for o in out)
    out = generate(m, prompts, 6, eos_token_id=EOS, token_constraint=a, prefill_chunk_size=4)
    assert all(torch.equal(x, _hf(m, p, 6, EOS, a)) for x, p in zip(out, prompts))


def test_none_allocates_and_launches_nothing(monkeypatch):
    m = _model('llama_mha')
    prompts = _prompts(seed=10)
    made = []

    class Spy(PromptDecoder):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            made.append(self)
    monkeypatch.setattr(D, 'PromptDecoder', Spy)
    want = generate(m, prompts, 8)
    got = generate(m, prompts, 8, token_constraint=None)
    got2 = generate(m, prompts, 8, token_constraint=[None] * len(prompts))
    assert all(torch.equal(x, y) and torch.equal(x, z) for x, y, z in zip(got, want, got2))
    assert len(made) == 3 and not any(d.constrained or hasattr(d, 'cstate') for d in made)


def test_argument_errors_are_raised_before_any_work(monkeypatch):
    def no_decoder(*a, **k):
        raise AssertionError('work started')
    for name in ('PromptDecoder', 'SpecDecoder', 'ContinuousDecoder', 'BeamDecoder'):
        monkeypatch.setattr(D, name, no_decoder)
    m = _model('llama_gqa')
    p = _prompts()
    a = TokenAutomaton.from_sequences(LABELS, EOS)
    cases = ((dict(token_constraint=a, num_beams=2), 'num_beams'),
             (dict(token_constraint=[a, a]), 'token_constraint'),
             (dict(token_constraint=TokenAutomaton({0: {V: 0}}, 0)), 'vocabulary'),
             (dict(token_constraint=[a, 'x', None]), 'TokenAutomaton'))
    for kw, msg in cases:
        with pytest.raises(ValueError, match=msg):
            generate(m, p, 5, **kw)
    with pytest.raises(ValueError, match='constraint=True'):
        PromptDecoder(m, max_len=8, batch=1, max_new=2).set_constraint(*pack_automata([a], V))
    with pytest.raises(ValueError, match='max_new'):
        PromptDecoder(m, max_len=8, batch=1, constraint=True)


def test_wrappers_check_and_refuse_cpu_tensors():
    from quip_b200 import fused
    offsets, ids, nxt, _ = pack_automata([TokenAutomaton.from_sequences(LABELS, EOS)], V)
    x = torch.zeros(2, V, dtype=torch.float16)
    st = torch.zeros(2, dtype=torch.int32)
    with pytest.raises(RuntimeError, match='CUDA device only'):
        fused.constrain_mask(x, 1, st, offsets, ids, nxt)
    with pytest.raises(ValueError, match='fp16'):
        fused.constrain_mask(x.float(), 1, st, offsets, ids, nxt)
    with pytest.raises(ValueError, match='state'):
        fused.constrain_mask(x, 1, st.long(), offsets, ids, nxt)
    with pytest.raises(ValueError, match='ids'):
        fused.constrain_mask(x, 1, st, offsets, ids.long(), nxt)
    with pytest.raises(ValueError, match='drafts'):
        fused.constrain_mask(x, 2, st, offsets, ids, nxt)
    with pytest.raises(ValueError, match='T must'):
        fused.constrain_mask(torch.zeros(18, V, dtype=torch.float16), 9, st, offsets, ids, nxt)
    with pytest.raises(ValueError, match='pass rows'):
        fused.constrain_mask(torch.zeros(3, V, dtype=torch.float16), 1, st, offsets, ids, nxt)
    with pytest.raises(RuntimeError, match='CUDA device only'):
        fused.constrain_advance(st, torch.zeros(2, 1, dtype=torch.long), offsets, ids, nxt)
    with pytest.raises(ValueError, match='counts'):
        fused.constrain_advance(st, torch.zeros(2, 1, dtype=torch.long), offsets, ids, nxt, counts=torch.zeros(2))


def test_c_abi_argument_errors_surface_as_messages():
    from quip_b200 import _lib
    lib = _lib.load()
    buf = 64

    def mask(R=2, T=1, V=50, ld=50, logits=buf, state=buf, tokens=None, S=1, nnz=1):
        return lib.quip_constrain_mask(logits, ld, R, T, V, None, tokens, state, 2, buf, buf, buf, S, nnz, None)
    assert mask(V=2 ** 18 + 1, ld=2 ** 18 + 1) == 1 and b'V' in lib.quip_last_error()
    assert mask(ld=10) == 1 and b'ld' in lib.quip_last_error()
    assert mask(R=18, T=9) == 1 and mask(R=3, T=2, tokens=buf) == 1
    assert mask(state=None) == 1 and b'null' in lib.quip_last_error()
    assert mask(T=2, R=2) == 1 and b'null' in lib.quip_last_error()              # drafts needed at T > 1
    assert mask(logits=65) == 1 and b'aligned' in lib.quip_last_error()
    assert mask(state=66) == 1 and b'aligned' in lib.quip_last_error()
    assert mask(S=-1) == 1 and mask(R=0) == 0                                      # no rows: nothing to launch

    def adv(N=2, T=1, ld=1, tok=buf, counts=None):
        return lib.quip_constrain_advance(buf, 2, tok, ld, N, T, None, counts, buf, buf, buf, 1, 1, None)
    assert adv(ld=0) == 1 and b'ld' in lib.quip_last_error()
    assert adv(tok=None) == 1 and b'null' in lib.quip_last_error()
    assert adv(counts=68) == 1 and b'aligned' in lib.quip_last_error()
    assert adv(N=0) == 0


def test_oracle_agrees_on_fp16_rows():
    x = np.array([-0.0, np.inf, np.nan, 1.5, -np.inf, 2.0], dtype=np.float16)
    offsets, ids, nxt = np.array([0, 2, 3]), np.array([0, 3]), np.array([1, 0])
    y = O.mask_row(x, offsets, ids, nxt, 0)
    assert y.dtype == np.float16 and y[0] == 0 and not np.signbit(y[0]) and y[3] == x[3]
    assert np.isnan(y[1]) and np.isnan(y[2]) and y[4] == -np.inf and y[5] == -np.inf
    assert np.array_equal(O.mask_row(x, offsets, ids, nxt, -1), x, equal_nan=True)
    assert O.walk(offsets, ids, nxt, 0, [3, 5, 0]) == 1 and O.walk(offsets, ids, nxt, 7, [0]) == 7
