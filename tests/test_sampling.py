"""Sampled token selection on the CPU: oracle/sampling.py (Philox known answers, HF's warpers on tie-free rows), the torch
restatement of the rule in quip_b200/decode.py against the oracle, generate(do_sample=True) on tiny HF models, and the
argument checks of generate, fused.sample and quip_sample."""
import numpy as np
import pytest
import torch

from oracle import sampling as S
from quip_b200 import _lib
from quip_b200 import decode
from quip_b200.decode import _sample_torch, generate

from test_generate import _hf_greedy, _model, _prompts


@pytest.mark.parametrize('counter, key, want', [
    ([0, 0, 0, 0], [0, 0], [0x6627e8d5, 0xe169c58d, 0xbc57ac4c, 0x9b00dbd8]),
    ([0xffffffff] * 4, [0xffffffff] * 2, [0x408f276d, 0x41c83b0e, 0xa20bc7c6, 0x6d5451fd]),
    ([0x243f6a88, 0x85a308d3, 0x13198a2e, 0x03707344], [0xa4093822, 0x299f31d0],
     [0xd16cfe09, 0x94fdcceb, 0x5001e420, 0x24126ea1]),
])
def test_oracle_philox_reproduces_the_random123_known_answers(counter, key, want):
    assert S.philox4x32_10(counter, key) == want


def test_decode_philox_equals_the_oracle():
    for seed in (0, 1, 2 ** 63, 2 ** 64 - 1, 0x123456789abcdef0):
        for t in (0, 1, 7, 2 ** 32 + 3):
            assert decode._philox_uniform(seed, t) == S.uniform(seed, t)


def _row(kind, V, g):
    """fp16-representable logits as float32: random (several scales), tie-heavy (few distinct values) or all equal."""
    if kind == 'random':
        x = torch.randn(V, generator=g) * float(torch.tensor([1.0, 3.0, 6.0])[torch.randint(0, 3, (1,), generator=g)])
    elif kind == 'ties':
        x = torch.randint(0, 6, (V,), generator=g).float() * 1.5
    else:
        x = torch.full((V,), 0.75)
    return x.half().float()


SETTINGS = [(0.0, 0, 1.0), (0.7, 1, 1.0), (0.7, 50, 0.9), (1.0, 0, 1.0), (1.0, 5, 1.0), (1.3, 0, 0.9), (0.5, 0, 0.3),
            (1.0, 0, 1e-6), (0.8, 10 ** 6, 0.95), (1.0, 3, 0.01), (2.0, 20, 1.0)]


def _cases(V, n, seed):
    g = torch.Generator().manual_seed(seed)
    for i in range(n):
        kind = ('random', 'ties', 'equal')[i % 3]
        T, k, p = SETTINGS[i % len(SETTINGS)]
        if k == 10 ** 6:
            k = V + 3                                                 # k >= V: every token a candidate
        sd = int(torch.randint(0, 2 ** 62, (1,), generator=g)) * 4 + i % 4
        yield _row(kind, V, g), T, k, p, sd, int(torch.randint(0, 1000, (1,), generator=g))


@pytest.mark.parametrize('V', [1, 7, 199, 32001])
def test_torch_restatement_picks_the_oracle_token(V):
    n = 24 if V == 32001 else 66
    amb = 0
    for x, T, k, p, sd, t in _cases(V, n, seed=V):
        want = S.sample_row(x.numpy(), T, k, p, sd, t)
        bits = torch.tensor([sd - 2 ** 64 if sd >= 2 ** 63 else sd])         # the int64 buffer holds the seed's bits
        got = int(_sample_torch(x[None], torch.tensor([T]), torch.tensor([k]), torch.tensor([p]), bits, t)[0])
        assert 0 <= got < V
        if want['ambiguous']:
            amb += 1
            assert got in want['kept'].tolist()
            continue
        assert got == want['token'], (T, k, p, sd, t)
    assert amb <= n // 2                      # flat rows with every token kept are near a boundary by the margin's measure


def test_kept_set_equals_hf_warpers_on_tie_free_rows():
    """HF applies Temperature -> TopK -> TopP (transformers' _get_logits_processor order); on rows without ties its kept
    set is the oracle's and softmax over it the oracle's probabilities."""
    from transformers.generation.logits_process import TemperatureLogitsWarper, TopKLogitsWarper, TopPLogitsWarper
    g = torch.Generator().manual_seed(3)
    checked = 0
    for i in range(60):
        V = (50, 199, 1000)[i % 3]
        x = torch.randn(V, generator=g, dtype=torch.float64).float() * 2
        assert torch.unique(x).numel() == V
        T, k, p = (0.7, 1.3, 1.0)[i % 3], (0, 5, 40, V)[i % 4], (1.0, 0.9, 0.5, 0.2, 0.97)[i % 5]
        want = S.sample_row(x.numpy(), T, k, p, i, 0)
        scores = TemperatureLogitsWarper(T)(None, x[None].clone())
        if 0 < k < V:
            scores = TopKLogitsWarper(k)(None, scores)
        if p < 1:
            scores = TopPLogitsWarper(p)(None, scores)
        keep = torch.isfinite(scores[0]).nonzero()[:, 0].numpy()
        if want['ambiguous']:                                         # HF's fp32 cumsum too close to the boundary to say
            continue
        assert sorted(keep.tolist()) == sorted(want['kept'].tolist()), (V, T, k, p)
        hf = torch.softmax(scores[0].double(), -1)[want['kept']].numpy()
        np.testing.assert_allclose(hf, want['probs'], rtol=1e-5, atol=1e-12)
        checked += 1
    assert checked >= 55


@pytest.mark.parametrize('kind', ['llama_mha', 'llama_gqa', 'opt_pre_ln'])
def test_generate_samples_reproducibly_per_seed_and_row(kind):
    m = _model(kind)
    prompts = _prompts()
    n = 12
    kw = dict(do_sample=True, temperature=1.5, top_k=40, top_p=0.95)
    a = generate(m, prompts, n, seed=11, **kw)
    b = generate(m, prompts, n, seed=11, **kw)
    c = generate(m, prompts, n, seed=12, **kw)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
    assert any(not torch.equal(x, y) for x, y in zip(a, c))
    seeds = [5, 2 ** 64 - 1, 2 ** 63]
    batched = generate(m, prompts, n, seed=seeds, **kw)
    for p, sd, got in zip(prompts, seeds, batched):
        alone, = generate(m, [p], n, seed=[sd], **kw)
        assert torch.equal(alone, got)
    # an int seed gives prompt b the seed seed + b
    assert torch.equal(generate(m, [prompts[1]], n, seed=[12], **kw)[0], a[1])


@pytest.mark.parametrize('kind', ['llama_gqa', 'opt_pre_ln'])
def test_top_k_one_and_temperature_zero_are_hf_greedy(kind):
    m = _model(kind)
    prompts = _prompts(seed=3)
    want = [_hf_greedy(m, p, 10) for p in prompts]
    for kw in (dict(top_k=1, temperature=1.7, top_p=0.5), dict(temperature=0.0)):
        got = generate(m, prompts, 10, do_sample=True, seed=[1, 2, 3], **kw)
        assert all(torch.equal(g, w) for g, w in zip(got, want)), kw


def test_sampled_generation_cuts_after_the_first_eos():
    m = _model('llama_gqa')
    prompts = _prompts(seed=2)
    n = 40 - max(p.numel() for p in prompts)
    kw = dict(do_sample=True, temperature=1.2, top_p=0.9, seed=[7, 8, 9])
    free = generate(m, prompts, n, **kw)
    eos = int(free[0][3])
    got = generate(m, prompts, n, eos_token_id=eos, **kw)
    for f, g in zip(free, got):
        hit = (f == eos).nonzero()
        assert torch.equal(g, f[:int(hit[0]) + 1] if hit.numel() else f)
    assert got[0].numel() <= 4 and int(got[0][-1]) == eos


def test_prompt_decoder_sampling_false_is_unchanged_and_set_sampling_checks():
    m = _model('llama_mha')
    prompts = _prompts()
    dec = decode.PromptDecoder(m, max_len=24, batch=3, max_new=4)
    with pytest.raises(ValueError, match='sampling=True'):
        dec.set_sampling(temperature=0.5)
    dec = decode.PromptDecoder(m, max_len=24, batch=3, max_new=4, sampling=True)
    with pytest.raises(ValueError, match='2 values'):
        dec.set_sampling(top_k=[1, 2])
    with pytest.raises(ValueError, match='2\\^64'):
        dec.set_sampling(seed=-1)
    dec.set_sampling(top_k=1, seed=torch.tensor([-1, 0, 5]))         # int64 bits: -1 is 2^64 - 1
    assert dec.seed.tolist() == [-1, 0, 5]
    dec.prefill(prompts)
    for _ in range(3):
        dec.step()
    want = [_hf_greedy(m, p, 4) for p in prompts]
    assert all(torch.equal(dec.generated[b], want[b]) for b in range(3))


def test_generate_rejects_bad_sampling_settings_before_any_work(monkeypatch):
    m = _model('llama_mha')
    p = _prompts()[:2]

    def no_work(*a, **k):
        raise AssertionError('a decoder was built')
    monkeypatch.setattr(decode, 'PromptDecoder', no_work)
    bad = [dict(temperature=-0.1), dict(temperature=float('nan')), dict(temperature=float('inf')), dict(top_p=0.0),
           dict(top_p=1.5), dict(top_p=float('nan')), dict(top_k=-1), dict(top_k=2.5), dict(seed=-1), dict(seed=2 ** 64),
           dict(seed=[1, 2, 3]), dict(temperature=[0.5]), dict(top_k=[1, 2, 3]), dict(seed=[1, -2])]
    for kw in bad:
        with pytest.raises(ValueError):
            generate(m, p, 4, do_sample=True, **kw)
    for kw in (dict(temperature=0.5), dict(top_k=5), dict(top_p=0.9), dict(seed=3), dict(seed=[0, 0])):
        with pytest.raises(ValueError, match='do_sample=True'):
            generate(m, p, 4, **kw)


def test_quip_sample_argument_errors_surface_as_messages():
    lib = _lib.load()
    buf = 64

    def call(B=2, V=320, logits=buf, seed=buf, step=buf, out=buf):
        return lib.quip_sample(logits, buf, buf, buf, seed, step, out, B, V, None)
    assert call(B=-1) == 1 and b'bad sizes' in lib.quip_last_error()
    assert call(V=0) == 1 and b'bad sizes' in lib.quip_last_error()
    assert call(V=(1 << 24) + 1) == 1 and b'bad sizes' in lib.quip_last_error()
    assert call(V=1 << 24) == 1 and b'bad sizes' in lib.quip_last_error()     # 2^24 weights of 2^40 wrap the sum
    for kw in (dict(logits=None), dict(seed=None), dict(step=None), dict(out=None)):
        assert call(**kw) == 1 and b'null' in lib.quip_last_error()
    with pytest.raises(_lib.QuipError, match='null pointer'):
        _lib.check(call(out=None))
    assert call(B=0) == 0                                             # no rows: nothing to launch


def test_sample_wrapper_checks_and_refuses_cpu_tensors():
    from quip_b200 import fused
    B, V = 3, 50
    args = dict(logits=torch.zeros(B, V, dtype=torch.float16), temperature=torch.ones(B), top_k=torch.zeros(B, dtype=torch.int32),
                top_p=torch.ones(B), seed=torch.zeros(B, dtype=torch.int64), step=torch.zeros(1, dtype=torch.int64),
                out=torch.zeros(B, dtype=torch.int64))
    with pytest.raises(RuntimeError, match='CUDA device only'):
        fused.sample(**args)
    for name, bad in (('logits', torch.zeros(B, V)), ('top_k', torch.zeros(B, dtype=torch.int64)),
                      ('seed', torch.zeros(B + 1, dtype=torch.int64)), ('step', torch.zeros(2, dtype=torch.int64))):
        with pytest.raises(ValueError, match=name):
            fused.sample(**{**args, name: bad})
    wide = torch.empty(B, 1 << 24, dtype=torch.float16)                # 2^24 weights of 2^40 would wrap the sum
    with pytest.raises(ValueError, match=r'sample: need 1 <= V <= 16777215'):
        fused.sample(**{**args, 'logits': wide})
    steps = torch.zeros(B, dtype=torch.int64)
    with pytest.raises(ValueError, match=r'sample_at: need 1 <= V <= 16777215'):
        fused.sample_at(wide.view(B, 1, -1), *[args[k] for k in ('temperature', 'top_k', 'top_p', 'seed')], steps,
                        args['out'].view(B, 1))
