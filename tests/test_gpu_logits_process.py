"""Logits processors on the GPU: quip_logits_process bit for bit against oracle/logits_process.py (NaNs counted equal),
the captured step against the eager one, generate() against the same decoders with the torch restatement in place of
the kernel, and the processors' guarantees on a 7B-shaped synthetic packed model at B = 32."""
import numpy as np
import pytest
import torch

import quip_b200.decode as D
from oracle.logits_process import process_row
from quip_b200 import fused
from quip_b200.decode import PromptDecoder, SpecDecoder, generate
from test_gpu_speculative import _tiny

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


def _same(a, b):
    a, b = torch.as_tensor(a), torch.as_tensor(b)
    nan = torch.isnan(a) & torch.isnan(b)
    return bool(((a.view(torch.int16) == b.view(torch.int16)) | nan).all())


def _case(B, T, V, seed, long_rows=2):
    """Histories (B, max_len) with heavy repetition, ids 0, V - 1 and out-of-range ones, drafts (B, T), settings and a
    bad-word list with every length 1 .. 16, several planted at history ends."""
    g = np.random.default_rng(seed)
    max_len = 4096 + 16
    hist = np.zeros((B, max_len), dtype=np.int64)
    last = np.zeros(B, dtype=np.int64)
    alpha = np.array([0, V - 1, 1, 2, 3, 5, 8] + list(g.integers(0, V, 9)))
    for b in range(B):
        L = int(g.integers(4000, 4096)) if b < long_rows else int(g.integers(1, 200))
        pool = alpha if b % 2 else g.integers(0, V, 40)
        hist[b, :L] = g.choice(pool, L)
        if b % 7 == 3:
            hist[b, int(g.integers(0, L))] = -3 if b % 2 else V + 5
        last[b] = L - 1
    tokens = g.choice(alpha, (B, T)).astype(np.int64)
    tokens[:, 0] = hist[np.arange(B), last]
    plen = np.array([int(g.integers(1, last[b] + 2)) for b in range(B)], dtype=np.int64)
    pen = g.choice(np.array([1.0, 1.3, 0.6, 2.5], dtype=np.float32), B)
    ngram = np.array([[0, 1, 2, 3, 4, int(last[b]) + 3][b % 6] for b in range(B)], dtype=np.int32)
    min_new = g.integers(0, 40, B).astype(np.int32)
    eos = [int(x) for x in g.choice(alpha, 1 + seed % 3, replace=False)]
    bad = [list(map(int, g.choice(alpha, l))) for l in range(1, 17)]
    for b in range(0, B, 5):                                         # suffixes of histories, so they match
        l = 2 + b % 4
        h = list(hist[b, :last[b] + 1])
        if len(h) >= l - 1:
            bad.append(h[len(h) - l + 1:] + [int(g.integers(0, V))])
    bad = bad[:256] + [[eos[0]]]
    return dict(hist=hist, last=last, tokens=tokens, plen=plen, pen=pen, ngram=ngram, min_new=min_new, eos=eos,
                bad=bad)


def _logits(R, V, seed, ld=None, off=0):
    g = torch.Generator().manual_seed(seed)
    ld = ld or V
    buf = (torch.randn(R * ld + off + 8, generator=g) * 4).half()
    x = buf[off:off + R * ld].view(R, ld)[:, :V]
    x[:, 0] = -0.0
    x[::3, V - 1] = float('inf')
    x[1::3, V // 2] = float('nan')
    x[::2, 1] = float('-inf')
    x[:, 2] = 0.0
    x[::4, 3] = -0.0
    return x


def _device_args(c, T):
    bad = torch.zeros(len(c['bad']), 16, dtype=torch.long)
    for j, w in enumerate(c['bad']):
        bad[j, :len(w)] = torch.tensor(w)
    t = lambda a, dt=None: torch.as_tensor(a, dtype=dt).to(DEV)
    return (T, t(c['hist']), t(c['last']), t(c['plen']), t(c['pen']), t(c['ngram']), t(c['min_new']),
            t(c['eos'], torch.long), bad.to(DEV), t([len(w) for w in c['bad']], torch.int32)), t(c['tokens'])


def _oracle(x, c, T, rows=None):
    out = x.numpy().copy()
    for r in range(x.shape[0]):
        b = r // T if rows is None else int(rows[r // T])
        i = r % T
        h = list(c['hist'][b, :c['last'][b] + 1]) + list(c['tokens'][b, 1:i + 1])
        out[r] = process_row(out[r], [int(v) for v in h], int(c['plen'][b]), float(c['pen'][b]), int(c['ngram'][b]),
                             int(c['min_new'][b]), c['eos'], c['bad'])
    return torch.from_numpy(out)


def _on_device(x, ld=None):
    if ld is None:
        return x.to(DEV)
    full = torch.zeros(x.shape[0], ld, dtype=torch.float16, device=DEV)
    full[:, :x.shape[1]] = x.to(DEV)
    return full[:, :x.shape[1]]


@pytest.mark.parametrize('V', [50, 32000, 50272, 128256])
@pytest.mark.parametrize('T', [1, 5, 8])
@pytest.mark.parametrize('B', [1, 32, 256])
def test_kernel_matches_the_oracle(B, T, V):
    c = _case(B, T, V, seed=B + T + V, long_rows=2 if B * T <= 256 else 1)
    ld = V + 3 if B == 32 else None                                 # strided rows once per V
    x = _logits(B * T, V, seed=B * T + V)
    args, tokens = _device_args(c, T)
    xd = _on_device(x, ld)
    fused.logits_process(xd, *args, tokens=tokens)
    want = _oracle(x, c, T)
    assert _same(xd.cpu(), want)
    xd2 = _on_device(x, ld)                                         # repeated launches: the same bits
    fused.logits_process(xd2, *args, tokens=tokens)
    assert torch.equal(xd.cpu().view(torch.int16), xd2.cpu().view(torch.int16))


def test_rows_mapping_a_row_alone_and_all_off_rows():
    B, V = 24, 32000
    c = _case(B, 1, V, seed=3)
    x = _logits(10, V, seed=4)
    rows = torch.tensor([5, 0, 23, 11, 5, 7, 2, 19, 30, -1])       # repeats, and rows outside [0, B) are untouched
    args, _ = _device_args(c, 1)
    xd = x.to(DEV)
    fused.logits_process(xd, *args, rows=rows.to(DEV))
    assert _same(xd[:8].cpu(), _oracle(x[:8], c, 1, rows=rows[:8]))
    assert torch.equal(xd[8:].cpu().view(torch.int16), x[8:].view(torch.int16))
    one = x[2:3].to(DEV)                                            # row 23 alone
    fused.logits_process(one, *args, rows=rows[2:3].to(DEV))
    assert torch.equal(one.cpu().view(torch.int16), xd[2:3].cpu().view(torch.int16))
    off = dict(c, pen=np.ones(B, np.float32), ngram=np.zeros(B, np.int32), min_new=np.zeros(B, np.int32), bad=[])
    args, _ = _device_args(off, 1)
    xd = _logits(B, V, seed=5).to(DEV)
    x0 = xd.clone()
    fused.logits_process(xd, *args)
    assert torch.equal(xd.view(torch.int16), x0.view(torch.int16))


def _decoder(model, prompts, cls, capture, **kw):
    dec = cls(model, max_len=64, batch=len(prompts), max_new=12, processing=True, **kw)
    if kw.get('sampling'):
        dec.set_sampling(0.9, 30, 0.95, [4, 5, 6])
    dec.set_processing([1.5, 1.0, 2.2], [2, 3, 1], [0, 4, 6], [[9], [30, 31], [100, 101, 102]], [17, 40])
    if capture:
        dec.capture()
    logs = [dec.prefill(prompts).clone()]
    for _ in range(6):
        logs.append(dec.step().clone())
    return dec, logs


@pytest.mark.parametrize('spec', [False, True])
def test_captured_step_equals_the_eager_step(spec):
    model = _tiny((2, 64))
    g = torch.Generator().manual_seed(1)
    base = [torch.randint(0, 320, (n,), generator=g) for n in (4, 3, 5)]
    prompts = [torch.cat((p, p, p)) for p in base]
    cls = SpecDecoder if spec else PromptDecoder
    kw = dict(draft_tokens=3) if spec else {}
    e, elog = _decoder(model, prompts, cls, False, sampling=True, **kw)
    c, clog = _decoder(model, prompts, cls, True, sampling=True, **kw)
    assert torch.equal(e.generated, c.generated) and torch.equal(e.hist, c.hist)
    for a, b in zip(elog, clog):
        assert torch.equal(a.view(torch.int16), b.view(torch.int16))


def _restated(x, T, *args, tokens=None, rows=None):
    return D._process_torch(x, T, *args, tokens=tokens, rows=rows)


@pytest.mark.parametrize('mode', ['greedy', 'sampled', 'spec', 'continuous'])
def test_generate_equals_the_decoder_with_the_torch_restatement(mode, monkeypatch):
    model = _tiny((4, 64) if mode != 'continuous' else 'opt')
    g = torch.Generator().manual_seed(2)
    base = [torch.randint(0, 320, (n,), generator=g) for n in (5, 2, 7, 3)]
    prompts = [torch.cat((p, p, p[:2])) for p in base]
    kw = dict(repetition_penalty=[1.4, 2.0, 1.0, 1.2], no_repeat_ngram_size=[2, 0, 3, 1], min_new_tokens=[3, 0, 8, 2],
              bad_words_ids=[[11], [12, 13], [50, 51, 52]], eos_token_id=[7, 99])
    if mode == 'sampled':
        kw.update(do_sample=True, temperature=0.8, top_p=0.9, seed=[1, 2, 3, 4])
    if mode == 'spec':
        kw.update(prompt_lookup_num_tokens=3)
    if mode == 'continuous':
        kw.update(max_batch_size=2, prefill_chunk_size=5)
    got = generate(model, prompts, 14, **kw)
    monkeypatch.setattr(fused, 'logits_process', _restated)
    monkeypatch.setattr(D.GraphDecoder, 'capture', lambda self: self)   # the restatement syncs: eager steps
    want = generate(model, prompts, 14, **kw)
    for b, (x, y) in enumerate(zip(got, want)):
        assert torch.equal(x, y), (mode, b, x, y)


def test_guarantees_on_a_7b_shaped_model_at_batch_32():
    """4 decoder layers of the Llama-2-7B shape (hidden 4096, vocab 32000), B = 32, 512-token prompts, 128 new tokens:
    no 3-gram repeats in prompt plus output, no banned token is emitted, no EOS before min_new_tokens."""
    from quip_b200.synth import build_synthetic_model, model_config
    cfg = model_config('llama7b', num_hidden_layers=4)
    model = build_synthetic_model(cfg, DEV, bits=2, seed=3, seqlen=1024)
    g = torch.Generator().manual_seed(3)
    prompts = [torch.randint(0, cfg.vocab_size, (512,), generator=g) for _ in range(32)]
    plain = generate(model, prompts, 128, prefill_chunk_size=512)
    counts = torch.bincount(torch.cat(plain), minlength=cfg.vocab_size)
    top = counts.argsort(descending=True)[:10].tolist()
    eos, banned = top[:2], top[2:]                                  # tokens the plain run emits most
    n, min_new = 3, 64
    out = generate(model, prompts, 128, prefill_chunk_size=512, no_repeat_ngram_size=n, repetition_penalty=1.3,
                   bad_words_ids=[[t] for t in banned], min_new_tokens=min_new, eos_token_id=eos)
    for p, o in zip(prompts, out):
        assert not set(o.tolist()) & set(banned)
        hits = [j for j, t in enumerate(o.tolist()) if t in eos]
        assert not hits or hits[0] >= min_new, hits
        assert o.numel() == 128 or int(o[-1]) in eos
        seq = torch.cat((p, o)).tolist()
        seen = {tuple(seq[e:e + n]) for e in range(p.numel() - n + 1)}
        for e in range(p.numel() - n + 1, len(seq) - n + 1):
            gram = tuple(seq[e:e + n])
            assert gram not in seen, e
            seen.add(gram)
