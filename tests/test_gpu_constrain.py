"""Constrained generation on the GPU: quip_constrain_mask and quip_constrain_advance bit for bit against
oracle/constrain.py (NaNs counted equal), the captured steps against eager ones, generate() against the same decoders
with the torch restatements in place of the kernels, and every output obeying its automaton on a 7B-shaped synthetic
packed model at B = 32."""
import numpy as np
import pytest
import torch

import quip_b200.decode as D
from oracle import constrain as O
from quip_b200 import fused
from quip_b200.constrain import TokenAutomaton, pack_automata
from quip_b200.decode import generate
from test_gpu_speculative import _tiny

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


def _same(a, b):
    a, b = torch.as_tensor(a), torch.as_tensor(b)
    nan = torch.isnan(a) & torch.isnan(b)
    return bool(((a.view(torch.int16) == b.view(torch.int16)) | nan).all())


def _table(V, seed):
    """A packed table of 12 states: 1 token, every token, 10 tokens, ids 0 and V - 1, a third of the vocabulary, and
    random sizes; every next state in range, so draft walks move between them."""
    g = np.random.default_rng(seed)
    sizes = [1, V, 10, 2, V // 3 + 1, 1, 5, V, 64, 3, 10, 1]
    offsets, ids = [0], []
    for j, k in enumerate(sizes):
        s = np.sort(g.choice(V, k, replace=False)) if k < V else np.arange(V)
        if j == 3:
            s = np.array([0, V - 1])
        ids.extend(int(v) for v in s)
        offsets.append(len(ids))
    nxt = g.integers(0, len(sizes), len(ids))
    return (np.array(offsets, np.int32), np.array(ids, np.int32), nxt.astype(np.int32))


def _case(B, T, V, seed, table):
    g = np.random.default_rng(seed)
    offsets, ids, nxt = table
    S = len(offsets) - 1
    state = g.integers(0, S, B).astype(np.int32)
    state[::5] = -1                                                 # unconstrained
    state[3::7] = S + 2                                             # out of range: untouched
    tokens = g.integers(0, V, (B, T))
    for b in range(B):                                              # drafts mostly along allowed arcs
        s = int(state[b])
        for j in range(1, T):
            if 0 <= s < S and g.random() < 0.8:
                lo, hi = offsets[s], offsets[s + 1]
                tokens[b, j] = ids[g.integers(lo, hi)]
            s = O.delta(offsets, ids, nxt, s, tokens[b, j])
    return state, tokens.astype(np.int64)


def _logits(R, V, seed, ld, off):
    g = torch.Generator().manual_seed(seed)
    buf = (torch.randn(R * ld + off + 8, generator=g) * 4).half()
    x = buf[off:off + R * ld].view(R, ld)[:, :V]
    x[:, 0] = -0.0
    x[::3, V - 1] = float('inf')
    x[1::3, V // 2] = float('nan')
    x[::2, min(1, V - 1)] = float('-inf')
    x[::4, V // 3] = -0.0
    return x


def _oracle(x, table, state, tokens, T, rows=None):
    out = x.numpy().copy()
    for r in range(x.shape[0]):
        b = r // T if rows is None else int(rows[r // T])
        if not 0 <= b < len(state):
            continue
        out[r] = O.mask_row(out[r], *table, int(state[b]), [int(v) for v in tokens[b, 1:r % T + 1]])
    return torch.from_numpy(out)


def _dev(table):
    return [torch.from_numpy(t).to(DEV) for t in table]


@pytest.mark.parametrize('V', [199, 32000, 50272, 2 ** 18])
@pytest.mark.parametrize('T', [1, 4, 8])
def test_mask_matches_the_oracle(T, V):
    B = 12 if V < 2 ** 18 else 6
    table = _table(V, seed=V + T)
    state, tokens = _case(B, T, V, V * T, table)
    for ld, off in ((V, 0), (V + 3, 1), (V + 13, 5)):               # dense rows, then misaligned starts with ld > V
        x = _logits(B * T, V, seed=V + ld, ld=ld, off=off)
        base = torch.zeros(B * T * ld + off + 8, dtype=torch.float16, device=DEV)
        xd = base[off:off + B * T * ld].view(B * T, ld)[:, :V]
        xd.copy_(x)
        args = (T, torch.from_numpy(state).to(DEV), *_dev(table))
        fused.constrain_mask(xd, *args, tokens=torch.from_numpy(tokens).to(DEV))
        assert _same(xd.cpu(), _oracle(x, table, state, tokens, T)), (ld, off)
        again = xd.clone()
        again.copy_(x)
        fused.constrain_mask(again, *args, tokens=torch.from_numpy(tokens).to(DEV))
        assert torch.equal(again.view(torch.int16), xd.view(torch.int16))      # repeated launches: the same bits
        assert torch.equal(base[:off].cpu(), torch.zeros(off, dtype=torch.float16))


@pytest.mark.parametrize('T', [1, 4])
def test_mask_through_rows(T):
    V, B = 32000, 9
    table = _table(V, seed=7)
    state, tokens = _case(B, T, V, 8, table)
    rows = np.array([4, 0, 8, 4, -1, 2, 11, 7])                      # repeats, and rows outside [0, B)
    x = _logits(len(rows) * T, V, seed=9, ld=V, off=0)
    xd = x.to(DEV)
    fused.constrain_mask(xd, T, torch.from_numpy(state).to(DEV), *_dev(table), tokens=torch.from_numpy(tokens).to(DEV),
                         rows=torch.from_numpy(rows).to(DEV))
    assert _same(xd.cpu(), _oracle(x, table, state, tokens, T, rows=rows))
    for j in (4, 6):
        assert torch.equal(xd[j * T:(j + 1) * T].cpu().view(torch.int16), x[j * T:(j + 1) * T].view(torch.int16))


@pytest.mark.parametrize('T', [1, 3, 8])
def test_advance_matches_the_oracle(T):
    V, B = 50272, 40
    table = _table(V, seed=T)
    state, tokens = _case(B, T, V, 11 + T, table)
    g = np.random.default_rng(T)
    counts = g.integers(-1, T + 2, B).astype(np.int64)
    st = torch.from_numpy(state).to(DEV)
    fused.constrain_advance(st, torch.from_numpy(tokens).to(DEV), *_dev(table), counts=torch.from_numpy(counts).to(DEV))
    assert st.cpu().numpy().tolist() == O.advance(state, tokens, *table, counts=counts).tolist()
    rows = g.permutation(B + 4)[:20] - 2                              # distinct, a few outside [0, B)
    sub = tokens[:20]
    st = torch.from_numpy(state).to(DEV)
    fused.constrain_advance(st, torch.from_numpy(sub).to(DEV), *_dev(table), rows=torch.from_numpy(rows).to(DEV))
    assert st.cpu().numpy().tolist() == O.advance(state, sub, *table, rows=rows).tolist()


def _automata(vocab, seed, n):
    g = torch.Generator().manual_seed(seed)
    out = []
    for j in range(n):
        if j % 3 == 0:
            seqs = [torch.randint(1, vocab, (1 + k % 4,), generator=g).tolist() for k in range(4)]
            out.append(TokenAutomaton.from_sequences([[v for v in s if v != 7] or [8] for s in seqs], 7))
        elif j % 3 == 1:
            trans = {}
            for s in range(5):
                k = [10, vocab, 1, 40, 3][s]
                ids = torch.randperm(vocab, generator=g)[:k].tolist()
                trans[s] = {v: int(torch.randint(0, 5, (1,), generator=g)) for v in ids}
            out.append(TokenAutomaton(trans, 0))
        else:
            out.append(None)
    return out


def _obeys(a, toks):
    s = a.start
    for t in toks:
        if t not in a.allowed(s):
            return False
        s = a.walk(s, [t])
    return True


MODES = [('plain', None, False), ('plain', torch.float8_e4m3fn, True), ('spec', None, True),
         ('spec', torch.float8_e4m3fn, False), ('continuous', None, True), ('continuous', torch.float8_e4m3fn, True)]


@pytest.mark.parametrize('mode,kv,paged', MODES)
def test_captured_steps_equal_eager_steps(mode, kv, paged, monkeypatch):
    model = _tiny((2, 64) if mode != 'continuous' else 'opt')
    g = torch.Generator().manual_seed(2)
    base = [torch.randint(0, 320, (n,), generator=g) for n in (5, 2, 7, 3)]
    prompts = [torch.cat((p, p, p[:2])) for p in base]
    kw = dict(token_constraint=_automata(320, 3, 4), eos_token_id=7, kv_dtype=kv, do_sample=True, seed=[1, 2, 3, 4],
              temperature=0.8, repetition_penalty=1.3)
    if mode == 'spec':
        kw.update(prompt_lookup_num_tokens=3)
    if mode == 'continuous':
        kw.update(max_batch_size=2, prefill_chunk_size=5)
    elif paged:
        kw.update(share_prompt_prefixes=True)
    lp = {}
    got = generate(model, prompts, 14, logprobs=lp, **kw)
    monkeypatch.setattr(D.GraphDecoder, 'capture', lambda self: self)
    lp2 = {}
    want = generate(model, prompts, 14, logprobs=lp2, **kw)
    for b, (x, y) in enumerate(zip(got, want)):
        assert torch.equal(x, y), (mode, b, x, y)
        assert torch.equal(lp['token'][b], lp2['token'][b])
    for a, o in zip(kw['token_constraint'], got):
        assert a is None or _obeys(a, o.tolist())


@pytest.mark.parametrize('mode', ['greedy', 'sampled', 'spec', 'continuous'])
def test_generate_equals_the_decoder_with_the_torch_restatements(mode, monkeypatch):
    model = _tiny((4, 64) if mode != 'continuous' else 'opt')
    g = torch.Generator().manual_seed(4)
    base = [torch.randint(0, 320, (n,), generator=g) for n in (5, 2, 7, 3)]
    prompts = [torch.cat((p, p, p[:2])) for p in base]
    kw = dict(token_constraint=_automata(320, 5, 4), eos_token_id=[7, 99], min_new_tokens=[3, 0, 8, 2],
              bad_words_ids=[[11]])
    if mode == 'sampled':
        kw.update(do_sample=True, temperature=0.8, top_p=0.9, seed=[1, 2, 3, 4])
    if mode == 'spec':
        kw.update(prompt_lookup_num_tokens=3)
    if mode == 'continuous':
        kw.update(max_batch_size=2, prefill_chunk_size=5)
    got = generate(model, prompts, 14, **kw)
    monkeypatch.setattr(fused, 'constrain_mask', D._constrain_torch)
    monkeypatch.setattr(fused, 'constrain_advance', D._constrain_advance_torch)
    monkeypatch.setattr(D.GraphDecoder, 'capture', lambda self: self)   # the restatements sync: eager steps
    want = generate(model, prompts, 14, **kw)
    for b, (x, y) in enumerate(zip(got, want)):
        assert torch.equal(x, y), (mode, b, x, y)


def test_every_output_obeys_its_automaton_on_a_7b_shaped_model_at_batch_32():
    """4 decoder layers of the Llama-2-7B shape (hidden 4096, vocab 32000), B = 32, 256-token prompts, 48 new tokens,
    greedy and sampled: label sets, cyclic automata with states of 1 .. 32000 tokens, and unconstrained rows."""
    from quip_b200.synth import build_synthetic_model, model_config
    cfg = model_config('llama7b', num_hidden_layers=4)
    model = build_synthetic_model(cfg, DEV, bits=2, seed=3, seqlen=512)
    g = torch.Generator().manual_seed(3)
    prompts = [torch.randint(0, cfg.vocab_size, (256,), generator=g) for _ in range(32)]
    auts = _automata(cfg.vocab_size, 6, 32)
    free = generate(model, prompts, 48, prefill_chunk_size=256)
    for kw in (dict(), dict(do_sample=True, seed=11, top_k=50)):
        out = generate(model, prompts, 48, prefill_chunk_size=256, eos_token_id=7, token_constraint=auts, **kw)
        for j, (a, o) in enumerate(zip(auts, out)):
            if a is None:
                assert kw or torch.equal(o, free[j][:o.numel()])
            else:
                assert _obeys(a, o.tolist()), (j, o)
