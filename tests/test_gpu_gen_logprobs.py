"""Log-probabilities of generation on the GPU: quip_token_topk_logprobs against oracle/topk_logprobs.py and the torch
restatement (ids exactly; every value bit for bit against quip_token_logprobs on the same row and id), its addressing
and column guards, captured steps against eager steps, and generate() end to end."""
import numpy as np
import pytest
import torch

import quip_b200.decode as D
from oracle.topk_logprobs import topk_row
from quip_b200 import fused
from quip_b200.decode import ContinuousDecoder, ContinuousSchedule, KV_PAGE, PromptDecoder, SpecDecoder, generate
from test_gpu_speculative import _tiny

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


def _logits(R, V, seed, ld, off):
    """fp16 rows (R, V) at row stride ld, starting off elements into the buffer (unaligned rows), with planted ties
    and +-0, a constant row (every id tied), a mostly -inf row, +-inf and NaN rows."""
    g = torch.Generator().manual_seed(seed)
    buf = torch.zeros(R * ld + off + 8, dtype=torch.float16)
    x = buf[off:off + R * ld].view(R, ld)[:, :V]
    x.copy_((torch.randn(R, V, generator=g) * 3).round(decimals=1).half())     # coarse: natural ties
    top = x.amax(-1)
    for r in range(0, R, 4):                                       # the max tied at a few ids, one of them -0 / +0
        x[r, torch.randint(0, V, (3,), generator=g)] = top[r]
    if V > 2:
        x[::5, :3] = torch.tensor([-0.0, 0.0, -0.0]).half()
    if R >= 8:
        x[1::8] = 0.75                                             # every id tied: the in-order tie scan
        x[2::8, 5:] = float('-inf')
        x[3::8, V // 2] = float('nan')
        x[4::8, V - 1] = float('-inf')
        x[5::8, [0, V // 3]] = float('inf')
    elif R > 1:
        x[-1, V // 2] = float('nan')
    return buf.to(DEV)[off:off + R * ld].view(R, ld)[:, :V]


def _tokens(R, V, seed):
    g = torch.Generator().manual_seed(seed)
    t = torch.randint(0, V, (R,), generator=g)
    t[::7] = -1
    t[3::7] = V
    return t.to(DEV)


def _check_values(x, tok, lp, ids, vals):
    """lp and every top value bit for bit against quip_token_logprobs on the same row and id (an id of -1 is out of
    range there too: NaN)."""
    R = x.shape[0]
    want = torch.empty(R, dtype=torch.float32, device=DEV)
    gr = torch.empty(R, dtype=torch.uint8, device=DEV)
    fused.token_logprobs(x, tok, want, gr)
    assert torch.equal(lp.view(torch.int32), want.view(torch.int32))
    for j in range(ids.shape[1]):
        fused.token_logprobs(x, ids[:, j].contiguous(), want, gr)
        assert torch.equal(vals[:, j].contiguous().view(torch.int32), want.view(torch.int32)), j


@pytest.mark.parametrize('n', [0, 1, 5, 20])
@pytest.mark.parametrize('V', [7, 50, 32000, 50272, 128256])
@pytest.mark.parametrize('T', [1, 5, 8])
@pytest.mark.parametrize('Rb', [1, 32, 256])
def test_kernel_matches_the_oracle(Rb, T, V, n):
    B = {1: 1, 32: 32 // T, 256: 256}[Rb]                         # R = T, about 32, and 256 T logits rows
    R = B * T
    ld, off = (V + 3, 1) if Rb == 32 else (V, 0)
    x = _logits(R, V, seed=R + V + n, ld=ld, off=off)
    tok = _tokens(R, V, seed=V + n)
    G = T + 2
    cols = torch.zeros(B, dtype=torch.long, device=DEV)
    lp = torch.full((B, G), 5.0, device=DEV)
    ids = torch.full((B, G, n), 9, dtype=torch.long, device=DEV) if n else None
    top = torch.full((B, G, n), 5.0, device=DEV) if n else None
    fused.token_topk_logprobs(x, tok, cols, lp, ids, top, T=T)
    got_lp = lp[:, :T].reshape(R)
    assert bool((lp[:, T:] == 5.0).all())
    if not n:
        _check_values(x, tok, got_lp, torch.zeros(R, 0, dtype=torch.long, device=DEV), torch.zeros(R, 0, device=DEV))
        return
    got_ids, got_top = ids[:, :T].reshape(R, n), top[:, :T].reshape(R, n)
    w_lp, w_ids, w_top = (torch.full_like(t, v) for t, v in ((lp, 5.0), (ids, 9), (top, 5.0)))
    D._token_topk_logprobs_torch(x, tok, cols, w_lp, w_ids, w_top, T=T)
    assert torch.equal(got_ids, w_ids[:, :T].reshape(R, n))
    assert bool((ids[:, T:] == 9).all())
    bad = got_ids < 0
    assert bool(torch.isnan(got_top[bad]).all())
    _check_values(x, tok, got_lp, got_ids, got_top)
    xc = x.cpu().numpy()
    for r in sorted({0, 1, 2, 3, 4, 5, R - 1} & set(range(R))):             # the numpy oracle on each row kind
        want_ids, want = topk_row(xc[r], n)
        assert np.array_equal(got_ids[r].cpu().numpy(), want_ids), r
        assert np.allclose(got_top[r].cpu().double().numpy(), want, atol=2e-5, rtol=0, equal_nan=True), r
    ids2, top2, lp2 = torch.zeros_like(ids), torch.zeros_like(top), torch.zeros_like(lp)
    fused.token_topk_logprobs(x, tok, cols, lp2, ids2, top2, T=T)             # repeated launches: the same bits
    assert torch.equal(ids2[:, :T], ids[:, :T]) and torch.equal(top2[:, :T].view(torch.int32),
                                                                 top[:, :T].view(torch.int32))
    assert torch.equal(lp2[:, :T].view(torch.int32), lp[:, :T].view(torch.int32))


@pytest.mark.parametrize('shared', [False, True])
@pytest.mark.parametrize('T', [1, 3])
def test_rows_map_and_column_guards(shared, T):
    B, G, n, V = 6, 5, 4, 32000
    rows = torch.tensor([4, -1, 0, 7, 2, 5], device=DEV)                # -1 and 7: outside [0, B), nothing written
    R = rows.numel() * T
    x = _logits(R, V, seed=11, ld=V, off=0)
    tok = _tokens(R, V, seed=12)
    cols = torch.tensor([3] if shared else [0, 9, -2, 0, 4, G - 1], device=DEV)
    lp = torch.full((B, G), 5.0, device=DEV)
    ids = torch.full((B, G, n), 9, dtype=torch.long, device=DEV)
    top = torch.full((B, G, n), 5.0, device=DEV)
    fused.token_topk_logprobs(x, tok, cols, lp, ids, top, T=T, rows=rows)
    w_lp, w_ids, w_top = torch.full_like(lp, 5.0), torch.full_like(ids, 9), torch.full_like(top, 5.0)
    D._token_topk_logprobs_torch(x, tok, cols, w_lp, w_ids, w_top, T=T, rows=rows)
    assert torch.equal(ids, w_ids)
    written = torch.zeros(B, G, dtype=torch.bool)
    for r in range(R):
        b = int(rows[r // T])
        if 0 <= b < B:
            c = int(cols[0 if shared else b]) + r % T
            if 0 <= c < G:
                written[b, c] = True
                one = torch.empty(1, device=DEV)
                fused.token_logprobs(x[r:r + 1], tok[r:r + 1], one, torch.empty(1, dtype=torch.uint8, device=DEV))
                assert torch.equal(lp[b, c:c + 1].view(torch.int32), one.view(torch.int32))
    assert written.any() and not written.all()
    keep = ~written.to(DEV)
    assert bool((lp[keep] == 5.0).all()) and bool((ids[keep] == 9).all()) and bool((top[keep] == 5.0).all())


def test_a_nan_row_gives_minus_one_and_nan_throughout():
    V, n = 50272, 20
    x = torch.randn(2, V, device=DEV).half()
    x[1, 17] = float('nan')
    lp = torch.zeros(2, 1, device=DEV)
    ids = torch.zeros(2, 1, n, dtype=torch.long, device=DEV)
    top = torch.zeros(2, 1, n, device=DEV)
    fused.token_topk_logprobs(x, torch.tensor([3, 3], device=DEV), torch.zeros(2, dtype=torch.long, device=DEV), lp,
                              ids, top)
    assert bool((ids[1] == -1).all()) and bool(torch.isnan(top[1]).all()) and bool(torch.isnan(lp[1]).all())
    assert bool((ids[0] >= 0).all()) and not bool(torch.isnan(top[0]).any())


# ---- decoders: captured against eager

def _prompt_run(model, prompts, cls, capture, processing, **kw):
    dec = cls(model, max_len=64, batch=len(prompts), max_new=12, processing=processing, sampling=True, logprobs=5,
              **kw)
    dec.set_sampling(0.9, 30, 0.95, [4, 5, 6])
    if processing:
        dec.set_processing([1.5, 1.0, 2.2], [2, 3, 1], [0, 4, 6], [[9], [30, 31], [100, 101, 102]], [17, 40])
    if capture:
        dec.capture()
    raws = [dec.prefill(prompts).clone()]
    for _ in range(6):
        raws.append(dec.step().clone())
    return dec, raws


@pytest.mark.parametrize('cls,processing', [(PromptDecoder, False), (PromptDecoder, True), (SpecDecoder, False),
                                            (SpecDecoder, True)])
def test_captured_step_equals_the_eager_step(cls, processing):
    model = _tiny((2, 64))
    g = torch.Generator().manual_seed(1)
    base = [torch.randint(0, 320, (n,), generator=g) for n in (4, 3, 5)]
    prompts = [torch.cat((p, p, p)) for p in base]
    kw = dict(draft_tokens=3) if cls is SpecDecoder else {}
    e, elog = _prompt_run(model, prompts, cls, False, processing, **kw)
    c, clog = _prompt_run(model, prompts, cls, True, processing, **kw)
    assert torch.equal(e.generated, c.generated)
    for a, b in ((e.lp, c.lp), (e.top_lp, c.top_lp)):
        assert torch.equal(a.view(torch.int32), b.view(torch.int32))
    assert torch.equal(e.top_ids, c.top_ids)
    if cls is PromptDecoder and not processing:
        # each column is quip_token_logprobs of that step's raw logits at the selected token
        for t, x in enumerate(elog):
            want = torch.empty(3, device=DEV)
            fused.token_logprobs(x, e.generated[:, t].contiguous(), want, torch.empty(3, dtype=torch.uint8, device=DEV))
            assert torch.equal(e.lp[:, t].contiguous().view(torch.int32), want.view(torch.int32)), t


def _serve(model, prompts, budgets, rows, chunk, capture):
    lens = [p.numel() for p in prompts]
    sched = ContinuousSchedule(lens, budgets, rows, rows * max(-(-(n + m) // KV_PAGE) for n, m in zip(lens, budgets)),
                               chunk)
    dec = ContinuousDecoder(model, max(n + m for n, m in zip(lens, budgets)), rows, len(sched.free_pages),
                            max(budgets), logprobs=3)
    if capture:
        dec.capture()
    out = [None] * len(prompts)
    while True:
        done, n_gen = dec.done.cpu(), dec.n_gen.cpu()
        for r, i in enumerate(sched.req):
            if i is not None and done[r]:
                k = int(n_gen[r])
                out[i] = (dec.generated[r, :k].cpu(), dec.lp[r, :k].cpu(), dec.top_ids[r, :k].cpu(),
                          dec.top_lp[r, :k].cpu())
                sched.retire(r)
                dec.retire(r)
        for r, i, pages in sched.admit():
            dec.admit(r, pages, budgets[i])
        if sched.finished:
            return out
        decoding, pieces = sched.plan()
        if pieces:
            dec.mixed_step(decoding, [(r, prompts[sched.req[r]][lo:lo + n], lo, lo + n == lens[sched.req[r]])
                                      for r, lo, n in pieces])
        else:
            dec.decode_step()


def test_continuous_captured_step_equals_the_eager_step():
    model = _tiny('opt')
    g = torch.Generator().manual_seed(3)
    prompts = [torch.randint(0, 320, (int(torch.randint(3, 40, (1,), generator=g)),), generator=g) for _ in range(7)]
    budgets = [12, 5, 20, 9, 3, 16, 7]
    e = _serve(model, prompts, budgets, rows=3, chunk=16, capture=False)
    c = _serve(model, prompts, budgets, rows=3, chunk=16, capture=True)
    for i in range(len(prompts)):
        assert e[i][0].numel() == budgets[i]
        for a, b in zip(e[i], c[i]):
            assert torch.equal(a.view(torch.int32) if a.dtype == torch.float32 else a,
                               b.view(torch.int32) if b.dtype == torch.float32 else b), i
        assert not bool(torch.isnan(e[i][1]).any())


# ---- generate() end to end

@pytest.mark.parametrize('kw', [dict(), dict(do_sample=True, temperature=0.8, top_p=0.9, seed=[1, 2, 3, 4]),
                                dict(prompt_lookup_num_tokens=3),
                                dict(repetition_penalty=1.4, no_repeat_ngram_size=2, bad_words_ids=[[11]]),
                                dict(max_batch_size=2, prefill_chunk_size=5, eos_token_id=[7])])
def test_tokens_are_bit_identical_with_logprobs_on(kw):
    model = _tiny((4, 64))
    g = torch.Generator().manual_seed(2)
    base = [torch.randint(0, 320, (n,), generator=g) for n in (5, 2, 7, 3)]
    prompts = [torch.cat((p, p, p[:2])) for p in base]
    off = generate(model, prompts, 14, **kw)
    lp = {}
    on = generate(model, prompts, 14, logprobs=lp, top_logprobs=20, **kw)
    for x, y, t, ids in zip(off, on, lp['token'], lp['top_ids']):
        assert torch.equal(x, y)
        assert t.shape == (x.numel(),) and ids.shape == (x.numel(), 20) and not bool(torch.isnan(t).any())
        if not kw.get('do_sample') and 'repetition_penalty' not in kw:
            assert torch.equal(ids[:, 0], x)


def test_sums_agree_with_score_on_a_7b_shaped_model_at_batch_32():
    """4 decoder layers of the Llama-2-7B shape (vocab 32000), B = 32, 256-token prompts, 64 new tokens: the logprob
    sums of generate against score of the same continuations, per token, within the 1.5e-2 rounding control of the
    score tests."""
    from quip_b200.decode import score
    from quip_b200.synth import build_synthetic_model, model_config
    cfg = model_config('llama7b', num_hidden_layers=4)
    model = build_synthetic_model(cfg, DEV, bits=2, seed=3, seqlen=512)
    g = torch.Generator().manual_seed(4)
    prompts = [torch.randint(0, cfg.vocab_size, (256,), generator=g) for _ in range(32)]
    lp = {}
    out = generate(model, prompts, 64, prefill_chunk_size=256, logprobs=lp, top_logprobs=5)
    assert all(torch.equal(x, y) for x, y in zip(out, generate(model, prompts, 64, prefill_chunk_size=256)))
    got = score(model, [p.tolist() for p in prompts], [o.tolist() for o in out], batch_size=32, max_length=512)
    worst = max(abs(float(t.double().sum()) - s) / t.numel() for t, (s, _) in zip(lp['token'], got))
    print(f'generate logprob sums against score: worst |diff| / tokens {worst:.2e}')
    assert worst <= 1.5e-2
    for t, ids, top in zip(lp['token'], lp['top_ids'], lp['top']):
        assert bool((top[:, :-1] >= top[:, 1:]).all()) and bool((top[:, 0] >= t).all())
