"""Continuous batching (generate(..., max_batch_size=n): ContinuousSchedule, ContinuousDecoder) on the tiny fp32 HF models
of test_generate on the CPU, where the mixed step's ragged attention is its torch restatement (per-sequence scatter
through the page table, SDPA under each sequence's causal mask)."""
import random

import pytest
import torch

from quip_b200 import _lib
from quip_b200.decode import KV_PAGE, ContinuousDecoder, ContinuousSchedule, PromptDecoder, generate
from test_generate import KINDS, _model, _prompts


# ---- the schedule on its own

def _simulate(lens, max_new, rows, n_pages, chunk, stop, check_every=1):
    """Drive a ContinuousSchedule as generate() does, with request i finishing after stop[i] tokens, and check the
    invariants after every admission and step.  Returns the admission order."""
    s = ContinuousSchedule(lens, max_new, rows, n_pages, chunk)
    need = [-(-(n + m) // KV_PAGE) for n, m in zip(lens, max_new)]
    n_gen = {}
    order = []
    steps = 0
    while True:
        if s.queue or steps % check_every == 0:
            for r, i in enumerate(s.req):
                if i is not None and n_gen.get(r, 0) >= stop[i]:
                    assert s.retire(r) == i
                    n_gen.pop(r)
            for r, i, pages in s.admit():
                assert len(pages) == need[i]
                order.append(i)
            owned = [p for ps in s.pages for p in ps]
            assert len(owned) == len(set(owned))                               # no page owned by two live rows
            assert len(owned) + len(s.free_pages) == n_pages
            assert not set(owned) & set(s.free_pages)
            if s.queue:                                                        # never idle while a request fits
                assert not s.free_rows or len(s.free_pages) < need[s.queue[0]]
        if s.finished:
            break
        decoding, pieces = s.plan()
        assert sum(n for _, _, n in pieces) <= chunk
        assert all(s.req[r] is not None for r in decoding)
        assert not set(decoding) & {r for r, _, _ in pieces}
        for r in decoding:
            n_gen[r] = n_gen.get(r, 0) + (n_gen.get(r, 0) < stop[s.req[r]])
        for r, lo, n in pieces:
            if lo + n == lens[s.req[r]]:
                n_gen[r] = 1                                                   # the first token comes from the prefill
        steps += 1
    assert sorted(s.free_pages) == list(range(n_pages)) and sorted(s.free_rows) == list(range(rows))
    return order


@pytest.mark.parametrize('seed', range(12))
def test_schedule_invariants_on_random_workloads(seed):
    g = random.Random(seed)
    n = g.randrange(1, 40)
    lens = [g.randrange(1, 300) for _ in range(n)]
    max_new = [g.randrange(1, 200) for _ in range(n)]
    stop = [g.randrange(1, m + 1) for m in max_new]
    need = max(-(-(a + b) // KV_PAGE) for a, b in zip(lens, max_new))
    rows = g.randrange(1, 9)
    n_pages = g.randrange(need, need * (rows + 1) + 1)
    order = _simulate(lens, max_new, rows, n_pages, g.choice([1, 7, 64, 512]), stop, check_every=g.choice([1, 16]))
    assert order == list(range(n))                                             # FIFO


def test_schedule_packs_short_prompts_into_one_step_and_spans_long_ones():
    s = ContinuousSchedule([3, 4, 20], [2, 2, 2], rows=3, n_pages=3, chunk=8)
    assert [(r, i) for r, i, _ in s.admit()] == [(0, 0), (1, 1), (2, 2)]
    assert s.plan() == ([], [(0, 0, 3), (1, 0, 4), (2, 0, 1)])
    assert s.plan() == ([0, 1], [(2, 1, 8)])
    assert s.plan() == ([0, 1], [(2, 9, 8)])
    assert s.plan() == ([0, 1], [(2, 17, 3)])
    assert s.plan() == ([0, 1, 2], [])


def test_schedule_waits_for_pages_and_refuses_a_budget_beyond_the_pool():
    s = ContinuousSchedule([100, 10, 10], [28, 5, 5], rows=3, n_pages=3, chunk=512)
    assert [(r, i, p) for r, i, p in s.admit()] == [(0, 0, [0, 1]), (1, 1, [2])]
    assert s.admit() == [] and list(s.queue) == [2]                            # a row is free, a page is not
    s.retire(1)
    assert s.admit() == [(1, 2, [2])]
    with pytest.raises(ValueError, match='pages'):
        ContinuousSchedule([100], [29], rows=1, n_pages=2, chunk=8)


# ---- generate(max_batch_size=...) against each prompt alone

def _workload(kind, seed=5):
    lens = (5, 11, 2, 7, 3, 9) if kind.startswith('llama') else (5, 11, 2, 7, 3)
    prompts = _prompts(seed=seed, lens=lens)
    budgets = [9, 4, 12, 6, 7, 3][:len(prompts)]
    return prompts, budgets


def _alone(m, prompts, budgets, C, kw, eos=None):
    out = []
    for i, (p, k) in enumerate(zip(prompts, budgets)):
        one = dict(kw)
        if 'seed' in one:
            one['seed'] = one['seed'] + i
        out.append(generate(m, [p], k, prefill_chunk_size=C, eos_token_id=eos, **one)[0])
    return out


@pytest.mark.parametrize('mode', ['greedy', 'sampled'])
@pytest.mark.parametrize('kv', ['fp32', 'e4m3'])
@pytest.mark.parametrize('kind', KINDS)
def test_continuous_generate_equals_each_prompt_alone(kind, kv, mode):
    m = _model(kind)
    prompts, budgets = _workload(kind)
    kw = dict(kv_dtype=torch.float8_e4m3fn) if kv == 'e4m3' else {}
    if mode == 'sampled':
        kw.update(do_sample=True, temperature=0.8, top_k=40, seed=11)
    free = _alone(m, prompts, budgets, 7, kw)
    eos = int(free[0][2])                                                      # row 0 stops at its third token
    want = {C: _alone(m, prompts, budgets, C, kw, eos=eos) for C in (1, 7, 64)}
    assert want[7][0].numel() <= 3 and int(want[7][0][-1]) == eos
    need = max(-(-(len(p) + k) // KV_PAGE) for p, k in zip(prompts, budgets))
    for B in (1, 2, 3, len(prompts)):
        for C in (1, 7, 64):
            got = generate(m, prompts, budgets, eos_token_id=eos, max_batch_size=B, prefill_chunk_size=C, **kw)
            assert len(got) == len(prompts)
            for i, (g, w) in enumerate(zip(got, want[C])):
                assert torch.equal(g, w), (B, C, i, g, w)
    # a pool of one request's pages: every admission waits for the previous request's pages
    got = generate(m, prompts, budgets, eos_token_id=eos, max_batch_size=3, prefill_chunk_size=7, kv_pages=need, **kw)
    for i, (g, w) in enumerate(zip(got, want[7])):
        assert torch.equal(g, w), (i, g, w)


def test_per_prompt_budgets_on_the_fixed_batch_paths():
    m = _model('llama_gqa')
    prompts, budgets = _workload('llama_gqa')
    full = generate(m, prompts, max(budgets))
    for kw in ({}, dict(prefill_chunk_size=4), dict(share_prompt_prefixes=True),
               dict(prompt_lookup_num_tokens=2)):
        got = generate(m, prompts, budgets, **kw)
        for g, f, k in zip(got, full, budgets):
            assert torch.equal(g, f[:k]), (kw, g, f, k)


# ---- the mixed step against the padded chunk path

@pytest.mark.parametrize('kv', ['fp32', 'e4m3'])
@pytest.mark.parametrize('kind', KINDS)
def test_mixed_step_equals_the_padded_chunk_path(kind, kv):
    m = _model(kind)
    kv_dtype = torch.float8_e4m3fn if kv == 'e4m3' else None
    prompts = _prompts(seed=7, lens=(9, 4, 13))
    max_len = 32
    ref = PromptDecoder(m, max_len=max_len, batch=3, kv_dtype=kv_dtype, n_pages=3,
                        page_table=torch.arange(3, dtype=torch.int32)[:, None])
    want = ref.prefill(prompts, chunk=5)
    dec = ContinuousDecoder(m, max_len, 3, n_pages=3, max_new=4, kv_dtype=kv_dtype)
    for b in range(3):
        dec.admit(b, [b], 4)
    # row 0 in two pieces over two steps, rows 1 and 2 whole in the first and second step
    dec.mixed_step([], [(0, prompts[0][:5], 0, False), (1, prompts[1], 0, True)])
    dec.mixed_step([1], [(0, prompts[0][5:], 5, True), (2, prompts[2], 0, True)])
    assert dec.n_gen.tolist() == [1, 2, 1]
    assert dec.generated[:, 0].tolist() == want.argmax(-1).tolist()
    assert dec.positions.tolist() == [9, 5, 13]
    tol = dict(rtol=0.13, atol=1e-2) if kv_dtype else dict(rtol=1e-5, atol=1e-5)   # e4m3: one rounding step
    for li in range(len(dec.layers)):
        for got, ref_kv in zip(dec._cached(li, torch.float32), ref._cached(li, torch.float32)):
            for b, p in enumerate(prompts):
                torch.testing.assert_close(got[b, :, :p.numel()], ref_kv[b, :, :p.numel()], **tol)
    # row 1's second token: the decode step of the padded decoder from the same cache
    ref.max_new = 0
    ref.positions.copy_(torch.tensor([9, 4, 13]))
    ref.step(torch.tensor([0, int(dec.generated[1, 0]), 0]))
    assert int(dec.generated[1, 1]) == int(ref.logits[1].argmax())


# ---- argument errors, before any work

def test_argument_errors_are_raised_before_any_work(monkeypatch):
    def no_decoder(*a, **k):
        raise AssertionError('work started')
    import quip_b200.decode as D
    monkeypatch.setattr(D, 'ContinuousDecoder', no_decoder)
    monkeypatch.setattr(D, 'PromptDecoder', no_decoder)
    m = _model('llama_gqa')
    p = _prompts()
    cases = ((dict(max_batch_size=2, prompt_lookup_num_tokens=2), 'prompt_lookup'),
             (dict(max_batch_size=2, share_prompt_prefixes=True), 'share'),
             (dict(max_batch_size=2, num_return_sequences=2, do_sample=True), 'num_return'),
             (dict(max_batch_size=0), '>= 1'), (dict(max_batch_size=True), '>= 1'), (dict(max_batch_size=1.5), '>= 1'),
             (dict(kv_pages=4), 'max_batch_size'), (dict(max_batch_size=2, kv_pages=0), 'kv_pages'),
             (dict(max_batch_size=2, prefill_chunk_size=0), 'chunk'))
    for kw, msg in cases:
        with pytest.raises(ValueError, match=msg):
            generate(m, p, 5, **kw)
    with pytest.raises(ValueError, match='pages'):                             # 11 + 60 tokens need 2 pages
        generate(m, p, 60, max_batch_size=2, kv_pages=1)
    with pytest.raises(ValueError, match='max_new_tokens'):
        generate(m, p, [5, 5], max_batch_size=2)
    with pytest.raises(ValueError, match='at least 1'):
        generate(m, p, [5, 0, 5], max_batch_size=2)


def test_ragged_wrappers_check_their_arguments_before_any_launch(monkeypatch):
    from quip_b200 import fused
    monkeypatch.setattr(_lib, 'load', lambda: (_ for _ in ()).throw(AssertionError('launched')))
    for bad in ([0], [1, 2], [0, 3, 2], [0, 1.5]):
        with pytest.raises(ValueError, match='seq_start'):
            fused.RaggedChunk(bad, 'cpu')
    seqs = fused.RaggedChunk([0, 1, 4], 'cpu')
    assert (seqs.S, seqs.N, seqs.max_count) == (2, 4, 3)
    pool = torch.zeros(3, 2, KV_PAGE, 64, dtype=torch.float16)
    pos = torch.zeros(2, dtype=torch.long)
    tbl = torch.zeros(2, 1, dtype=torch.int32)
    k = torch.zeros(4, 2, 64, dtype=torch.float16)
    q = torch.zeros(4, 4, 64, dtype=torch.float16)
    with pytest.raises(ValueError, match='RaggedChunk'):
        fused.kv_append_ragged(k, k, pool, pool, [0, 1, 4], pos, tbl)
    with pytest.raises(ValueError, match='paged only'):
        fused.prefill_attention_ragged(q, pool, pool, seqs, pos, None, 1.0)
    with pytest.raises(ValueError, match='page_table'):
        fused.kv_append_ragged(k, k, pool, pool, seqs, pos, tbl[:1])
    with pytest.raises(ValueError, match='positions'):
        fused.kv_append_ragged(k, k, pool, pool, seqs, pos[:1], tbl)
    with pytest.raises(ValueError, match='k_scale'):
        fused.kv_append_ragged(k, k, pool.to(torch.float8_e4m3fn), pool.to(torch.float8_e4m3fn), seqs, pos, tbl)
    with pytest.raises(ValueError, match='CUDA'):
        fused.prefill_attention_ragged(q, pool, pool, seqs, pos, tbl, 1.0)            # CPU tensors: never launched
