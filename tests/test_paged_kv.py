"""Paged KV cache (PromptDecoder(n_pages=...), plan_prefix_pages, generate(share_prompt_prefixes=...,
num_return_sequences=...)) on the tiny fp32 HF models of test_generate on the CPU, where reads gather pool[page_table]
into the contiguous view and writes go through the same page translation."""
import random

import pytest
import torch

from quip_b200 import _lib
from quip_b200.decode import KV_PAGE, PromptDecoder, SpecDecoder, generate, plan_prefix_pages
from test_generate import KINDS, _model, _prompts


def _plan(prompts, extra=8):
    return plan_prefix_pages(prompts, [len(p) + extra for p in prompts])


def _seq(n, seed=0):
    g = random.Random(seed)
    return [g.randrange(3, 199) for _ in range(n)]


# ---- the plan on named cases

def test_plan_identical_prompts_share_every_full_page_but_the_last_token_one():
    p = _seq(200)                                  # pages 0, 1, 2 shareable (192 <= 199); page 3 holds token 199
    table, n, starts = _plan([p, p, p])
    assert starts == [0, 192, 192]
    assert table[1, :3].tolist() == table[0, :3].tolist() == table[2, :3].tolist() == [0, 1, 2]
    own = [set(table[r, 3:].tolist()) for r in range(3)]
    assert not own[0] & own[1] and not own[1] & own[2] and not own[0] & own[2]
    assert n == 3 + 3 * 1                          # ceil(208 / 64) = 4 pages per row, 3 of them shared


def test_plan_prompts_differing_inside_page_0_share_nothing():
    a = _seq(300)
    b = list(a)
    b[10] += 1
    table, n, starts = _plan([a, b])
    assert starts == [0, 0] and n == 2 * 5 and not set(table[0].tolist()) & set(table[1].tolist())


def test_plan_difference_at_a_page_boundary_and_in_the_last_token_of_a_full_page():
    a = _seq(300)
    at_boundary = list(a)
    at_boundary[128] += 1                          # first token of page 2: pages 0, 1 shared
    last_of_page = list(a)
    last_of_page[127] += 1                         # last token of page 1: page 0 shared only
    table, n, starts = _plan([a, at_boundary, last_of_page])
    assert starts == [0, 128, 64]
    assert table[1, :2].tolist() == [0, 1] and table[1, 2] not in table[0].tolist()
    assert table[2, 0] == 0 and table[2, 1] not in table[0].tolist() + table[1].tolist()
    assert n == 5 + 3 + 4


def test_plan_length_a_multiple_of_64_does_not_share_its_last_page():
    p = _seq(128)                                  # page 1 holds the last prompt token: 128 <= 127 fails
    table, n, starts = _plan([p, p])
    assert starts == [0, 64] and table[1, 0] == 0 and table[1, 1] != table[0, 1]


def test_plan_one_token_prompts_share_nothing():
    table, n, starts = _plan([[5], [5], [5]], extra=1)
    assert starts == [0, 0, 0] and n == 3 and table[:, 0].tolist() == [0, 1, 2]


def test_plan_a_broken_shared_run_does_not_resume():
    a = _seq(400)
    b = list(a)
    b[70] += 1                                     # differs on page 1, equal again on pages 2..
    table, n, starts = _plan([a, b])
    assert starts == [0, 64] and table[1, 0] == 0
    assert not set(table[1, 1:].tolist()) & set(table[0].tolist())


def test_plan_leaves_unneeded_entries_unmapped_and_checks_budgets():
    table, n, starts = plan_prefix_pages([_seq(10), _seq(100)], [20, 200], max_pages=6)
    assert table.shape == (2, 6) and table.dtype == torch.int32
    assert table[0].tolist() == [0, -1, -1, -1, -1, -1] and table[1, :4].tolist() == [1, 2, 3, 4]
    with pytest.raises(ValueError, match='budget'):
        plan_prefix_pages([_seq(10)], [9])
    with pytest.raises(ValueError, match='max_pages'):
        plan_prefix_pages([_seq(10)], [200], max_pages=3)


@pytest.mark.parametrize('seed', range(8))
def test_plan_invariants_on_random_prompt_sets(seed):
    g = random.Random(seed)
    base = [_seq(g.randrange(1, 400), seed=100 + i) for i in range(3)]
    prompts, budgets = [], []
    for _ in range(g.randrange(1, 9)):
        p = list(base[g.randrange(3)])[:g.randrange(1, 400)] or [7]
        if g.random() < 0.4 and len(p) > 1:
            p[g.randrange(len(p))] += 1
        prompts.append(p)
        budgets.append(len(p) + g.randrange(0, 130))
    table, n, starts = plan_prefix_pages(prompts, budgets)
    B = len(prompts)
    used = set()
    owner_of = {}                                  # page id -> (row, page index) of its first mapping
    for r, p in enumerate(prompts):
        need = -(-budgets[r] // KV_PAGE)
        row = table[r].tolist()
        assert all(x >= 0 for x in row[:need]) and all(x == -1 for x in row[need:])
        S = starts[r] // KV_PAGE
        for q in range(need):
            pid = row[q]
            used.add(pid)
            if pid not in owner_of:
                owner_of[pid] = (r, q)
                continue
            r0, q0 = owner_of[pid]
            assert q < S and q == q0 and r0 < r                            # shared: leading run, same page index
            assert KV_PAGE * (q + 1) <= len(p) - 1 and KV_PAGE * (q + 1) <= len(prompts[r0]) - 1
            assert p[:KV_PAGE * (q + 1)] == prompts[r0][:KV_PAGE * (q + 1)]
        for q in range(S):
            assert owner_of[row[q]][0] != r                                # the leading run is shared
        if S < need and KV_PAGE * (S + 1) <= len(p) - 1:                  # the next shareable page has no earlier twin
            assert not any(KV_PAGE * (S + 1) <= len(prompts[r0]) - 1 and
                           prompts[r0][:KV_PAGE * (S + 1)] == p[:KV_PAGE * (S + 1)] for r0 in range(r))
    assert used == set(range(n)) and B == len(starts)


# ---- a paged decoder without sharing is the contiguous decoder

def _perm_table(B, max_len, seed):
    mp = -(-max_len // KV_PAGE)
    g = torch.Generator().manual_seed(seed)
    return torch.randperm(B * mp, generator=g).to(torch.int32).view(B, mp), B * mp


def _run(dec, prompts, steps, chunk):
    out = [dec.prefill(prompts, chunk=chunk).clone()]
    for _ in range(steps):
        out.append(dec.step().clone())
    return out, dec.generated.clone()


@pytest.mark.parametrize('mode', ['greedy', 'sample', 'spec'])
@pytest.mark.parametrize('kv', ['fp16', 'e4m3'])
@pytest.mark.parametrize('kind', KINDS)
def test_paged_decoder_on_shuffled_pages_equals_contiguous_bit_for_bit(kind, kv, mode):
    m = _model(kind)
    prompts = _prompts(seed=9, lens=(5, 11, 2))
    max_len = 30
    table, n = _perm_table(3, max_len, seed=len(kind) + len(mode))
    kw = dict(max_len=max_len, batch=3, max_new=8, kv_dtype=torch.float8_e4m3fn if kv == 'e4m3' else None,
              sampling=mode == 'sample')
    runs = []
    for pages in ({}, dict(page_table=table, n_pages=n)):
        dec = SpecDecoder(m, draft_tokens=3, **kw, **pages) if mode == 'spec' else PromptDecoder(m, **kw, **pages)
        if mode == 'sample':
            dec.set_sampling(temperature=0.8, top_k=30, seed=[4, 5, 6])
        runs.append(_run(dec, prompts, 5, chunk=4))
        if pages:
            assert dec.k_cache.shape[1:3] == (n, dec.nkv) and dec.k_cache.shape[3] == KV_PAGE
    (la, ga), (lb, gb) = runs
    assert all(torch.equal(x, y) for x, y in zip(la, lb))
    assert torch.equal(ga, gb)


def test_paged_cache_reads_back_through_the_table_and_reset_unmaps():
    m = _model('llama_gqa')
    prompts = _prompts(seed=3, lens=(5, 11, 2))
    table, n = _perm_table(3, 20, seed=1)
    a = PromptDecoder(m, max_len=20, batch=3)
    b = PromptDecoder(m, max_len=20, batch=3, page_table=table, n_pages=n)
    assert (b.page_table == -1).all()
    a.prefill(prompts, chunk=3)
    b.prefill(prompts, chunk=3)
    assert torch.equal(b.page_table.cpu(), table)
    for li in range(len(a.layers)):
        kb, vb = b._cached(li, torch.float32)
        for r, p in enumerate(prompts):
            assert torch.equal(kb[r, :, :p.numel()], a.k_cache[li, r, :, :p.numel()])
            assert torch.equal(vb[r, :, :p.numel()], a.v_cache[li, r, :, :p.numel()])
    b.reset()
    assert (b.page_table == -1).all() and not b.k_cache.any()


# ---- generate with shared prefixes and several samples

def _shared_prompts(n_shared_pages, seed):
    """Llama prompts (no learned-position limit) sharing n_shared_pages full pages: lengths past the shared run."""
    g = torch.Generator().manual_seed(seed)
    pre = torch.randint(3, 199, (KV_PAGE * n_shared_pages,), generator=g)
    return [torch.cat((pre, torch.randint(3, 199, (n,), generator=g))) for n in (7, 30, 70)]


@pytest.mark.parametrize('n_shared', [0, 1, 3])
@pytest.mark.parametrize('kind', ['llama_mha', 'llama_gqa'])
def test_generate_sharing_prefixes_equals_generate(kind, n_shared):
    m = _model(kind)
    prompts = _shared_prompts(n_shared, seed=n_shared)
    lens = [len(p) for p in prompts]
    _, _, starts = _plan(prompts, extra=6)
    assert starts[0] == 0 and starts[1] == starts[2] == KV_PAGE * n_shared
    want = generate(m, prompts, 6)
    for C in (32, 100):
        got = generate(m, prompts, 6, share_prompt_prefixes=True, prefill_chunk_size=C)
        assert all(torch.equal(g, w) for g, w in zip(got, want)), (C, lens)


@pytest.mark.parametrize('kind', KINDS)
def test_generate_sharing_without_full_pages_equals_generate(kind):
    m = _model(kind)
    prompts = _prompts(seed=5, lens=(5, 11, 2))
    want = generate(m, prompts, 10)
    got = generate(m, prompts, 10, share_prompt_prefixes=True)
    assert all(torch.equal(g, w) for g, w in zip(got, want))


@pytest.mark.parametrize('kw', [dict(eos_token_id=None), dict(kv_dtype=torch.float8_e4m3fn),
                                dict(prompt_lookup_num_tokens=3), dict(top_k=20, seed=[1, 2, 3, 4, 5, 6])])
def test_num_return_sequences_is_the_repeated_prompt_call(kw):
    m = _model('llama_gqa')
    prompts = _shared_prompts(2, seed=7)[:2]
    n = 3
    kw = dict(do_sample=True, temperature=0.9, **kw)
    if 'seed' in kw:
        prompts = prompts[:1] + [prompts[1][:40]]
    if 'eos_token_id' in kw:
        free = generate(m, prompts, 8, do_sample=True, temperature=0.9)
        kw['eos_token_id'] = int(free[0][2])
    got = generate(m, prompts, 8, num_return_sequences=n, **kw)
    want = generate(m, [p for p in prompts for _ in range(n)], 8, share_prompt_prefixes=True, **kw)
    assert len(got) == len(prompts) * n
    assert all(torch.equal(g, w) for g, w in zip(got, want))
    if 'seed' not in kw or not isinstance(kw['seed'], list):
        assert not all(torch.equal(got[0], got[i]) for i in range(1, n))   # different seeds, different samples


# ---- argument errors before any work

def test_argument_errors_are_raised_before_any_work(monkeypatch):
    m = _model('llama_mha')
    p = _prompts()[0]

    def boom(*a, **k):
        raise AssertionError('work started')
    monkeypatch.setattr(PromptDecoder, 'prefill', boom)
    with pytest.raises(ValueError, match='do_sample'):
        generate(m, [p], 3, num_return_sequences=2)
    for bad in (0, -1, 1.5, True):
        with pytest.raises(ValueError, match='num_return_sequences'):
            generate(m, [p], 3, num_return_sequences=bad, do_sample=True)
    with pytest.raises(ValueError, match='seed: 2 values for 4 prompts'):
        generate(m, [p, p], 3, num_return_sequences=2, do_sample=True, seed=[1, 2])
    with pytest.raises(ValueError, match='temperature'):
        generate(m, [p], 3, num_return_sequences=2, do_sample=True, temperature=[1.0])
    monkeypatch.undo()
    dec = PromptDecoder(m, max_len=8, batch=1, n_pages=1)
    with pytest.raises(ValueError, match='chunked prefill'):
        dec.prefill([p])
    assert (dec.page_table == -1).all()
    with pytest.raises(ValueError, match='starts'):
        PromptDecoder(m, max_len=80, batch=1, n_pages=2).prefill([torch.arange(3, 73)], chunk=8, starts=[32])
    with pytest.raises(ValueError, match='paged'):
        PromptDecoder(m, max_len=80, batch=1).prefill([torch.arange(3, 73)], chunk=8, starts=[64])
    with pytest.raises(ValueError, match='page ids'):
        PromptDecoder(m, max_len=8, batch=1, page_table=[[3]], n_pages=2)
    with pytest.raises(ValueError, match=r'page_table must be \(batch'):
        PromptDecoder(m, max_len=8, batch=1, page_table=[[0, 1]], n_pages=2)
    with pytest.raises(ValueError, match='n_pages'):
        PromptDecoder(m, max_len=8, batch=1, page_table=[[0]])


def test_cache_descriptors_check_their_page_table_before_any_launch():
    lib = _lib.load()
    buf, ws = 64, 1 << 20
    B, nh, nkv, hd = 2, 8, 2, 128
    for table, mp, n, what in ((None, 4, 8, 'page_table'), (buf + 2, 4, 8, 'page_table'), (buf, 0, 8, 'max_pages'),
                               (buf, 1 << 26, 8, 'max_pages'), (buf, 4, 0, 'n_pages')):
        def kv(fp8):
            return _lib.QuipKvCache(k=buf, v=buf, k_scale=buf if fp8 else None, v_scale=buf if fp8 else None,
                                    format=_lib.QUIP_KV_E4M3 if fp8 else _lib.QUIP_KV_FP16, nkv=nkv, hd=hd,
                                    page_table=table, max_pages=mp, n_pages=n)
        # ragged launches and the fork are paged only: a null table is refused; elsewhere it means contiguous
        calls = {'quip_kv_append_ragged': lambda: lib.quip_kv_append_ragged(kv(False), buf, buf, buf, buf, B, 4, 2, None),
                 'quip_prefill_attention_ragged':
                     lambda: lib.quip_prefill_attention_ragged(kv(True), buf, buf, buf, buf, B, 4, 2, nh, 1.0, None),
                 'quip_kv_beam_fork': lambda: lib.quip_kv_beam_fork(kv(True), 1, buf, buf, buf, B, 0, None)}
        if table is not None:
            calls.update({
                'quip_decode_attention':
                    lambda: lib.quip_decode_attention(kv(False), buf, buf, buf, buf, buf, B, nh, 1.0, buf, ws, None),
                'quip_extend_attention':
                    lambda: lib.quip_extend_attention(kv(True), buf, buf, buf, buf, buf, B, 2, nh, 1.0, buf, ws, None),
                'quip_kv_append': lambda: lib.quip_kv_append(kv(False), buf, buf, buf, buf, B, 2, None),
                'quip_prefill_attention':
                    lambda: lib.quip_prefill_attention(kv(True), buf, buf, buf, buf, B, 2, nh, 1.0, None)})
        for fn, call in calls.items():
            assert call() != 0
            msg = lib.quip_last_error().decode()
            assert msg.startswith(fn + ':') and 'page_table' in msg, (what, msg)
