"""The prefix cache of continuous batching (generate(..., max_batch_size=n, prefix_cache=True), ContinuousSchedule with
prompts): the schedule's invariants on random workloads whose prompts share heads at page boundaries, hand-built
admission, readiness and eviction cases, and generate() against the cache off and each prompt alone on the tiny fp32 HF
models of test_generate on the CPU."""
import random

import pytest
import torch

from quip_b200.constrain import TokenAutomaton
from quip_b200.decode import KV_PAGE, ContinuousSchedule, generate, plan_prefix_pages, shareable_pages
from test_generate import KINDS, _model, _prompts


# ---- the schedule on its own

def _check_pool(s, n_pages):
    held = [r for r, i in enumerate(s.req) if i is not None]
    maps = {}
    for r in held:
        assert len(set(s.pages[r])) == len(s.pages[r])
        for p in s.pages[r]:
            maps[p] = maps.get(p, 0) + 1
    for p in range(n_pages):
        assert s.ref[p] == maps.get(p, 0), p                                   # a count is the rows that map it
    owned = [p for r in held for p in s.pages[r][s.shared[s.req[r]]:]]
    assert len(owned) == len(set(owned))                                       # no page owned twice
    free, cached, mapped = set(s.free_pages), set(s.cached), set(maps)
    assert len(free) == len(s.free_pages)
    assert not free & cached and not free & mapped and not cached & mapped
    assert len(free) + len(cached) + len(mapped) == n_pages
    assert all(p in s.entry for p in cached)
    for r in held:                                                             # a shared page is still indexed
        assert all(p in s.entry for p in s.pages[r][:s.shared[s.req[r]]])


def _simulate(prompts, max_new, rows, n_pages, chunk, stop, check_every=1):
    """Drive a prefix-cached ContinuousSchedule as generate() does, with request i finishing after stop[i] tokens, and
    check the invariants after every admission and step, against the test's own record of which pages hold which
    prefix and which have been written.  Returns the admission order and the schedule."""
    lens = [len(p) for p in prompts]
    s = ContinuousSchedule(lens, max_new, rows, n_pages, chunk, prompts=prompts)
    need = [-(-(n + m) // KV_PAGE) for n, m in zip(lens, max_new)]
    content, written = {}, set()                                               # page -> prefix it holds; pages written
    n_gen, order, steps = {}, [], 0
    while True:
        if s.queue or steps % check_every == 0:
            for r, i in enumerate(s.req):
                if i is not None and n_gen.get(r, 0) >= stop[i]:
                    assert s.retire(r) == i
                    n_gen.pop(r)
            for r, i, pages in s.admit():
                S = s.shared[i]
                assert pages == s.pages[r] and len(pages) == need[i] and S <= shareable_pages(lens[i])
                assert s.fed[r] == KV_PAGE * S
                for j in range(S):                                             # the shared pages hold this prefix
                    assert content[pages[j]] == tuple(prompts[i][:KV_PAGE * (j + 1)]), (i, j)
                for j, p in enumerate(pages[S:], S):
                    written.discard(p)
                    content.pop(p, None)
                    if j < shareable_pages(lens[i]):
                        content[p] = tuple(prompts[i][:KV_PAGE * (j + 1)])
                order.append(i)
            _check_pool(s, n_pages)
        if s.finished:
            break
        filling = list(s.filling)
        decoding, pieces = s.plan()
        assert not filling or pieces                                           # a filling step always has a piece
        assert sum(n for _, _, n in pieces) <= chunk
        assert [r for r, _, _ in pieces] == [r for r in filling if r in {q for q, _, _ in pieces}]
        for r, lo, n in pieces:
            i = s.req[r]
            assert all(p in written for p in s.pages[r][:s.shared[i]]), (r, i)  # never before its shared pages
            for j in range(s.shared[i], shareable_pages(lens[i])):
                if KV_PAGE * (j + 1) <= lo + n:
                    written.add(s.pages[r][j])
            if lo + n == lens[i]:
                n_gen[r] = 1
        for r in decoding:
            n_gen[r] = n_gen.get(r, 0) + (n_gen.get(r, 0) < stop[s.req[r]])
        steps += 1
    assert sorted(s.free_pages + list(s.cached)) == list(range(n_pages)) and not any(s.ref)
    assert s.prefilled == sum(n - KV_PAGE * S for n, S in zip(lens, s.shared))
    return order, s


def _shared_heads(g, n, V=4):
    """n prompts cut from a few random heads at random page boundaries, plus random tails (a small vocabulary, so
    tails collide too); some repeat an earlier prompt."""
    heads = [[g.randrange(V) for _ in range(6 * KV_PAGE)] for _ in range(3)]
    out = []
    for _ in range(n):
        if out and g.random() < 0.2:
            out.append(list(g.choice(out)))
            continue
        k = g.randrange(0, 6)
        out.append(g.choice(heads)[:KV_PAGE * k] + [g.randrange(V) for _ in range(g.randrange(0 if k else 1, 150))])
    return out


@pytest.mark.parametrize('seed', range(16))
def test_schedule_invariants_on_random_workloads_with_shared_heads(seed):
    g = random.Random(seed)
    n = g.randrange(1, 40)
    prompts = _shared_heads(g, n)
    max_new = [g.randrange(1, 200) for _ in range(n)]
    stop = [g.randrange(1, m + 1) for m in max_new]
    need = max(-(-(len(a) + b) // KV_PAGE) for a, b in zip(prompts, max_new))
    rows = g.randrange(1, 9)
    n_pages = g.randrange(need, need * (rows + 1) + 1)
    order, s = _simulate(prompts, max_new, rows, n_pages, g.choice([1, 7, 64, 512]), stop,
                         check_every=g.choice([1, 16]))
    assert order == list(range(n))                                             # FIFO


def test_random_workloads_share_pages():
    """The random workloads above do reuse pages, so the invariants are checked where they bite."""
    g = random.Random(100)
    prompts = _shared_heads(g, 30)
    _, s = _simulate(prompts, [20] * 30, 4, 4 * 12, 64, [20] * 30)
    assert sum(s.shared) > 10 and s.prefilled < sum(map(len, prompts))


def test_identical_prompts_admitted_together_follow_the_owner_in_the_same_step():
    p = list(range(200))                                                       # 3 shareable pages
    s = ContinuousSchedule([200, 200], [8, 8], rows=2, n_pages=8, chunk=130, prompts=[p, p])
    (r0, _, a), (r1, _, b) = s.admit()
    assert s.shared == [0, 3] and b[:3] == a[:3] and not set(b[3:]) & set(a)
    assert s.ref[a[0]] == 2 and s.ref[a[3]] == 1
    assert s.plan() == ([], [(r0, 0, 130)])                                    # page 2 not written: row 1 waits
    assert s.plan() == ([], [(r0, 130, 70), (r1, 192, 8)])                     # its owner writes it in this step
    assert s.prefilled == 208 and s.filling == []


def test_a_finished_requests_pages_serve_a_later_one():
    head = list(range(128))
    s = ContinuousSchedule([150, 140], [10, 10], rows=1, n_pages=3, chunk=512,
                           prompts=[head + [1] * 22, head + [2] * 12])
    (_, _, a), = s.admit()
    assert s.plan() == ([], [(0, 0, 150)])
    assert s.admit() == []                                                     # no free row
    s.retire(0)
    assert sorted(s.cached) == a[:2] and s.free_pages == [a[2]]
    (_, _, b), = s.admit()
    assert b == a[:2] + [a[2]] and s.shared == [0, 2]
    assert s.plan() == ([], [(0, 128, 12)])
    assert s.prefilled == 150 + 12


def test_eviction_takes_the_least_recently_released_leaf_first():
    g = torch.Generator().manual_seed(0)
    A, B, C, D = (torch.randint(0, 1000, (n,), generator=g).tolist() for n in (130, 130, 300, 70))
    s = ContinuousSchedule([130, 130, 300, 70], [10, 10, 20, 10], rows=2, n_pages=8, chunk=512, prompts=[A, B, C, D])
    assert [p for _, _, p in s.admit()] == [[0, 1, 2], [3, 4, 5]]
    s.plan()
    s.retire(1)                                                                # B's chain 3 -> 4 released first
    s.retire(0)                                                                # then A's 0 -> 1
    assert s.cached == {0, 1, 3, 4} and s.free_pages == [2, 5, 6, 7]
    (_, _, c), (_, _, d) = s.admit()
    assert c == [2, 5, 6, 7, 4]                                    # C: 4 free pages, then B's leaf, not its root 3
    assert d == [3, 1]                                             # D: nothing free; B's root, then A's leaf, not 0
    assert s.cached == {0} and s.shared == [0, 0, 0, 0]


def test_waits_for_pages_when_the_evictable_ones_are_its_own_match():
    g = torch.Generator().manual_seed(1)
    A, X = torch.randint(0, 1000, (130,), generator=g).tolist(), [5] * 10
    Bp = A[:128] + torch.randint(0, 1000, (72,), generator=g).tolist()
    s = ContinuousSchedule([130, 10, 200], [10, 10, 100], rows=2, n_pages=5, chunk=512, prompts=[A, X, Bp])
    assert [p for _, _, p in s.admit()] == [[0, 1, 2], [3]]
    s.plan()
    s.retire(0)
    assert s.cached == {0, 1} and s.free_pages == [2, 4]
    assert s.admit() == []                                     # needs 3 own pages: 2 free, its 2 cached ones matched
    assert list(s.queue) == [2] and s.free_rows == [0]
    s.retire(1)
    (_, _, b), = s.admit()
    assert b == [0, 1, 2, 3, 4] and s.shared[2] == 2 and s.fed[0] == 128


def test_a_prompt_of_whole_pages_keeps_its_last_page_and_one_token_shares_nothing():
    p = list(range(128))
    s = ContinuousSchedule([128, 128, 1, 1], [4, 4, 4, 4], rows=4, n_pages=8, chunk=512, prompts=[p, p, [7], [7]])
    got = s.admit()
    assert s.shared == [0, 1, 0, 0]
    a, b = got[0][2], got[1][2]
    assert b[0] == a[0] and b[1] != a[1]                       # the last token's page is its own
    assert not set(got[2][2]) & set(got[3][2])
    assert s.plan() == ([], [(0, 0, 128), (1, 64, 64), (2, 0, 1), (3, 0, 1)])
    assert s.prefilled == 128 + 64 + 2


def test_without_prompts_the_schedule_is_unchanged():
    s = ContinuousSchedule([100, 10, 10], [28, 5, 5], rows=3, n_pages=3, chunk=512)
    assert [(r, i, p) for r, i, p in s.admit()] == [(0, 0, [0, 1]), (1, 1, [2])]
    assert s.plan() == ([], [(0, 0, 100), (1, 0, 10)]) and s.prefilled == 110 and s.shared == [0, 0, 0]
    with pytest.raises(ValueError, match='lengths'):
        ContinuousSchedule([3, 4], [2, 2], rows=2, n_pages=4, chunk=8, prompts=[[1, 2, 3], [1, 2]])


def test_plan_prefix_pages_and_the_cache_share_the_same_pages():
    g = random.Random(3)
    prompts = _shared_heads(g, 12)
    table, _, starts = plan_prefix_pages(prompts, [len(p) + 5 for p in prompts])
    s = ContinuousSchedule([len(p) for p in prompts], [5] * 12, rows=12, n_pages=12 * 9, chunk=64, prompts=prompts)
    s.admit()
    assert [KV_PAGE * S for S in s.shared] == starts


# ---- generate(max_batch_size=..., prefix_cache=True) against the cache off and each prompt alone

def _workload(seed=5):
    """Prompts longer than a page with shared heads: a repeat, a head of two pages, one of one page, a prompt whose
    last token starts a page, and one of its own."""
    head, tails = _prompts(seed=seed, lens=(200,))[0], _prompts(seed=seed + 1, lens=(5, 11, 7, 3, 9))
    prompts = [torch.cat((head[:140], tails[0])), torch.cat((head[:130], tails[1])), torch.cat((head[:140], tails[0])),
               tails[2], torch.cat((head[:64], tails[3])), head[:129], torch.cat((head[:70], tails[4]))]
    return prompts, [9, 4, 12, 6, 7, 3, 5]


def _alone(m, prompts, budgets, C, kw):
    out, lps = [], []
    for i, (p, k) in enumerate(zip(prompts, budgets)):
        one = {a: (v[i:i + 1] if isinstance(v, list) and a != 'bad_words_ids' else v) for a, v in kw.items()}
        if 'seed' in one:
            one['seed'] = one['seed'] + i
        lp = {} if 'logprobs' in kw else None
        if lp is not None:
            one['logprobs'] = lp
        out.append(generate(m, [p], k, prefill_chunk_size=C, **one)[0])
        lps.append(lp)
    return out, lps


@pytest.mark.parametrize('mode', ['greedy', 'sampled'])
@pytest.mark.parametrize('kv', ['fp32', 'e4m3'])
@pytest.mark.parametrize('kind', ['llama_mha', 'llama_gqa'])
def test_prefix_cache_equals_the_cache_off_and_each_prompt_alone(kind, kv, mode):
    m = _model(kind)
    prompts, budgets = _workload()
    kw = dict(kv_dtype=torch.float8_e4m3fn) if kv == 'e4m3' else {}
    if mode == 'sampled':
        kw.update(do_sample=True, temperature=0.8, top_k=40, seed=11)
    for C in (1, 7, 64):
        want, _ = _alone(m, prompts, budgets, C, kw)
        for B in (1, 2, 3, len(prompts)):
            off = generate(m, prompts, budgets, max_batch_size=B, prefill_chunk_size=C, **kw)
            on = generate(m, prompts, budgets, max_batch_size=B, prefill_chunk_size=C, prefix_cache=True, **kw)
            for i, (a, b, w) in enumerate(zip(on, off, want)):
                assert torch.equal(a, w) and torch.equal(b, w), (B, C, i, a, b, w)


def test_prefix_cache_shares_and_counts_the_prompt_tokens_it_prefills(monkeypatch):
    import quip_b200.decode as D
    made = []

    class Spy(D.ContinuousSchedule):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            made.append(self)

    monkeypatch.setattr(D, 'ContinuousSchedule', Spy)
    m = _model('llama_gqa')
    prompts, budgets = _workload()
    lens = [p.numel() for p in prompts]
    generate(m, prompts, budgets, max_batch_size=3, prefill_chunk_size=7, prefix_cache=True)
    generate(m, prompts, budgets, max_batch_size=3, prefill_chunk_size=7)
    on, off = made
    assert on.shared == [0, 2, 2, 0, 1, 2, 1]
    assert on.prefilled == sum(n - KV_PAGE * S for n, S in zip(lens, on.shared)) < off.prefilled == sum(lens)
    assert off.tokens is None and off.shared == [0] * len(prompts)


@pytest.mark.parametrize('kv', ['fp32', 'e4m3'])
def test_prefix_cache_with_processors_constraint_and_logprobs(kv):
    m = _model('llama_mha')
    prompts, budgets = _workload(seed=8)
    a = TokenAutomaton.from_sequences([[10, 11, 12], [10, 20], [30], [40, 41, 42, 43]], 7)
    n = len(prompts)
    kw = dict(repetition_penalty=[1.5, 1.0, 2.0, 1.2, 1.0, 1.3, 1.1], no_repeat_ngram_size=2, bad_words_ids=[[4, 5]],
              token_constraint=[a, None, a, None, None, a, None], eos_token_id=7, top_logprobs=3,
              kv_dtype=torch.float8_e4m3fn if kv == 'e4m3' else None)
    want, want_lp = _alone(m, prompts, budgets, 7, dict(kw, logprobs={}))
    for B in (2, n):
        runs = []
        for cache in (False, True):
            lp = {}
            runs.append((generate(m, prompts, budgets, max_batch_size=B, prefill_chunk_size=7, prefix_cache=cache,
                                  logprobs=lp, **kw), lp))
        for got, lp in runs:                  # logprobs: the log_softmax of other row counts rounds apart, cache or not
            for i in range(n):
                assert torch.equal(got[i], want[i]), (B, i, got[i], want[i])
                assert torch.equal(lp['top_ids'][i], want_lp[i]['top_ids'][0]), (B, i)
                for key in ('token', 'top'):
                    assert lp[key][i].shape == want_lp[i][key][0].shape
                    assert float((lp[key][i] - want_lp[i][key][0]).abs().max()) <= 1e-5, (B, i, key)


@pytest.mark.parametrize('kind', ['opt_pre_ln', 'opt_post_ln'])
def test_prefix_cache_is_a_no_op_on_models_too_short_for_a_shareable_page(kind, monkeypatch):
    import quip_b200.decode as D
    made = []

    class Spy(D.ContinuousSchedule):
        def __init__(self, *a, **k):
            super().__init__(*a, **k)
            made.append(self)

    monkeypatch.setattr(D, 'ContinuousSchedule', Spy)
    m = _model(kind)
    p = _prompts(seed=3, lens=(30,))[0]
    prompts = [p, p, p[:20], _prompts(seed=4, lens=(9,))[0]]
    budgets = [6, 9, 4, 7]
    for kw in ({}, dict(do_sample=True, seed=2)):
        on = generate(m, prompts, budgets, max_batch_size=2, prefill_chunk_size=7, prefix_cache=True, **kw)
        off = generate(m, prompts, budgets, max_batch_size=2, prefill_chunk_size=7, **kw)
        assert all(torch.equal(a, b) for a, b in zip(on, off))
    assert all(S == 0 for s in made for S in s.shared)


def test_prefix_cache_argument_errors_are_raised_before_any_work(monkeypatch):
    def no_decoder(*a, **k):
        raise AssertionError('work started')
    import quip_b200.decode as D
    monkeypatch.setattr(D, 'ContinuousDecoder', no_decoder)
    monkeypatch.setattr(D, 'PromptDecoder', no_decoder)
    m = _model('llama_gqa')
    p = _prompts()
    for kw, msg in ((dict(prefix_cache=True), 'max_batch_size'), (dict(prefix_cache=1, max_batch_size=2), 'True or False'),
                    (dict(prefix_cache='yes', max_batch_size=2), 'True or False'),
                    (dict(prefix_cache=None), 'True or False'),
                    (dict(prefix_cache=True, max_batch_size=2, share_prompt_prefixes=True), 'share'),
                    (dict(prefix_cache=True, max_batch_size=2, num_return_sequences=2, do_sample=True), 'num_return'),
                    (dict(prefix_cache=True, max_batch_size=2, prompt_lookup_num_tokens=2), 'prompt_lookup')):
        with pytest.raises(ValueError, match=msg):
            generate(m, p, 5, **kw)
