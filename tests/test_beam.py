"""Beam search (generate(..., num_beams=K): BeamDecoder and the torch restatements of csrc/beam.cu's rules) on the tiny
fp32 HF models of test_generate on the CPU, against HF's own beam search run one prompt at a time."""
import pytest
import torch

import quip_b200.decode as D
from oracle.beam import gathered
from quip_b200 import _lib
from quip_b200.decode import KV_PAGE, BeamDecoder, PromptDecoder, generate, plan_prefix_pages
from test_generate import KINDS, _model, _prompts


def _quiet(m):
    m.generation_config.eos_token_id = None             # HF would otherwise add the config's EOS id
    m.generation_config.pad_token_id = None
    return m


def _cut(row, eos):
    hit = [i for i, t in enumerate(row.tolist()) if t in eos]
    return row[:hit[0] + 1] if hit else row


def _hf(m, p, n, K, es, lp, r, eos):
    with torch.no_grad():
        out = m.generate(p[None], num_beams=K, do_sample=False, max_new_tokens=n, num_return_sequences=r,
                         early_stopping=es, length_penalty=lp, eos_token_id=eos, pad_token_id=0,
                         output_scores=True, return_dict_in_generate=True)
    seqs = [_cut(out.sequences[k, p.numel():], eos or []) for k in range(r)]
    return seqs, out.sequences_scores.tolist()


@pytest.mark.parametrize('K', [2, 3, 4])
@pytest.mark.parametrize('kind', KINDS)
def test_beam_search_equals_hf_for_each_prompt_alone(kind, K):
    m = _quiet(_model(kind))
    prompts = _prompts(seed=4, lens=(5, 11, 2))
    budgets = [9, 5, 7]
    free, = generate(m, [prompts[0]], 6, num_beams=K)
    eos = [int(free[2])]                                # the best hypothesis ends at its third token
    cases = [(es, lp) for es in (False, True, 'never') for lp in (0.0, 1.0, 2.0)]
    for c, (es, lp) in enumerate(cases):
        r = K if c % 2 else 1
        chunk = (1, 7, 64)[c % 3]
        use_eos = eos if c % 3 != 2 else None
        stats = {}
        got = generate(m, prompts, budgets, num_beams=K, early_stopping=es, length_penalty=lp,
                       num_return_sequences=r, eos_token_id=use_eos, prefill_chunk_size=chunk, beam_stats=stats)
        assert len(got) == len(prompts) * r and len(stats['scores']) == len(got)
        for i, (p, n) in enumerate(zip(prompts, budgets)):
            want, scores = _hf(m, p, n, K, es, lp, r, use_eos)
            for k in range(r):
                assert torch.equal(got[i * r + k], want[k]), (es, lp, i, k, got[i * r + k], want[k])
                assert abs(stats['scores'][i * r + k] - scores[k]) <= 1e-5, (es, lp, i, k)


def test_hypotheses_finish_mid_run_and_budgets_cut_each_prompt():
    m = _quiet(_model('llama_gqa'))
    prompts = _prompts(seed=4, lens=(5, 11, 2))
    free, = generate(m, [prompts[0]], 6, num_beams=3)
    got = generate(m, prompts, [9, 5, 7], num_beams=3, num_return_sequences=3, eos_token_id=int(free[2]))
    assert any(g.numel() and int(g[-1]) == int(free[2]) and g.numel() < 9 for g in got[:3])
    assert all(g.numel() <= n for g, n in zip(got, [9] * 3 + [5] * 3 + [7] * 3))


def test_num_beams_one_is_the_plain_call():
    m = _model('opt_pre_ln')
    prompts = _prompts()
    for kw in ({}, dict(prefill_chunk_size=5), dict(do_sample=True, seed=3, top_k=20)):
        a = generate(m, prompts, 7, **kw)
        b = generate(m, prompts, 7, num_beams=1, **kw)
        assert all(torch.equal(x, y) for x, y in zip(a, b)), kw


# ---- the fork

def _pools(L, N, nkv, hd, fp8, seed=0):
    g = torch.Generator().manual_seed(seed)
    k = torch.randn(L, N, nkv, KV_PAGE, hd, generator=g)
    v = torch.randn(L, N, nkv, KV_PAGE, hd, generator=g)
    if not fp8:
        return k, v, None, None
    ks = torch.rand(L, N, nkv, KV_PAGE, generator=g) + 0.5
    vs = torch.rand(L, N, nkv, KV_PAGE, generator=g) + 0.5
    return k.to(torch.float8_e4m3fn), v.to(torch.float8_e4m3fn), ks, vs


FORK_CASES = {'identity': [0, 1, 2, 3], 'one_parent': [2, 2, 2, 2], 'cycle': [1, 2, 3, 0], 'swap': [1, 0, 3, 3]}


@pytest.mark.parametrize('fp8', [False, True])
@pytest.mark.parametrize('slot', [0, 62, 63])
@pytest.mark.parametrize('case', list(FORK_CASES))
def test_fork_gives_each_row_its_parents_slots(case, slot, fp8):
    R, P, L = 4, 4, 2
    pos = 2 * KV_PAGE + slot                                   # the slot the step just wrote
    table = torch.tensor([[0, 1, 2 + r, 6 + r] for r in range(R)], dtype=torch.int32)   # 2 shared pages, then own
    k, v, ks, vs = _pools(L, 10 + R, 2, 16, fp8)
    parents = torch.tensor(FORK_CASES[case])
    lens = torch.full((R,), pos + 1)
    before = [gathered(x, table) for x in (k, v, ks, vs) if x is not None]
    untouched = [10 + r for r in range(R)] + [6 + r for r in range(R)]
    spare = [x[:, untouched].clone() for x in (k, v, ks, vs) if x is not None]
    tbl = table.clone()
    D._beam_fork_torch(k, v, tbl, parents, lens, ks, vs)
    after = [gathered(x, tbl) for x in (k, v, ks, vs) if x is not None]
    for b, a in zip(before, after):
        for r in range(R):
            assert torch.equal(a[r, :pos + 1], b[int(parents[r]), :pos + 1]), (case, r)
    for s, x in zip(spare, [x for x in (k, v, ks, vs) if x is not None]):
        assert torch.equal(s.float(), x[:, untouched].float())       # pages of later spans and scratch: untouched
    for r in range(R):
        assert tbl[r, 2] == table[r, 2] and tbl[r, 3] == table[r, 3]  # the current span and later stay the row's own


@pytest.mark.parametrize('kv', ['fp32', 'e4m3'])
def test_fork_invariant_after_every_step_of_a_run(kv, monkeypatch):
    m = _quiet(_model('llama_gqa'))
    seen = []
    orig = D._beam_fork_torch

    def spy(k, v, table, parents, lens, k_scale=None, v_scale=None):
        before = [gathered(x, table) for x in (k, v)]
        orig(k, v, table, parents, lens, k_scale, v_scale)
        after = [gathered(x, table) for x in (k, v)]
        for b, a in zip(before, after):
            for r in range(table.shape[0]):
                n = int(lens[r])
                assert torch.equal(a[r, :n], b[int(parents[r]), :n]), r
        seen.append(sorted(set(parents.tolist())))
    monkeypatch.setattr(D, '_beam_fork_torch', spy)
    prompts = _prompts(seed=5, lens=(60, 3))
    generate(m, prompts, 12, num_beams=4, prefill_chunk_size=16,
             kv_dtype=torch.float8_e4m3fn if kv == 'e4m3' else None)
    assert len(seen) >= 11 and any(len(s) < 8 for s in seen)               # beams forked from shared parents


def test_pool_never_exceeds_the_stated_bound(monkeypatch):
    m = _quiet(_model('opt_pre_ln'))
    made = []
    orig = BeamDecoder.__init__

    def spy(self, *a, **kw):
        orig(self, *a, **kw)
        made.append(self)
    monkeypatch.setattr(BeamDecoder, '__init__', spy)
    prompts = _prompts(seed=6, lens=(30, 7, 19))
    budgets, K = [8, 4, 9], 3
    generate(m, prompts, budgets, num_beams=K, prefill_chunk_size=8)
    dec, = made
    rows = [p for p in prompts for _ in range(K)]
    _, n_plan, _ = plan_prefix_pages(rows, [p.numel() + budgets[r // K] for r, p in enumerate(rows)])
    bound = sum((p.numel() - 1) // KV_PAGE + K * (-(-(p.numel() + n) // KV_PAGE) - (p.numel() - 1) // KV_PAGE)
                for p, n in zip(prompts, budgets)) + len(prompts) * K
    assert dec.n_pages == n_plan + len(prompts) * K <= bound
    assert int(dec.page_table.max()) < n_plan                              # scratch pages are never mapped


def test_e4m3_beam_search_is_deterministic_and_scores_match_teacher_forcing():
    m = _quiet(_model('llama_mha'))
    prompts = _prompts(seed=8, lens=(9, 4))
    kw = dict(num_beams=3, num_return_sequences=3, kv_dtype=torch.float8_e4m3fn, prefill_chunk_size=8)
    s1, s2 = {}, {}
    a = generate(m, prompts, 6, beam_stats=s1, **kw)
    b = generate(m, prompts, 6, beam_stats=s2, **kw)
    assert all(torch.equal(x, y) for x, y in zip(a, b)) and s1 == s2
    for i, p in enumerate(prompts):
        for k in range(3):
            toks = a[i * 3 + k]
            dec = PromptDecoder(m, max_len=p.numel() + toks.numel(), batch=1, kv_dtype=torch.float8_e4m3fn)
            lp, _ = dec.prefill_scores([torch.cat([p, toks[:-1]])], [toks], chunk=8)
            want = float(lp.double().sum()) / toks.numel()
            assert abs(s1['scores'][i * 3 + k] - want) < 1e-4, (i, k)


def test_argument_errors_are_raised_before_any_work(monkeypatch):
    def no_decoder(*a, **k):
        raise AssertionError('work started')
    monkeypatch.setattr(D, 'BeamDecoder', no_decoder)
    monkeypatch.setattr(D, 'PromptDecoder', no_decoder)
    m = _model('llama_gqa')
    p = _prompts()
    cases = ((dict(num_beams=2, do_sample=True), 'do_sample'), (dict(num_beams=2, prompt_lookup_num_tokens=2), 'prompt'),
             (dict(num_beams=2, max_batch_size=2), 'max_batch_size'),
             (dict(num_beams=2, share_prompt_prefixes=True), 'share'),
             (dict(num_beams=2, num_return_sequences=3), 'exceeds'), (dict(num_beams=17), 'num_beams'),
             (dict(num_beams=0), 'num_beams'), (dict(num_beams=True), 'num_beams'),
             (dict(num_beams=2, early_stopping='sometimes'), 'early_stopping'),
             (dict(num_beams=2, length_penalty=float('nan')), 'length_penalty'),
             (dict(num_beams=2, eos_token_id=[3, 4, 5, 6]), 'EOS'), (dict(num_beams=2, temperature=0.5), 'sampling'),
             (dict(num_beams=2, prefill_chunk_size=0), 'chunk'))
    for kw, msg in cases:
        with pytest.raises(ValueError, match=msg):
            generate(m, p, 5, **kw)


def test_beam_wrappers_check_their_arguments_before_any_launch(monkeypatch):
    from quip_b200 import fused
    monkeypatch.setattr(_lib, 'load', lambda: (_ for _ in ()).throw(AssertionError('launched')))
    x = torch.zeros(4, 50, dtype=torch.float16)
    sc = torch.zeros(4)
    cs, ci = torch.zeros(4, 8), torch.zeros(4, 8, dtype=torch.int32)
    with pytest.raises(ValueError, match='fp16'):
        fused.beam_candidates(x.float(), sc, 2, 8, cs, ci)
    with pytest.raises(ValueError, match='K <= 16'):
        fused.beam_candidates(x, sc, 2, 65, cs, ci)
    with pytest.raises(ValueError, match='cand_i'):
        fused.beam_candidates(x, sc, 2, 8, cs, ci.long())
    with pytest.raises(RuntimeError, match='CUDA'):
        fused.beam_candidates(x, sc, 2, 8, cs, ci)
    pool = torch.zeros(2, 12, 2, KV_PAGE, 64, dtype=torch.float16)
    tbl = torch.zeros(4, 3, dtype=torch.int32)
    par = torch.zeros(4, dtype=torch.long)
    with pytest.raises(ValueError, match='scratch'):
        fused.kv_beam_fork(pool, pool, tbl, tbl.clone(), par, par, 9)
    with pytest.raises(ValueError, match='k_scale'):
        fused.kv_beam_fork(pool.to(torch.float8_e4m3fn), pool.to(torch.float8_e4m3fn), tbl, tbl.clone(), par, par, 0)
    with pytest.raises(RuntimeError, match='CUDA'):
        fused.kv_beam_fork(pool, pool, tbl, tbl.clone(), par, par, 8)
    st = dict(score=torch.zeros(4), hist=torch.zeros(2, 2, 5, dtype=torch.long))
    with pytest.raises(ValueError, match='early_stopping'):
        fused.beam_select(cs, ci, torch.zeros(1, dtype=torch.long), torch.zeros(2, dtype=torch.long),
                          torch.zeros(1, dtype=torch.long), torch.ones(6), st, 2, 50, 'x', False)
