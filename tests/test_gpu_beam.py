"""Beam search on the GPU: quip_beam_candidates against oracle/beam.py, quip_beam_select bit for bit against its torch
restatement, quip_kv_beam_fork (fp16 and e4m3) bit for bit against the torch fork on shuffled NaN-poisoned pools, the captured
step against the eager one, and generate(num_beams=K) against the torch restatement on the tiny packed models, away
from near ties."""
import pytest
import torch

import quip_b200.decode as D
from oracle.beam import candidates as oracle_candidates
from quip_b200 import fused
from quip_b200.decode import KV_PAGE, BeamDecoder, plan_prefix_pages
from test_gpu_speculative import _tiny

pytestmark = pytest.mark.gpu
DEV = torch.device('cuda:0')


def _logits(R, V, seed, ld=None, off=0):
    g = torch.Generator().manual_seed(seed)
    ld = ld or V
    buf = (torch.randn(R * ld + off + 8, generator=g) * 3).half()
    x = buf[off:off + R * ld].view(R, ld)[:, :V]
    return buf, x


def _check_candidates(x, scores, K, C):
    xd, sd = x.to(DEV), scores.to(DEV)
    if x.stride(0) != x.shape[1]:                       # keep the row stride on the device
        full = torch.empty(x.shape[0], x.stride(0), dtype=torch.float16, device=DEV)
        full[:, :x.shape[1]] = xd
        xd = full[:, :x.shape[1]]
    R = x.shape[0]
    cs = torch.empty(R, C, device=DEV)
    ci = torch.empty(R, C, dtype=torch.int32, device=DEV)
    fused.beam_candidates(xd, sd, K, C, cs, ci)
    ws, wi = oracle_candidates(x, scores, K, C)
    assert torch.equal(ci.cpu(), wi), (ci.cpu(), wi)
    torch.testing.assert_close(cs.cpu(), ws, rtol=2e-6, atol=2e-5, equal_nan=True)
    cs2, ci2 = torch.empty_like(cs), torch.empty_like(ci)
    fused.beam_candidates(xd, sd, K, C, cs2, ci2)
    assert torch.equal(cs.view(torch.int32), cs2.view(torch.int32)) and torch.equal(ci, ci2)


@pytest.mark.parametrize('V', [50, 32000, 50272, 128256])
@pytest.mark.parametrize('R', [1, 4, 256])
def test_candidates_match_the_oracle(R, V):
    K = 4 if R % 4 == 0 else 1
    for C, ld, off in ((8, V, 0), (64, V + 3, 1)):
        buf, x = _logits(R, V, seed=R + V + C, ld=ld, off=off)
        x = x.clone() if ld == V else x
        g = torch.Generator().manual_seed(C)
        scores = torch.randn(R, generator=g) * 5
        scores[::3] = -1e9
        if R > 1:
            x[1] = x[0]                                               # identical rows: ties across rows
            x[R - 1] = float('nan') if R > 2 else x[R - 1]
        x[0, 7] = x[0, 11] = x[0, 3] = x[0].float().max().half()     # planted exact ties at the top
        if R >= 4:
            x[2] = float('-inf')
            scores[3] = float('-inf')
        _check_candidates(x, scores, K, C)


def _rand_state(B, K, max_new, seed):
    g = torch.Generator().manual_seed(seed)
    st = dict(score=torch.randn(B * K, generator=g) * 3,
              hist=torch.randint(0, 50, (B, K, max_new), generator=g),
              hist_tmp=torch.zeros(B, K, max_new, dtype=torch.long),
              fin_score=-torch.rand(B, K, generator=g) * 10,
              fin_len=torch.randint(1, 4, (B, K), generator=g),
              fin_tok=torch.randint(0, 50, (B, K, max_new), generator=g),
              fin_tmp=torch.zeros(B, K, max_new, dtype=torch.long),
              fin_filled=(torch.rand(B, K, generator=g) < 0.5).to(torch.uint8),
              heur=(torch.rand(B, generator=g) < 0.8).to(torch.uint8),
              done=(torch.rand(B, generator=g) < 0.15).to(torch.uint8),
              tokens=torch.zeros(B * K, dtype=torch.long), parents=torch.zeros(B * K, dtype=torch.long),
              adv=torch.zeros(B * K, dtype=torch.long))
    st['fin_score'] = torch.where(st['fin_filled'].bool(), st['fin_score'], torch.full_like(st['fin_score'], -1e9))
    return st


@pytest.mark.parametrize('es', [False, True, 'never'])
@pytest.mark.parametrize('K,n_eos', [(2, 0), (4, 1), (3, 3), (16, 3)])
def test_select_matches_the_torch_rule_bit_for_bit(K, n_eos, es):
    B, V, max_new = 6, 50, 9
    C = max(2, 1 + n_eos) * K
    st = _rand_state(B, K, max_new, seed=K * 10 + n_eos)
    sd = {n: t.to(DEV) for n, t in st.items()}
    sd['tokens'] = sd['tokens'].clone()
    eos = torch.tensor([5, 9, 13][:n_eos], dtype=torch.long)
    budget = torch.tensor([3, 9, 6, 2, 9, 5], dtype=torch.long)
    pen = torch.tensor([float(n) ** 1.5 if n else 1.0 for n in range(max_new + 1)], dtype=torch.float32)
    g = torch.Generator().manual_seed(K)
    for t in range(max_new):
        x = (torch.randn(B * K, V, generator=g) * 2).half()
        x[:, 5] = x[:, 5].float().add(3).half()                      # EOS ids among the candidates
        x[::2, 17] = x[::2, 18]                                      # exact ties
        cs, ci = D._beam_candidates_torch(x.float(), st['score'], K, C)
        step = torch.tensor([t])
        D._beam_select_torch(cs, ci, eos, budget, step, pen, st, K, V, es, es == 'never')
        fused.beam_select(cs.to(DEV), ci.to(DEV), eos.to(DEV), budget.to(DEV), step.to(DEV), pen.to(DEV), sd, K, V,
                          es, es == 'never')
        for n in st:
            if n.endswith('_tmp'):                               # the kernel's scratch copies
                continue
            a, b = st[n], sd[n].cpu()
            if a.dtype == torch.float32:
                a, b = a.view(torch.int32), b.view(torch.int32)
            assert torch.equal(a.to(b.dtype), b), (t, n, a, b)


@pytest.mark.parametrize('hd', [64, 128])
@pytest.mark.parametrize('fp8', [False, True])
def test_fork_matches_the_torch_fork_bit_for_bit(fp8, hd):
    L, nkv, R, P = 3, 2, 8, 5
    N = R * P + R + 7
    g = torch.Generator().manual_seed(hd + fp8)
    perm = torch.randperm(R * P + 7, generator=g)[:R * P].view(R, P).int()     # shuffled; scratch pages after them
    perm[:, :2] = perm[0, :2]                                                    # two shared prompt pages
    perm[5, 4] = -1                                                              # an unmapped page
    table = perm.contiguous()
    k = torch.randn(L, N, nkv, KV_PAGE, hd, generator=g)
    v = torch.randn(L, N, nkv, KV_PAGE, hd, generator=g)
    used = torch.zeros(N, dtype=torch.bool)
    used[table[table >= 0].long()] = True
    k[:, ~used] = float('nan')                                                   # poison: pages nothing maps
    v[:, ~used] = float('nan')
    dt = torch.float8_e4m3fn if fp8 else torch.float16
    k, v = k.to(dt), v.to(dt)
    ks = vs = None
    if fp8:
        ks, vs = torch.rand(L, N, nkv, KV_PAGE, generator=g), torch.rand(L, N, nkv, KV_PAGE, generator=g)
    parents = torch.tensor([3, 3, 0, 2, 4, 6, 5, 7])                            # fan-out, a cycle, a swap, identity
    for lens in ([2 * KV_PAGE + 1] * R, [3 * KV_PAGE - 1] * R, [3 * KV_PAGE] * R, [1, 64, 65, 127, 128, 320, 200, 0]):
        lens = torch.tensor(lens)
        ref = [x.clone() if x is not None else None for x in (k, v, ks, vs)]
        tbl = table.clone()
        D._beam_fork_torch(ref[0], ref[1], tbl, parents, lens, ref[2], ref[3])
        dev = [x.to(DEV) if x is not None else None for x in (k, v, ks, vs)]
        td = table.to(DEV)
        fused.kv_beam_fork(dev[0], dev[1], td, torch.empty_like(td), parents.to(DEV), lens.to(DEV), R * P + 7,
                           k_scale=dev[2], v_scale=dev[3])
        assert torch.equal(td.cpu(), tbl)
        for a, b in zip(ref, dev):
            if a is not None:
                a8, b8 = a.contiguous().view(torch.uint8), b.cpu().contiguous().view(torch.uint8)
                # scratch pages hold whatever the gather put there; every other page must match byte for byte
                assert torch.equal(a8[:, :R * P + 7], b8[:, :R * P + 7])


def _beam_run(model, prompts, budgets, K, capture, kernel=True, kv_dtype=None, eos=()):
    rows = [p for p in prompts for _ in range(K)]
    B, max_new = len(prompts), max(budgets)
    max_len = max(p.numel() for p in prompts) + max_new
    table, n_plan, starts = plan_prefix_pages(rows, [rows[r].numel() + budgets[r // K] for r in range(B * K)],
                                              max_pages=-(-max_len // KV_PAGE))
    dec = BeamDecoder(model, max_len, B, K, max_new, table, n_plan, budgets, eos=eos, kv_dtype=kv_dtype)
    dec._kernel = kernel
    if capture:
        dec.capture()
    logs, sel = [], []
    with torch.no_grad():
        logs.append(dec.prefill(rows, chunk=16, starts=starts).float().cpu())
        sel.append((dec.beam['tokens'].cpu().clone(), dec.beam['parents'].cpu().clone(), dec.cand_s.cpu().clone(),
                    dec.cand_i.cpu().clone()))
        for _ in range(max_new - 1):
            logs.append(dec.step().float().cpu())
            sel.append((dec.beam['tokens'].cpu().clone(), dec.beam['parents'].cpu().clone(), dec.cand_s.cpu().clone(),
                        dec.cand_i.cpu().clone()))
    return dec, logs, sel


@pytest.mark.parametrize('kind', [(2, 64), 'opt'])
def test_graph_step_equals_the_eager_step(kind):
    model = _tiny(kind)
    g = torch.Generator().manual_seed(2)
    prompts = [torch.randint(0, 320, (n,), generator=g) for n in (70, 9, 33)]
    budgets = [12, 5, 10]
    e, e_log, e_sel = _beam_run(model, prompts, budgets, 4, capture=False)
    c, c_log, c_sel = _beam_run(model, prompts, budgets, 4, capture=True)
    for a, b in zip(e_log, c_log):
        assert torch.equal(a, b)
    for a, b in zip(e_sel, c_sel):
        assert all(torch.equal(x, y) for x, y in zip(a, b))
    for n in e.beam:
        assert torch.equal(e.beam[n], c.beam[n]), n
    assert torch.equal(e.page_table, c.page_table)


@pytest.mark.parametrize('kv_dtype', [None, torch.float8_e4m3fn])
@pytest.mark.parametrize('kind', [(4, 64), (2, 128), 'opt'])
def test_beam_tokens_match_the_torch_restatement_away_from_near_ties(kind, kv_dtype):
    """The kernels compute the log-softmax and the attention in another order than the torch restatement, so scores
    differ by rounding.  The running beams are the top K candidates in order, so the compared scores are a prompt's
    top K + 1.  Up to the first step where two of them lie within twice the largest difference of the two runs'
    log-probs at those candidates, the running beams (tokens and parents) must agree."""
    model = _tiny(kind)
    g = torch.Generator().manual_seed(6)
    prompts = [torch.randint(0, 320, (n,), generator=g) for n in (66, 12, 30, 5)]
    budgets, K = [14, 10, 16, 8], 3
    _, k_log, k_sel = _beam_run(model, prompts, budgets, K, capture=True, kv_dtype=kv_dtype)
    _, t_log, t_sel = _beam_run(model, prompts, budgets, K, capture=False, kernel=False, kv_dtype=kv_dtype)
    checked, total, notes = 0, 0, []
    for b in range(len(prompts)):
        rows = slice(b * K, (b + 1) * K)
        for s in range(budgets[b]):
            total += 1
            top = t_sel[s][2][rows].reshape(-1)
            top = top[torch.isfinite(top) & (top > -1e8)].sort(descending=True)
            vals, idx = top.values[:K + 1], t_sel[s][3][rows].reshape(-1)[top.indices[:K + 1]].long()
            lk = torch.log_softmax(k_log[s][rows], -1).reshape(-1)[idx]
            lt = torch.log_softmax(t_log[s][rows], -1).reshape(-1)[idx]
            diff = float((lk - lt).abs().max())
            if bool((vals[:-1] - vals[1:] <= 2 * diff).any()):
                notes.append((b, s, diff, (vals[:-1] - vals[1:]).min().item()))
                break
            assert torch.equal(k_sel[s][0][rows], t_sel[s][0][rows]), (b, s)
            assert torch.equal(k_sel[s][1][rows], t_sel[s][1][rows]), (b, s)
            checked += 1
    assert checked >= total // 2, (checked, total, notes)


def test_generate_beam_runs_on_the_gpu_and_cuts_at_eos():
    model = _tiny((2, 64))
    g = torch.Generator().manual_seed(9)
    prompts = [torch.randint(0, 320, (n,), generator=g) for n in (20, 7)]
    stats = {}
    got = D.generate(model, prompts, [10, 6], num_beams=4, num_return_sequences=2, beam_stats=stats)
    assert [x.numel() for x in got] == [10, 10, 6, 6] and stats['steps'] <= 10
    eos = int(got[0][3])
    cut = D.generate(model, prompts, [10, 6], num_beams=4, num_return_sequences=2, eos_token_id=eos)
    assert all(eos not in x[:-1].tolist() for x in cut)
