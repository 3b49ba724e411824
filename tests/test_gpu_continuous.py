"""Continuous batching on the GPU: the ragged kernels (quip_kv_append_ragged, quip_prefill_attention_ragged, fp16 and
e4m3, every head grouping and head size) bit for bit against the paged launch with padded B x T over the same bytes, on
shuffled NaN-poisoned pools; the decode graph against the eager step; and generate(max_batch_size=...) against each
prompt run alone on the tiny packed models, away from near ties."""
import pytest
import torch

from quip_b200 import fused
from quip_b200.decode import KV_PAGE, ContinuousDecoder, ContinuousSchedule, PromptDecoder, generate
from test_gpu_paged_kv import DEV, NKV, Paged, _q, _same
from test_gpu_speculative import _tiny

pytestmark = pytest.mark.gpu

GRID = [(fp8, hd, G) for fp8 in (False, True) for hd in (64, 128) for G in range(1, 9)]
IDS = [f'{"e4m3" if f else "fp16"}-hd{hd}-G{G}' for f, hd, G in GRID]

# (position, length): decode rows (length 1) and chunks, at and around page boundaries
SEQS = [(0, 1), (64, 63), (127, 64), (1, 65), (0, 512), (200, 1), (63, 7), (320, 1), (191, 130)]


def _padded(x, offs, T):
    """(N, ...) packed rows to (S, T, ...), row s holding sequence s's rows and zeros past them."""
    out = torch.zeros((len(offs) - 1, T) + tuple(x.shape[1:]), dtype=x.dtype, device=x.device)
    for s in range(len(offs) - 1):
        out[s, :offs[s + 1] - offs[s]] = x[offs[s]:offs[s + 1]]
    return out


def _run_both(fp8, hd, G, seqs, seed, unmap=None):
    """The same chunk through the padded paged launch and the ragged one, each on its own copy of one pool.  unmap:
    (sequence, page) set to -1 in both tables.  Returns (padded outputs, ragged outputs, offsets, the two caches)."""
    S = len(seqs)
    max_len = 12 * KV_PAGE
    need = [(p + n - 1) // KV_PAGE + 1 for p, n in seqs]
    a = Paged(S, max_len, hd, fp8, need, seed)
    b = Paged(S, max_len, hd, fp8, need, seed, table=a.table.clone(), n_pages=a.n_pages)
    if unmap is not None:
        for c in (a, b):
            c.table[unmap] = -1
            c.tdev = c.table.to(DEV)
    counts = [n for _, n in seqs]
    offs = [0]
    for n in counts:
        offs.append(offs[-1] + n)
    N, T = offs[-1], max(counts)
    q = _q((N, NKV * G, hd), seed + 1)
    kn, vn = _q((N, NKV, hd), seed + 2), _q((N, NKV, hd), seed + 3)
    pos = torch.tensor([p for p, _ in seqs], dtype=torch.long, device=DEV)
    cnt = torch.tensor(counts, dtype=torch.long, device=DEV)
    (kp, vp), pk = a.paged()
    fused.kv_append(_padded(kn, offs, T), _padded(vn, offs, T), kp, vp, pos, cnt, **pk)
    want = fused.prefill_attention(_padded(q, offs, T), kp, vp, pos, cnt, 0.1, **pk)
    seq = fused.RaggedChunk(offs, DEV)
    (kr, vr), rk = b.paged()
    table = rk.pop('page_table')
    fused.kv_append_ragged(kn, vn, kr, vr, seq, pos, table, **rk)
    got = fused.prefill_attention_ragged(q, kr, vr, seq, pos, table, 0.1, **rk)
    again = fused.prefill_attention_ragged(q, kr, vr, seq, pos, table, 0.1, **rk)
    _same(got, again, 'repeated launch')
    return want, got, offs, a, b


def _pools_equal(a, b, what):
    for x, y in ((a.kp, b.kp), (a.vp, b.vp)) + (((a.ksp, b.ksp), (a.vsp, b.vsp)) if a.fp8 else ()):
        _same(x, y, what)


@pytest.mark.parametrize('fp8,hd,G', GRID, ids=IDS)
def test_ragged_equals_the_padded_paged_launch_per_sequence(fp8, hd, G):
    want, got, offs, a, b = _run_both(fp8, hd, G, SEQS, seed=G + 10 * hd + int(fp8))
    for s in range(len(SEQS)):
        _same(got[offs[s]:offs[s + 1]], want[s, :offs[s + 1] - offs[s]], f'sequence {s}')
    assert not torch.isnan(got.float()).any()
    _pools_equal(a, b, 'appended bytes')


@pytest.mark.parametrize('fp8', [False, True])
def test_ragged_sequence_on_an_unmapped_page_gets_nan_and_writes_nothing_there(fp8):
    seqs = [(0, 1), (100, 70), (5, 3), (60, 9)]
    want, got, offs, a, b = _run_both(fp8, 128, 4, seqs, seed=3, unmap=(1, 2))     # slots 128 .. 169 of sequence 1
    for s in range(len(seqs)):
        _same(got[offs[s]:offs[s + 1]], want[s, :offs[s + 1] - offs[s]], f'sequence {s}')
    lost = got[offs[1]:offs[2]].float()
    assert torch.isnan(lost[128 - 100:]).all() and not torch.isnan(lost[:128 - 100]).any()
    assert not torch.isnan(got[:offs[1]].float()).any() and not torch.isnan(got[offs[2]:].float()).any()
    _pools_equal(a, b, 'appended bytes')


def test_ragged_wrappers_check_shapes_before_the_launch():
    seq = fused.RaggedChunk([0, 1, 4], DEV)
    pool = torch.zeros(3, NKV, KV_PAGE, 64, dtype=torch.float16, device=DEV)
    pos = torch.zeros(2, dtype=torch.long, device=DEV)
    tbl = torch.zeros(2, 1, dtype=torch.int32, device=DEV)
    k = torch.zeros(3, NKV, 64, dtype=torch.float16, device=DEV)
    with pytest.raises(ValueError, match='N=4'):
        fused.kv_append_ragged(k, k, pool, pool, seq, pos, tbl)
    with pytest.raises(ValueError, match='N=4'):
        fused.prefill_attention_ragged(torch.zeros(3, 4, 64, dtype=torch.float16, device=DEV), pool, pool, seq, pos,
                                       tbl, 1.0)
    with pytest.raises(ValueError, match='offsets live'):
        fused.kv_append_ragged(k, k, pool, pool, fused.RaggedChunk([0, 1, 3], 'cpu'), pos, tbl)


# ---- the decoder

def _prompts(n, seed=3, lo=3, hi=40):
    g = torch.Generator().manual_seed(seed)
    return [torch.randint(0, 320, (int(torch.randint(lo, hi, (1,), generator=g)),), generator=g) for _ in range(n)]


def _serve(model, prompts, budgets, rows, chunk, capture, kv_dtype=None):
    """generate()'s continuous loop with the done flags read after every step, recording for each request the logits
    that selected each of its tokens: {request: {token index: logits (vocab,) fp32}} and the outputs."""
    lens = [p.numel() for p in prompts]
    sched = ContinuousSchedule(lens, budgets, rows, rows * max(-(-(n + m) // KV_PAGE) for n, m in zip(lens, budgets)),
                               chunk)
    dec = ContinuousDecoder(model, max(n + m for n, m in zip(lens, budgets)), rows, len(sched.free_pages),
                            max(budgets), kv_dtype=kv_dtype)
    if capture:
        dec.capture()
    logs = {i: {} for i in range(len(prompts))}
    out = [None] * len(prompts)
    while True:
        done, n_gen = dec.done.cpu(), dec.n_gen.cpu()
        for r, i in enumerate(sched.req):
            if i is not None and done[r]:
                out[sched.retire(r)] = dec.generated[r, :int(n_gen[r])].cpu()
                dec.retire(r)
        for r, i, pages in sched.admit():
            dec.admit(r, pages, budgets[i])
        if sched.finished:
            return out, logs
        decoding, pieces = sched.plan()
        n_gen, done = dec.n_gen.cpu(), dec.done.cpu()
        if pieces:
            ends = [r for r, lo, n in pieces if lo + n == lens[sched.req[r]]]
            logits = dec.mixed_step(decoding, [(r, prompts[sched.req[r]][lo:lo + n], lo, r in ends)
                                               for r, lo, n in pieces])
            out_rows = list(decoding) + ends
        else:
            logits = dec.decode_step()
            out_rows = list(range(rows))
        if logits is None:
            continue
        logits = logits.float().cpu()
        for j, r in enumerate(out_rows):
            i = sched.req[r]
            if i is not None and not done[r]:
                logs[i][int(n_gen[r])] = logits[j]


@pytest.mark.parametrize('kind', [(2, 64), 'opt'])
def test_graph_step_equals_the_eager_step(kind):
    model = _tiny(kind)
    prompts, budgets = _prompts(7), [12, 5, 20, 9, 3, 16, 7]
    e_out, e_log = _serve(model, prompts, budgets, rows=3, chunk=16, capture=False)
    g_out, g_log = _serve(model, prompts, budgets, rows=3, chunk=16, capture=True)
    for i in range(len(prompts)):
        assert torch.equal(e_out[i], g_out[i]), i
        assert e_out[i].numel() == budgets[i]
        assert e_log[i].keys() == g_log[i].keys() == set(range(budgets[i]))
        for j in e_log[i]:
            assert torch.equal(e_log[i][j], g_log[i][j]), (i, j)


def _alone(model, p, n, chunk, kv_dtype):
    dec = PromptDecoder(model, max_len=p.numel() + n, batch=1, max_new=n, kv_dtype=kv_dtype).capture()
    with torch.no_grad():
        logits = [dec.prefill([p], chunk=chunk).float().cpu()[0]]
        logits += [dec.step().float().cpu()[0] for _ in range(n - 1)]
    return dec.generated[0].cpu(), logits


@pytest.mark.parametrize('kv_dtype', [None, torch.float8_e4m3fn])
@pytest.mark.parametrize('kind', [(4, 64), (2, 128), 'opt'])
def test_continuous_tokens_equal_each_request_alone_away_from_near_ties(kind, kv_dtype):
    """The mixed steps run the linears and attention at other token counts than a request run alone, so logits differ
    by rounding.  A token can differ only where the alone run's top-2 gap is at most twice the largest logit difference
    of the two runs there; up to the first such position each request's tokens must agree."""
    model = _tiny(kind)
    prompts, budgets = _prompts(9, seed=4), [14, 6, 20, 3, 11, 17, 8, 12, 5]
    out, logs = _serve(model, prompts, budgets, rows=4, chunk=24, capture=True, kv_dtype=kv_dtype)
    checked = 0
    for i, (p, n) in enumerate(zip(prompts, budgets)):
        assert out[i].numel() == n
        want, wlog = _alone(model, p, n, 24, kv_dtype)
        for j in range(n):
            top2 = wlog[j].topk(2).values
            diff = float((logs[i][j] - wlog[j]).abs().max())
            if float(top2[0] - top2[1]) <= 2 * diff:
                break
            assert int(out[i][j]) == int(want[j]), (i, j)
            checked += 1
    assert checked >= sum(budgets) // 2, checked


def test_generate_continuous_sampled_runs_and_keeps_each_requests_budget_and_eos():
    model = _tiny((2, 64))
    prompts, budgets = _prompts(6, seed=5), [9, 4, 15, 2, 7, 11]
    got = generate(model, prompts, budgets, do_sample=True, temperature=0.9, top_k=50, seed=3, max_batch_size=2,
                   prefill_chunk_size=8)
    assert [g.numel() for g in got] == budgets
    again = generate(model, prompts, budgets, do_sample=True, temperature=0.9, top_k=50, seed=3, max_batch_size=2,
                     prefill_chunk_size=8)
    assert all(torch.equal(a, b) for a, b in zip(got, again))
    eos = int(got[2][1])
    cut = generate(model, prompts, budgets, do_sample=True, temperature=0.9, top_k=50, seed=3, max_batch_size=2,
                   prefill_chunk_size=8, eos_token_id=eos)
    assert cut[2].numel() <= 2 and int(cut[2][-1]) == eos
