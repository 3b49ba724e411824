"""The prefix cache of continuous batching on the GPU: one ragged quip_kv_append_ragged + quip_prefill_attention_ragged
pair in which a sequence maps pages that another sequence of the same launch pair writes, bit for bit against the same
pair with private copies of those pages (fp16 and e4m3, every head grouping and head size); and generate()'s continuous
loop with the cache on the tiny packed models against each request run alone, away from near ties."""
import pytest
import torch

from quip_b200 import fused
from quip_b200.decode import KV_PAGE, ContinuousDecoder, ContinuousSchedule, generate
from test_gpu_continuous import GRID, IDS, _alone
from test_gpu_paged_kv import DEV, NKV, Paged, _q, _same
from test_gpu_speculative import _tiny

pytestmark = pytest.mark.gpu

# (position, length) of each sequence, and the leading pages it maps from the sequence named: D reads page 0 and B
# pages 0 and 1 of A, which A writes in the same launch pair; D comes before A in the packing, B after it
SEQS = [(64, 5), (0, 200), (300, 1), (128, 70)]
SHARES = {0: (1, 1), 3: (1, 2)}


def _launch(c, table, seqs, q, kn, vn, pools):
    offs = [0]
    for _, n in seqs:
        offs.append(offs[-1] + n)
    seq = fused.RaggedChunk(offs, DEV)
    pos = torch.tensor([p for p, _ in seqs], dtype=torch.long, device=DEV)
    kp, vp, ksp, vsp = pools
    kw = dict(k_scale=ksp, v_scale=vsp) if c.fp8 else {}
    t = table.to(DEV)
    fused.kv_append_ragged(kn, vn, kp, vp, seq, pos, t, **kw)
    return fused.prefill_attention_ragged(q, kp, vp, seq, pos, t, 0.1, **kw), offs


@pytest.mark.parametrize('fp8,hd,G', GRID, ids=IDS)
def test_sequence_reading_pages_written_in_the_same_launch_pair_equals_private_copies(fp8, hd, G):
    need = [(p + n - 1) // KV_PAGE + 1 for p, n in SEQS]
    c = Paged(len(SEQS), 6 * KV_PAGE, hd, fp8, need, seed=G + 10 * hd + int(fp8))
    private = c.table
    shared = private.clone()
    for s, (src, S) in SHARES.items():
        shared[s, :S] = private[src, :S]
    N = sum(n for _, n in SEQS)
    q = _q((N, NKV * G, hd), 1)
    kn, vn = _q((N, NKV, hd), 2), _q((N, NKV, hd), 3)
    base = [c.kp, c.vp] + ([c.ksp, c.vsp] if fp8 else [None, None])
    xs = [None if x is None else x.clone() for x in base]
    got, offs = _launch(c, shared, SEQS, q, kn, vn, xs)
    ys = [None if x is None else x.clone() for x in base]
    for s, (src, S) in SHARES.items():                  # private copies of what A wrote there in the shared launch
        for j in range(S):
            for x, y in zip(xs, ys):
                if x is not None:
                    y[int(private[s, j])] = x[int(private[src, j])]
    want, _ = _launch(c, private, SEQS, q, kn, vn, ys)
    _same(got, want, 'outputs')
    assert not torch.isnan(got.float()).any()
    mine = [int(private[s, j]) for s in range(len(SEQS)) for j in range(SHARES.get(s, (0, 0))[1], need[s])]
    idx = torch.tensor(mine, device=DEV)
    for x, y in zip(xs, ys):                           # every page a sequence writes itself holds the same bytes
        if x is not None:
            _same(x[idx], y[idx], 'own pages')


# ---- generate()'s loop with the cache on

def _prompts(seed=4):
    g = torch.Generator().manual_seed(seed)
    head = torch.randint(0, 320, (200,), generator=g)

    def tail(n):
        return torch.randint(0, 320, (n,), generator=g)
    t0 = tail(5)
    return [torch.cat((head[:140], t0)), torch.cat((head[:130], tail(11))), torch.cat((head[:140], t0)), tail(30),
            torch.cat((head[:70], tail(3))), head[:129], torch.cat((head[:190], tail(9))), tail(12),
            torch.cat((head[:64], tail(40)))]


def _serve(model, prompts, budgets, rows, chunk, kv_dtype=None):
    """generate()'s continuous loop with the prefix cache, the done flags read after every step, recording for each
    request the logits that selected each of its tokens.  Returns the outputs, the logits and the schedule."""
    lens = [p.numel() for p in prompts]
    n_pages = rows * max(-(-(n + m) // KV_PAGE) for n, m in zip(lens, budgets))
    sched = ContinuousSchedule(lens, budgets, rows, n_pages, chunk, prompts=prompts)
    dec = ContinuousDecoder(model, max(n + m for n, m in zip(lens, budgets)), rows, n_pages, max(budgets),
                            kv_dtype=kv_dtype)
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
            dec.admit(r, pages, budgets[i], start=KV_PAGE * sched.shared[i])
        if sched.finished:
            return out, logs, sched
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


@pytest.mark.parametrize('kv_dtype', [None, torch.float8_e4m3fn])
@pytest.mark.parametrize('kind', [(4, 64), (2, 128)])
def test_prefix_cached_tokens_equal_each_request_alone_away_from_near_ties(kind, kv_dtype):
    """As test_continuous_tokens_equal_each_request_alone_away_from_near_ties: up to the first position where the alone
    run's top-2 gap is at most twice the largest logit difference of the two runs, each request's tokens agree."""
    model = _tiny(kind)
    prompts, budgets = _prompts(), [14, 6, 20, 3, 11, 17, 8, 12, 5]
    out, logs, sched = _serve(model, prompts, budgets, rows=4, chunk=24, kv_dtype=kv_dtype)
    lens = [p.numel() for p in prompts]
    assert sched.shared == [0, 2, 2, 0, 1, 2, 2, 0, 1]
    assert sched.prefilled == sum(lens) - KV_PAGE * sum(sched.shared) < sum(lens)
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


def test_generate_with_the_prefix_cache_keeps_budgets_and_repeats_itself():
    model = _tiny((2, 64))
    prompts, budgets = _prompts(seed=6), [9, 4, 15, 2, 7, 11, 6, 3, 8]
    kw = dict(do_sample=True, temperature=0.9, top_k=50, seed=3, max_batch_size=3, prefill_chunk_size=16,
              prefix_cache=True, kv_dtype=torch.float8_e4m3fn)
    got = generate(model, prompts, budgets, **kw)
    assert [g.numel() for g in got] == budgets
    again = generate(model, prompts, budgets, **kw)
    assert all(torch.equal(a, b) for a, b in zip(got, again))
