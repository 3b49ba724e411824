"""Paged KV cache on the GPU: every paged kernel (quip_decode_attention, quip_extend_attention, quip_kv_append,
quip_prefill_attention with a page table, each fp16 and e4m3) against its contiguous twin over the same cached
bytes -- bit for bit, outputs and appended bytes and scales -- with pools built by scattering the contiguous cache into
shuffled pages, unused pages NaN-poisoned and table entries past each row's slots unmapped; shared pages; the guard
on page ids outside the pool; and the decoder and generate() end to end."""
import pytest
import torch

from quip_b200 import fused
from quip_b200.decode import KV_PAGE, PromptDecoder, generate

pytestmark = pytest.mark.gpu

DEV = 'cuda:0'
E4 = torch.float8_e4m3fn
NKV = 2
GRID = [(fp8, hd, G) for fp8 in (False, True) for hd in (64, 128) for G in (1, 4, 8)]
IDS = [f'{"e4m3" if f else "fp16"}-hd{hd}-G{G}' for f, hd, G in GRID]


def _bits(x):
    return x.view(torch.uint8) if x.dtype == E4 else x.contiguous().view(torch.int16 if x.element_size() == 2
                                                                           else torch.int32)


def _same(a, b, what):
    assert torch.equal(_bits(a), _bits(b)), what


def _cache(B, max_len, hd, fp8, seed):
    g = torch.Generator().manual_seed(seed)
    k = torch.randn(B, NKV, max_len, hd, generator=g)
    v = torch.randn(B, NKV, max_len, hd, generator=g)
    if not fp8:
        return k.half().to(DEV), v.half().to(DEV), None, None
    ks = torch.rand(B, NKV, max_len, generator=g) * 0.02 + 1e-3
    vs = torch.rand(B, NKV, max_len, generator=g) * 0.02 + 1e-3
    return k.to(E4).to(DEV), v.to(E4).to(DEV), ks.to(DEV), vs.to(DEV)


def _table(B, max_pages, need, seed, spare=3):
    """Row b's pages 0 .. need[b] - 1 on shuffled page ids, -1 past them; n_pages includes `spare` unused pages."""
    n_pages = sum(need) + spare
    ids = torch.randperm(n_pages, generator=torch.Generator().manual_seed(seed)).tolist()
    table = torch.full((B, max_pages), -1, dtype=torch.int32)
    for b in range(B):
        for p in range(need[b]):
            table[b, p] = ids.pop()
    return table, n_pages


def _poison(dtype, shape):
    if dtype == E4:
        return torch.full(shape, 0x7F, dtype=torch.uint8, device=DEV).view(E4)
    return torch.full(shape, float('nan'), dtype=dtype, device=DEV)


def _scatter(x, table, n_pages):
    """Pool (n_pages, nkv, 64, ...) holding slot j of row b of the contiguous x (B, nkv, max_len, ...) at slot j % 64 of
    page table[b, j // 64] (mapped entries only); every other page NaN."""
    B, nkv, max_len = x.shape[:3]
    pool = _poison(x.dtype, (n_pages, nkv, KV_PAGE) + tuple(x.shape[3:]))
    for b in range(B):
        for p in range(max_len // KV_PAGE):
            if 0 <= int(table[b, p]) < n_pages:
                pool[int(table[b, p])] = x[b, :, KV_PAGE * p:KV_PAGE * (p + 1)]
    return pool


class Paged:
    """A contiguous cache and its paged twin (pools, scales and table on the device)."""

    def __init__(self, B, max_len, hd, fp8, need, seed, table=None, n_pages=None):
        assert max_len % KV_PAGE == 0
        self.fp8 = fp8
        self.kc, self.vc, self.ks, self.vs = _cache(B, max_len, hd, fp8, seed)
        if table is None:
            table, n_pages = _table(B, max_len // KV_PAGE, need, seed)
        self.table, self.n_pages = table, n_pages
        self.tdev = table.to(DEV)
        self.kp, self.vp = _scatter(self.kc, table, n_pages), _scatter(self.vc, table, n_pages)
        self.ksp = self.vsp = None
        if fp8:
            self.ksp, self.vsp = _scatter(self.ks, table, n_pages), _scatter(self.vs, table, n_pages)

    def contiguous(self):
        return (self.kc, self.vc), (dict(k_scale=self.ks, v_scale=self.vs) if self.fp8 else {})

    def paged(self):
        sc = dict(k_scale=self.ksp, v_scale=self.vsp) if self.fp8 else {}
        return (self.kp, self.vp), dict(page_table=self.tdev, **sc)

    def assert_pools_hold(self, what):
        """The pools equal the contiguous cache (after the same launches) scattered through the table: appended bytes and
        scales landed where the table says, and no unused page was touched."""
        pairs = [(self.kp, self.kc), (self.vp, self.vc)]
        if self.fp8:
            pairs += [(self.ksp, self.ks), (self.vsp, self.vs)]
        for pool, x in pairs:
            _same(pool, _scatter(x, self.table, self.n_pages), what)


def _need(pos_last):
    return [p // KV_PAGE + 1 for p in pos_last]


def _q(shape, seed):
    return (torch.randn(shape, generator=torch.Generator().manual_seed(seed)) * 0.5).half().to(DEV)


# ---- bit-identity with the contiguous kernels

def _decode_edges(max_len, chunk):
    last = (max_len // chunk - 1) * chunk
    return [p for p in dict.fromkeys([0, 63, 64, 65, chunk - 1, chunk, last - 1, last, max_len - 1]) if 0 <= p < max_len]


@pytest.mark.parametrize('fp8,hd,G', GRID, ids=IDS)
def test_decode_paged_equals_contiguous(fp8, hd, G):
    max_len = 5 * KV_PAGE
    for B in (7, 48):                          # 64-slot chunks at 7 rows, 128-slot chunks at 48 (2 kv heads, 320 slots)
        pos = (_decode_edges(max_len, 128) * 8)[:B]
        c = Paged(B, max_len, hd, fp8, _need(pos), seed=B + hd + G)
        q = _q((B, NKV * G, hd), 1)
        kn, vn = _q((B, NKV, hd), 2), _q((B, NKV, hd), 3)
        positions = torch.tensor(pos, device=DEV)
        (kc, vc), sc = c.contiguous()
        want = fused.decode_attention(q, kn, vn, kc, vc, positions, 0.1, **sc)
        (kp, vp), pk = c.paged()
        got = fused.decode_attention(q, kn, vn, kp, vp, positions, 0.1, **pk)
        torch.cuda.synchronize()
        _same(got, want, ('decode', B))
        assert not got.isnan().any()
        c.assert_pools_hold(('decode', B))


@pytest.mark.parametrize('fp8,hd,G', GRID, ids=IDS)
def test_extend_paged_equals_contiguous(fp8, hd, G):
    max_len = 4 * KV_PAGE
    for T in (1, 5, 8):
        pos = [p for p in dict.fromkeys([0, 64 - (T + 1) // 2, 63, 64, 128 - T, max_len - T]) if 0 <= p <= max_len - T]
        B = len(pos)
        c = Paged(B, max_len, hd, fp8, _need([p + T - 1 for p in pos]), seed=T + hd + G)
        q = _q((B, T, NKV * G, hd), 4)
        kn, vn = _q((B, T, NKV, hd), 5), _q((B, T, NKV, hd), 6)
        positions = torch.tensor(pos, device=DEV)
        (kc, vc), sc = c.contiguous()
        want = fused.extend_attention(q, kn, vn, kc, vc, positions, 0.1, **sc)
        (kp, vp), pk = c.paged()
        got = fused.extend_attention(q, kn, vn, kp, vp, positions, 0.1, **pk)
        torch.cuda.synchronize()
        _same(got, want, ('extend', T))
        assert not got.isnan().any()
        c.assert_pools_hold(('extend', T))


@pytest.mark.parametrize('fp8,hd,G', GRID, ids=IDS)
def test_append_and_prefill_paged_equal_contiguous(fp8, hd, G):
    for T in (1, 16, 100):
        max_len = T + 3 * KV_PAGE + 40
        max_len = -(-max_len // KV_PAGE) * KV_PAGE
        rows = [(0, T), (5, 0), (63, T), (64, max(1, T - 3)), (max_len - T, T), (17, (T + 1) // 2)]
        pos, cnt = zip(*rows)
        B = len(rows)
        c = Paged(B, max_len, hd, fp8, _need([p + max(n, 1) - 1 for p, n in rows]), seed=T + hd + G)
        q = _q((B, T, NKV * G, hd), 7)
        kn, vn = _q((B, T, NKV, hd), 8), _q((B, T, NKV, hd), 9)
        positions, counts = torch.tensor(pos, device=DEV), torch.tensor(cnt, device=DEV)
        (kc, vc), sc = c.contiguous()
        fused.kv_append(kn, vn, kc, vc, positions, counts, **sc)
        want = fused.prefill_attention(q, kc, vc, positions, counts, 0.1, **sc)
        (kp, vp), pk = c.paged()
        fused.kv_append(kn, vn, kp, vp, positions, counts, **pk)
        got = fused.prefill_attention(q, kp, vp, positions, counts, 0.1, **pk)
        torch.cuda.synchronize()
        _same(got, want, ('prefill', T))
        assert not got.isnan().any()
        c.assert_pools_hold(('prefill', T))


# ---- shared pages

@pytest.mark.parametrize('fp8', [False, True], ids=['fp16', 'e4m3'])
def test_rows_sharing_prefix_pages_equal_rows_with_private_copies(fp8):
    """Rows 1..3 map their first S pages to row 0's; the contiguous twin holds copies of them in every row."""
    hd, G, S, max_len = 128, 4, 2, 6 * KV_PAGE
    B = 4
    c = Paged(B, max_len, hd, fp8, [6] * B, seed=11)
    for x in (c.kc, c.vc) + ((c.ks, c.vs) if fp8 else ()):
        x[1:, :, :S * KV_PAGE] = x[0, :, :S * KV_PAGE]
    table = c.table.clone()
    table[1:, :S] = table[0, :S]                              # rows 1..3's own first pages become unused
    _rebuild(c, table)
    (kc, vc), sc = c.contiguous()
    (kp, vp), pk = c.paged()
    pos = torch.tensor([S * KV_PAGE + 3, S * KV_PAGE, 5 * KV_PAGE - 1, 4 * KV_PAGE + 9], device=DEV)
    q, kn, vn = _q((B, NKV * G, hd), 12), _q((B, NKV, hd), 13), _q((B, NKV, hd), 14)
    _same(fused.decode_attention(q, kn, vn, kp, vp, pos, 0.1, **pk),
          fused.decode_attention(q, kn, vn, kc, vc, pos, 0.1, **sc), 'decode')
    T = 5
    q, kn, vn = _q((B, T, NKV * G, hd), 15), _q((B, T, NKV, hd), 16), _q((B, T, NKV, hd), 17)
    _same(fused.extend_attention(q, kn, vn, kp, vp, pos, 0.1, **pk),
          fused.extend_attention(q, kn, vn, kc, vc, pos, 0.1, **sc), 'extend')
    T = 40
    pos = torch.tensor([S * KV_PAGE] * B, device=DEV)
    counts = torch.tensor([T, T - 7, 1, T], device=DEV)
    q, kn, vn = _q((B, T, NKV * G, hd), 18), _q((B, T, NKV, hd), 19), _q((B, T, NKV, hd), 20)
    fused.kv_append(kn, vn, kc, vc, pos, counts, **sc)
    fused.kv_append(kn, vn, kp, vp, pos, counts, **pk)
    _same(fused.prefill_attention(q, kp, vp, pos, counts, 0.1, **pk),
          fused.prefill_attention(q, kc, vc, pos, counts, 0.1, **sc), 'prefill')
    torch.cuda.synchronize()
    c.assert_pools_hold('shared')


def _rebuild(c, table):
    """c's contiguous cache (rows sharing table's shared pages hold equal copies) scattered through table."""
    c.table, c.tdev = table, table.to(DEV)
    c.kp, c.vp = _scatter(c.kc, table, c.n_pages), _scatter(c.vc, table, c.n_pages)
    if c.fp8:
        c.ksp, c.vsp = _scatter(c.ks, table, c.n_pages), _scatter(c.vs, table, c.n_pages)
    return c


# ---- the guard on page ids outside the pool

@pytest.mark.parametrize('fp8', [False, True], ids=['fp16', 'e4m3'])
@pytest.mark.parametrize('bad', [-1, 'n_pages'])
def test_pages_outside_the_pool_give_nan_rows_and_are_never_written(fp8, bad):
    hd, G, max_len = 64, 4, 4 * KV_PAGE
    pos = [70, 130, 200, 5]                   # row 0: its append page bad; row 1: an earlier page bad; rows 2, 3 fine
    B = len(pos)
    c = Paged(B, max_len, hd, fp8, _need([p + 7 for p in pos]), seed=21)
    table = c.table.clone()
    badid = -1 if bad == -1 else c.n_pages
    table[0, 1] = badid
    table[1, 0] = badid
    _rebuild(c, table)
    (kc, vc), sc = c.contiguous()
    (kp, vp), pk = c.paged()
    positions = torch.tensor(pos, device=DEV)
    ok = torch.tensor([False, False, True, True], device=DEV)

    def check(got, want, what, rows_nan):
        torch.cuda.synchronize()
        assert got[rows_nan].isnan().all(), what
        _same(got[~rows_nan], want[~rows_nan], what)

    # decode: row 0 writes nothing (its slot's page is bad); row 1 appends on its valid page and reads NaN
    q, kn, vn = _q((B, NKV * G, hd), 22), _q((B, NKV, hd), 23), _q((B, NKV, hd), 24)
    want = fused.decode_attention(q, kn, vn, kc, vc, positions, 0.1, **sc)
    got = fused.decode_attention(q, kn, vn, kp, vp, positions, 0.1, **pk)
    check(got, want, 'decode', ~ok)
    c.assert_pools_hold('decode')             # row 0's write went nowhere: the contiguous slot has no page here
    # extend: the same rows
    T = 6
    q, kn, vn = _q((B, T, NKV * G, hd), 25), _q((B, T, NKV, hd), 26), _q((B, T, NKV, hd), 27)
    want = fused.extend_attention(q, kn, vn, kc, vc, positions, 0.1, **sc)
    got = fused.extend_attention(q, kn, vn, kp, vp, positions, 0.1, **pk)
    check(got, want, 'extend', ~ok)
    c.assert_pools_hold('extend')
    # append + prefill: the tokens that read or write a bad page are NaN (row 0 from slot 64 on), the others not
    T = 8
    positions = torch.tensor([60, 100, 190, 0], device=DEV)
    counts = torch.tensor([T, T, T, T], device=DEV)
    q, kn, vn = _q((B, T, NKV * G, hd), 28), _q((B, T, NKV, hd), 29), _q((B, T, NKV, hd), 30)
    fused.kv_append(kn, vn, kc, vc, positions, counts, **sc)
    want = fused.prefill_attention(q, kc, vc, positions, counts, 0.1, **sc)
    fused.kv_append(kn, vn, kp, vp, positions, counts, **pk)
    got = fused.prefill_attention(q, kp, vp, positions, counts, 0.1, **pk)
    torch.cuda.synchronize()
    lost = torch.zeros(B, T, dtype=torch.bool, device=DEV)
    lost[0, 4:] = True                        # slots 64.. of row 0
    lost[1] = True                            # row 1 reads its page 0
    assert got[lost].isnan().all()
    _same(got[~lost], want[~lost], 'prefill')
    c.assert_pools_hold('append')


# ---- the decoder and generate()

def _tiny(kind):
    from test_gpu_generate import _tiny as tiny
    return tiny(kind)


def _prompts(lens, seed, prefix=0):
    g = torch.Generator().manual_seed(seed)
    pre = torch.randint(0, 320, (prefix,), generator=g)
    return [torch.cat((pre, torch.randint(0, 320, (n,), generator=g))) for n in lens]


def _decode_run(model, prompts, pages, n, kv_dtype, capture):
    dec = PromptDecoder(model, max_len=120, batch=len(prompts), max_new=n, kv_dtype=kv_dtype, **pages)
    if capture:
        dec.capture()
    with torch.no_grad():
        lg = [dec.prefill(prompts, chunk=32).clone()]
        lg += [dec.step().clone() for _ in range(n - 1)]
    return lg, dec.generated.clone()


@pytest.mark.parametrize('kv_dtype', [None, E4], ids=['fp16', 'e4m3'])
@pytest.mark.parametrize('kind', [(4, 64), (2, 128), 'opt'])
def test_paged_decoder_on_shuffled_pages_equals_contiguous_and_its_graph_equals_eager(kind, kv_dtype):
    model = _tiny(kind)
    prompts = _prompts((70, 9, 101), seed=9)
    mp = 2                                                     # ceil(120 / 64)
    table = torch.randperm(3 * mp, generator=torch.Generator().manual_seed(3)).to(torch.int32).view(3, mp)
    pages = dict(page_table=table, n_pages=3 * mp)
    want = _decode_run(model, prompts, {}, 12, kv_dtype, capture=True)
    for capture in (True, False):
        got = _decode_run(model, prompts, pages, 12, kv_dtype, capture)
        assert all(torch.equal(_bits(a), _bits(b)) for a, b in zip(got[0], want[0])), capture
        assert torch.equal(got[1], want[1])


@pytest.mark.parametrize('kind', [(4, 64), 'opt'])
def test_generate_paged_without_shared_pages_equals_contiguous_generate(kind):
    model = _tiny(kind)
    prompts = _prompts((70, 9, 101), seed=4)
    for kw in (dict(), dict(do_sample=True, seed=[1, 2, 3], top_k=40), dict(prompt_lookup_num_tokens=3)):
        want = generate(model, prompts, 12, prefill_chunk_size=32, **kw)
        got = generate(model, prompts, 12, prefill_chunk_size=32, share_prompt_prefixes=True, **kw)
        assert all(torch.equal(g, w) for g, w in zip(got, want)), kw


def _agree_away_from_ties(model, prompts, n, kw_a, kw_b, min_checked):
    """Generate with kw_a and kw_b; compare the tokens of each row up to its first near-tie: a position whose top-2
    logit gap is at most twice the largest logit difference of the two runs (the bound of test_gpu_prefill_chunked)."""
    runs = []
    for kw in (kw_a, kw_b):
        plan = None
        dec_kw = dict(max_len=max(len(p) for p in prompts) + n, batch=len(prompts), max_new=n)
        if kw.get('share'):
            from quip_b200.decode import plan_prefix_pages
            table, n_pages, starts = plan_prefix_pages(prompts, [len(p) + n for p in prompts],
                                                       max_pages=-(-dec_kw['max_len'] // KV_PAGE))
            dec_kw.update(page_table=table, n_pages=n_pages)
            plan = starts
        dec = PromptDecoder(model, kv_dtype=kw.get('kv_dtype'), **dec_kw).capture()
        with torch.no_grad():
            lg = [dec.prefill(prompts, chunk=64, starts=plan).float().clone()]
            lg += [dec.step().float().clone() for _ in range(n - 1)]
        runs.append((dec.generated.cpu(), lg))
    (g0, l0), (g1, l1) = runs
    checked = 0
    for b in range(len(prompts)):
        for j in range(n):
            top2 = l0[j][b].topk(2).values
            if float(top2[0] - top2[1]) <= 2 * float((l1[j][b] - l0[j][b]).abs().max()):
                break
            assert int(g0[b, j]) == int(g1[b, j]), (b, j)
            checked += 1
    assert checked >= min_checked, checked


@pytest.mark.parametrize('kv_dtype', [None, E4], ids=['fp16', 'e4m3'])
@pytest.mark.parametrize('kind', [(4, 64), (2, 128)])
def test_shared_prefix_generation_equals_unshared_away_from_near_ties(kind, kv_dtype):
    model = _tiny(kind)
    prompts = _prompts((5, 40, 1, 60), seed=6, prefix=130)       # 2 shared pages
    _agree_away_from_ties(model, prompts, 16, dict(kv_dtype=kv_dtype), dict(kv_dtype=kv_dtype, share=True),
                          16 if kv_dtype is None else 3)


def test_num_return_sequences_equals_the_repeated_prompt_call_and_shares_the_prompt():
    model = _tiny((2, 128))
    prompts = _prompts((150, 75), seed=8)
    n = 4
    got = generate(model, prompts, 10, num_return_sequences=n, do_sample=True, temperature=0.8, seed=5)
    want = generate(model, [p for p in prompts for _ in range(n)], 10, share_prompt_prefixes=True, do_sample=True,
                    temperature=0.8, seed=5)
    assert len(got) == 2 * n and all(torch.equal(g, w) for g, w in zip(got, want))
    _agree_away_from_ties(model, [p for p in prompts for _ in range(n)], 10, dict(), dict(share=True), 20)
