"""The extend-attention kernel (quip_extend_attention, csrc/attn_decode.cu) and kv_append + prefill attention
(quip_kv_append, quip_prefill_attention, csrc/attn_prefill.cu) on exact multi-token cases
(oracle/exact_causal.py), compared bit for bit with fp16_rn(fp32(O) / fp32(L)): every (cache dtype, head_dim, heads per
kv head) instantiation at tokens per row and positions that straddle 64-slot chunks, blocks and query tiles, wide and
long grids, rows out of range, a stale workspace, and the kernels against each other.  The cases are deterministic;
tests/test_exact_causal_cases.py proves each one's budget on the host."""
import ctypes as C
import dataclasses

import numpy as np
import pytest
import torch

from oracle import exact_causal as ec

pytestmark = pytest.mark.gpu

NKV = 2
BLOCK = ec.BLOCK
GRID = [(fp8, hd, G) for fp8 in (False, True) for hd in (64, 128) for G in range(1, 9)]
GRID_IDS = [f'{"e4m3" if f else "fp16"}-hd{hd}-G{G}' for f, hd, G in GRID]
EXTEND_T = (1, 2, 3, 5, 8)
PREFILL_T = (1, 7, 22, 100, 257)


def _dt(fp8):
    return 'e4m3' if fp8 else 'fp16'


# ---- cases ----
def extend_max_lens(T):
    return (T, 3 * BLOCK + 40)


def extend_positions(T, max_len):
    """0, both sides of the first chunk edge (new slots straddling it), 128 - T (ending at the second edge) and
    max_len - T: those a row of T new tokens can take."""
    ps = [0, BLOCK - -(-T // 2), BLOCK - 1, BLOCK, 2 * BLOCK - T, max_len - T]
    return [p for p in dict.fromkeys(ps) if 0 <= p <= max_len - T]


def extend_case(fp8, hd, G, T, max_len):
    seed = 1000 * fp8 + 100 * T + 10 * hd + G + max_len
    return ec.make_case('extend', fp8, hd, G, NKV, max_len, T, extend_positions(T, max_len), seed=seed)


def prefill_rows(T, max_len):
    """(position, count): a full chunk at 0, an empty row, chunks starting just before and at a block edge, one that
    ends at max_len, and a half-counted row."""
    return [(0, T), (5, 0), (BLOCK - 1, T), (BLOCK, max(1, T - 3)), (max_len - T, T), (17, (T + 1) // 2)]


def prefill_case(fp8, hd, G, T):
    max_len = T + 3 * BLOCK + 40
    pos, cnt = zip(*prefill_rows(T, max_len))
    seed = 1000 * fp8 + 7 * T + 10 * hd + G
    return ec.make_case('prefill', fp8, hd, G, NKV, max_len, T, pos, cnt, seed=seed)


def wide_case(fp8):
    """64 rows of 8 kv heads with 8 query heads and 8 tokens each over 4096 slots: up to 64 chunks in the combine."""
    B, nkv, T, max_len = 64, 8, 8, 4096
    pos = np.random.default_rng(64).integers(0, max_len - T + 1, size=B)
    pos[:6] = [max_len - T, 0, BLOCK - 4, BLOCK - 1, 31 * BLOCK - 3, 31 * BLOCK]
    return ec.make_case('extend', fp8, 64, 8, nkv, max_len, T, pos, seed=64 + fp8)


def zlimit_case(fp8):
    """B = 65535 rows, the grid.z limit the argument check accepts."""
    B = 65535
    return ec.make_case('extend', fp8, 64, 3, 1, 2, 2, np.zeros(B, np.int64), seed=7 + fp8)


def long_case(fp8):
    """512 tokens per row at positions up to about 3000, 8 query heads per kv head: 8 query tiles, 55 blocks."""
    max_len = 3000
    rows = [(max_len - 512, 512), (1000, 300), (BLOCK * 20 - 7, 512)]
    pos, cnt = zip(*rows)
    return ec.make_case('prefill', fp8, 128, 8, 1, max_len, 512, pos, cnt, seed=512 + fp8)


def extend_oob_case(fp8, hd, G):
    T, max_len = 3, 3 * BLOCK + 40
    pos = [5, -1, max_len - T + 1, max_len - T, 0, 1 << 40, BLOCK - 1]
    return ec.make_case('extend', fp8, hd, G, NKV, max_len, T, pos, seed=hd + G)


def prefill_oob_case(fp8, hd, G):
    T, max_len = 22, 3 * BLOCK + 40
    rows = [(5, 22), (-1, 4), (9, -1), (30, T + 1), (max_len - 10, 11), (max_len - 22, 22), (0, 0), (BLOCK, 13)]
    pos, cnt = zip(*rows)
    return ec.make_case('prefill', fp8, hd, G, NKV, max_len, T, pos, cnt, seed=hd + G + 3)


def stale_case(fp8):
    return ec.make_case('extend', fp8, 128, 5, NKV, 3 * BLOCK + 40, 5, [0, 60, 64, 200, 227, 123, 1], seed=5 + fp8)


def cross_case(fp8):
    """The extend grid's positions at T = 5, G = 4: one case all three kernels can run."""
    return ec.make_case('extend', fp8, 128, 4, NKV, 3 * BLOCK + 40, 5, extend_positions(5, 3 * BLOCK + 40), seed=45 + fp8)


def chunked_case(fp8):
    T, max_len = 100, 300
    rows = [(0, 100), (BLOCK - 3, 100), (7, 41), (max_len - 100, 100), (130, 0)]
    pos, cnt = zip(*rows)
    return ec.make_case('prefill', fp8, 64, 3, NKV, max_len, T, pos, cnt, seed=100 + fp8)


def cases():
    """Every case of this file, for the host-side tests: (name, thunk that builds it)."""
    for fp8, hd, G in GRID:
        for T in EXTEND_T:
            for max_len in extend_max_lens(T):
                yield (f'extend {_dt(fp8)} hd={hd} G={G} T={T} max_len={max_len}',
                       lambda a=(fp8, hd, G, T, max_len): extend_case(*a))
        for T in PREFILL_T:
            yield f'prefill {_dt(fp8)} hd={hd} G={G} T={T}', lambda a=(fp8, hd, G, T): prefill_case(*a)
    for fp8 in (False, True):
        yield f'wide {_dt(fp8)}', lambda fp8=fp8: wide_case(fp8)
        yield f'grid.z limit {_dt(fp8)}', lambda fp8=fp8: zlimit_case(fp8)
        yield f'long prefill {_dt(fp8)}', lambda fp8=fp8: long_case(fp8)
        for hd, G in ((64, 4), (128, 7)):
            yield f'extend out of range {_dt(fp8)} hd={hd} G={G}', lambda a=(fp8, hd, G): extend_oob_case(*a)
            yield f'prefill out of range {_dt(fp8)} hd={hd} G={G}', lambda a=(fp8, hd, G): prefill_oob_case(*a)
        yield f'stale workspace {_dt(fp8)}', lambda fp8=fp8: stale_case(fp8)
        yield f'cross-kernel {_dt(fp8)}', lambda fp8=fp8: cross_case(fp8)
        yield f'chunked prefill {_dt(fp8)}', lambda fp8=fp8: chunked_case(fp8)


def subcase(c, rows, **kw):
    """The case restricted to `rows` (and with the fields in kw replaced)."""
    rows = np.asarray(rows)
    f = dict(q=c.q[rows], k_new=c.k_new[rows], v_new=c.v_new[rows], k_cache=c.k_cache[rows], v_cache=c.v_cache[rows],
             k_scale=None if c.k_scale is None else c.k_scale[rows],
             v_scale=None if c.v_scale is None else c.v_scale[rows], positions=c.positions[rows],
             counts=c.counts[rows], sel=c.sel[rows], zero=c.zero[rows], kinds=[c.kinds[b] for b in rows])
    f.update(kw)
    return dataclasses.replace(c, **f)


# ---- running a case ----
def _dev(c):
    def t(a):
        return torch.from_numpy(np.ascontiguousarray(a)).cuda()
    d = dict(q=t(c.q), kn=t(c.k_new), vn=t(c.v_new), pos=t(c.positions), cnt=t(c.counts), kc=t(c.k_cache),
             vc=t(c.v_cache))
    if c.fp8:
        d['kc'], d['vc'] = d['kc'].view(torch.float8_e4m3fn), d['vc'].view(torch.float8_e4m3fn)
        d['ks'], d['vs'] = t(c.k_scale), t(c.v_scale)
    return d


def _sc(d):
    return dict(k_scale=d.get('ks'), v_scale=d.get('vs'))


def workspace_bytes(c):
    from quip_b200 import _lib
    B, T, nh, nkv, hd, max_len = c.shape
    need = C.c_size_t(0)
    _lib.check(_lib.load().quip_extend_attention_workspace_bytes(B, T, nh, hd, max_len, C.byref(need)))
    return max(int(need.value), 16)


def run(c, ws=None):
    """One call on fresh device copies of the case -> (out (B, T, nh, hd) fp16 numpy, device tensors after the call).
    Extend: ws a uint8 workspace for a direct call through _lib, None through fused.extend_attention.  Prefill:
    fused.kv_append, then fused.prefill_attention."""
    from quip_b200 import _lib, fused
    d = _dev(c)
    if c.kernel == 'prefill':
        fused.kv_append(d['kn'], d['vn'], d['kc'], d['vc'], d['pos'], d['cnt'], **_sc(d))
        out = fused.prefill_attention(d['q'], d['kc'], d['vc'], d['pos'], d['cnt'], c.scale, **_sc(d))
    elif ws is None:
        out = fused.extend_attention(d['q'], d['kn'], d['vn'], d['kc'], d['vc'], d['pos'], c.scale, **_sc(d))
    else:
        B, T, nh, nkv, hd, max_len = c.shape
        lib = _lib.load()
        out = torch.empty_like(d['q'])
        kv = _lib.QuipKvCache(k=d['kc'].data_ptr(), v=d['vc'].data_ptr(), nkv=nkv, hd=hd, max_len=max_len,
                              format=_lib.QUIP_KV_E4M3 if c.fp8 else _lib.QUIP_KV_FP16)
        if c.fp8:
            kv.k_scale, kv.v_scale = d['ks'].data_ptr(), d['vs'].data_ptr()
        _lib.check(lib.quip_extend_attention(C.byref(kv), *[d[k].data_ptr() for k in ('q', 'kn', 'vn', 'pos')],
                                             out.data_ptr(), B, T, nh, C.c_float(c.scale), ws.data_ptr(), ws.numel(),
                                             torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return out.cpu().numpy(), d


def _which_slot(c, b, h, row):
    """For a one-slot token: the slots of the row (as the kernel should read them, and the decoys the new slots held
    before the call) whose V the output row equals."""
    kv = h // c.G
    hits = []
    for pre, name in ((False, 'slot {}'), (True, 'the decoy of new slot {}')):
        _, V, _, vs = (a[0] for a in c.slots([b], pre=pre))
        cand = (V[kv] * vs[kv][:, None]).astype(np.float16).view(np.uint16)
        js = np.nonzero((cand == row.view(np.uint16)).all(1))[0]
        if pre:
            p = int(c.positions[b])
            js = [j for j in js if p <= j < p + c.count(b)]
        hits += [name.format(int(j)) for j in js]
    return ', '.join(hits) or 'none'


def assert_attention_bits_equal(c, got, want, what):
    """fp16 bit patterns of the valid rows equal (tokens past a count +0); rows out of range are all NaN.  On a
    mismatch report the count, the first (b, i, h, d), the token's visible |S|, and for a one-slot token the slot whose
    V the output equals."""
    valid = np.array([c.valid(b) for b in range(len(c.positions))])
    assert np.isnan(got[~valid].astype(np.float32)).all(), f'{what}: a row out of range is not all NaN'
    g, w = got[valid].view(np.uint16), want[valid].view(np.uint16)
    if np.array_equal(g, w):
        return
    bad = np.argwhere(g != w)
    rows = np.nonzero(valid)[0]
    b, i, h, d = int(rows[bad[0][0]]), int(bad[0][1]), int(bad[0][2]), int(bad[0][3])
    vis, _ = ec.visible(c, [b])
    S = np.nonzero(vis[0, i, h])[0]
    msg = (f'{what}: {len(bad)} of {g.size} outputs differ from fp16(fp32(O) / fp32(L)); first at (b, i, h, d) = '
           f'({b}, {i}, {h}, {d}), position {int(c.positions[b])}, count {int(c.counts[b])}, head kind '
           f'{c.kinds[b][h]}{" with q = 0" if c.zero[b, i, h] else ""}, visible |S| = {len(S)}: got {got[b, i, h, d]!r} '
           f'want {want[b, i, h, d]!r}')
    if len(S) == 1:
        msg += f'; S = {{{int(S[0])}}}, the output row equals the V of {_which_slot(c, b, h, got[b, i, h])}'
    raise AssertionError(msg)


def assert_cache_after(c, d, what):
    """Only slots positions[b] .. positions[b] + count - 1 of each valid row changed, to the new tokens (e4m3: their
    kvfp8.quantize)."""
    for name, want in zip(('kc', 'vc', 'ks', 'vs'), c.caches_after()):
        if want is None:
            continue
        got = d[name].cpu()
        got = got.view(torch.uint8) if got.dtype == torch.float8_e4m3fn else got.view(torch.int16) if got.dtype == torch.float16 else got
        want = torch.from_numpy(want)
        want = want.view(torch.int16) if want.dtype == torch.float16 else want
        if not torch.equal(got, want):
            bad = (got != want).nonzero()[0].tolist()
            raise AssertionError(f'{what}: {name} differs after the call at {bad} (position {c.positions[bad[0]]}, '
                                 f'count {c.counts[bad[0]]})')


def check(c, what, ws=None):
    want, _ = ec.reference(c)
    got, d = run(c, ws)
    assert_attention_bits_equal(c, got, want, what)
    assert_cache_after(c, d, what)
    return got


# ---- every instantiation ----
@pytest.mark.parametrize('fp8,hd,G', GRID, ids=GRID_IDS)
def test_extend_every_instantiation_bit_exact(fp8, hd, G):
    for T in EXTEND_T:
        for max_len in extend_max_lens(T):
            check(extend_case(fp8, hd, G, T, max_len), f'extend {_dt(fp8)} hd={hd} G={G} T={T} max_len={max_len}')


@pytest.mark.parametrize('fp8,hd,G', GRID, ids=GRID_IDS)
def test_prefill_every_instantiation_bit_exact(fp8, hd, G):
    for T in PREFILL_T:
        check(prefill_case(fp8, hd, G, T), f'prefill {_dt(fp8)} hd={hd} G={G} T={T}')


# ---- wide and long grids ----
@pytest.mark.parametrize('fp8', [False, True], ids=['fp16', 'e4m3'])
def test_extend_wide_grid_bit_exact(fp8):
    check(wide_case(fp8), f'wide extend {_dt(fp8)}')


@pytest.mark.parametrize('fp8', [False, True], ids=['fp16', 'e4m3'])
def test_extend_grid_z_limit_bit_exact(fp8):
    check(zlimit_case(fp8), f'extend B = 65535 {_dt(fp8)}')


@pytest.mark.parametrize('fp8', [False, True], ids=['fp16', 'e4m3'])
def test_prefill_long_chunk_bit_exact(fp8):
    check(long_case(fp8), f'long prefill {_dt(fp8)}')


# ---- rows out of range ----
@pytest.mark.parametrize('fp8,hd,G', [(f, hd, G) for f in (False, True) for hd, G in ((64, 4), (128, 7))])
def test_extend_out_of_range_rows_give_nan_and_write_nothing(fp8, hd, G):
    """Rows at -1, max_len - T + 1 and 2^40 come out all NaN and leave their cache bytes and scales alone; the valid
    rows equal a run of them alone, bit for bit."""
    c = extend_oob_case(fp8, hd, G)
    got = check(c, f'extend out of range {_dt(fp8)} hd={hd} G={G}')
    rows = np.array([b for b in range(len(c.positions)) if c.valid(b)])
    assert 0 < len(rows) < len(c.positions)
    alone = check(subcase(c, rows), 'the valid rows alone')
    assert np.array_equal(alone.view(np.uint16), got[rows].view(np.uint16))


@pytest.mark.parametrize('fp8,hd,G', [(f, hd, G) for f in (False, True) for hd, G in ((64, 4), (128, 7))])
def test_prefill_invalid_rows_give_nan_and_write_nothing(fp8, hd, G):
    """Rows with pos < 0, count < 0, count > T or pos + count > max_len come out all NaN and write nothing."""
    c = prefill_oob_case(fp8, hd, G)
    assert sum(not c.valid(b) for b in range(len(c.positions))) == 4
    check(c, f'prefill invalid rows {_dt(fp8)} hd={hd} G={G}')


# ---- stale workspace ----
@pytest.mark.parametrize('fp8', [False, True], ids=['fp16', 'e4m3'])
def test_extend_descriptor_launch_combine_reads_only_its_own_partials(fp8):
    """A workspace of NaN bytes (0xFF), then one left by a call with every row at max_len - T (all chunks written):
    both give the clean result bit for bit."""
    c = stale_case(fp8)
    clean = check(c, 'clean workspace')
    nan_ws = torch.full((workspace_bytes(c),), 0xFF, dtype=torch.uint8, device='cuda')
    got = check(c, 'NaN workspace', ws=nan_ws)
    assert np.array_equal(got.view(np.uint16), clean.view(np.uint16))
    B, T, nh, nkv, hd, max_len = c.shape
    full = ec.make_case('extend', fp8, 128, 5, NKV, max_len, T, [max_len - T] * B, seed=99)
    used = torch.zeros((workspace_bytes(c),), dtype=torch.uint8, device='cuda')
    check(full, 'every chunk of every row', ws=used)
    got = check(c, 'workspace of an earlier call at larger positions', ws=used)
    assert np.array_equal(got.view(np.uint16), clean.view(np.uint16))


# ---- the kernels against each other (each equals the reference, so they equal each other) ----
@pytest.mark.parametrize('fp8', [False, True], ids=['fp16', 'e4m3'])
def test_decode_extend_and_prefill_agree_bit_for_bit(fp8):
    from quip_b200 import fused
    c = cross_case(fp8)
    ext = check(c, f'cross-kernel extend {_dt(fp8)}')
    pre = check(dataclasses.replace(c, kernel='prefill'), f'cross-kernel prefill {_dt(fp8)}')
    assert np.array_equal(pre.view(np.uint16), ext.view(np.uint16))
    d = _dev(c)
    dec = fused.decode_attention(d['q'][:, 0].contiguous(), d['kn'][:, 0].contiguous(), d['vn'][:, 0].contiguous(),
                                 d['kc'], d['vc'], d['pos'], c.scale, **_sc(d))
    dec = dec.cpu().numpy()
    assert np.array_equal(dec.view(np.uint16), ext[:, 0].view(np.uint16)), 'decode differs from token 0 of extend'


@pytest.mark.parametrize('fp8', [False, True], ids=['fp16', 'e4m3'])
def test_prefill_in_chunks_equals_one_call(fp8):
    """The prompt appended and attended C tokens at a time (C = 1, 5, 64) gives the one-call output and cache bits."""
    from quip_b200 import fused
    c = chunked_case(fp8)
    one = check(c, f'one call {_dt(fp8)}')
    B, T, nh, nkv, hd, max_len = c.shape
    for C_ in (1, 5, 64):
        d = _dev(c)
        outs = []
        for s in range(0, T, C_):
            e = min(T, s + C_)
            pos = d['pos'] + s
            cnt = (d['cnt'] - s).clamp(0, e - s)
            kn, vn = d['kn'][:, s:e].contiguous(), d['vn'][:, s:e].contiguous()
            fused.kv_append(kn, vn, d['kc'], d['vc'], pos, cnt, **_sc(d))
            outs.append(fused.prefill_attention(d['q'][:, s:e].contiguous(), d['kc'], d['vc'], pos, cnt, c.scale,
                                                **_sc(d)))
        got = torch.cat(outs, 1).cpu().numpy()
        torch.cuda.synchronize()
        assert_attention_bits_equal(c, got, one, f'chunks of {C_} {_dt(fp8)}')
        assert_cache_after(c, d, f'chunks of {C_} {_dt(fp8)}')
