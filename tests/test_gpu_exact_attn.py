"""The decode-attention kernels (quip_decode_attention on fp16 and e4m3 caches, csrc/attn_decode.cu) on exact
cases (oracle/exact_attn.py), compared bit for bit with fp16_rn(fp32(O) / fp32(L)): every (cache dtype, head_dim, heads
per kv head) instantiation at both chunk sizes, the cache after the append, a wide grid, the grid.z limit, positions
out of range, and a stale workspace.  The cases are deterministic; tests/test_exact_attn_cases.py proves each one's
budget on the host."""
import ctypes as C

import numpy as np
import pytest
import torch

from oracle import exact_attn as ea

from test_gpu_generate import CHUNK, _chunk

pytestmark = pytest.mark.gpu

NKV = 2
MAX_LENS = [1, 37, 3 * CHUNK + 40]
GRID = [(fp8, hd, G) for fp8 in (False, True) for hd in (64, 128) for G in range(1, 9)]


def rows_for(chunk, max_len):
    """A row count at which the kernel takes `chunk`-slot chunks for NKV kv heads and max_len slots."""
    B = 7 if chunk == 64 else -(-2 * 132 // (NKV * -(-max_len // CHUNK)))
    assert _chunk(B, NKV, max_len) == chunk
    return B


def edge_positions(B, chunk, max_len, seed):
    """0, chunk - 1, chunk, chunk + 1, both sides of the last chunk start and max_len - 1 (those in range), then random."""
    last = (-(-max_len // chunk) - 1) * chunk
    edge = [p for p in dict.fromkeys([0, chunk - 1, chunk, chunk + 1, last - 1, last, max_len - 1]) if 0 <= p < max_len]
    rng = np.random.default_rng(seed)
    return (edge + [int(p) for p in rng.integers(0, max_len, size=B)])[:B]


def grid_case(fp8, hd, G, chunk, max_len):
    B = rows_for(chunk, max_len)
    seed = 1000 * fp8 + 10 * hd + G + chunk + max_len
    return ea.make_case(fp8, hd, G, NKV, max_len, edge_positions(B, chunk, max_len, seed), chunk, seed)


def wide_case(fp8):
    """64 rows of 8 kv heads with 8 query heads each over 4096 slots: 32 chunks per row in the combine."""
    B, nkv, max_len = 64, 8, 4096
    pos = np.random.default_rng(64).integers(0, max_len, size=B)
    pos[:6] = [max_len - 1, 0, CHUNK - 1, CHUNK, 31 * CHUNK - 1, 31 * CHUNK]
    return ea.make_case(fp8, 64, 8, nkv, max_len, pos, _chunk(B, nkv, max_len), seed=64 + fp8)


def zlimit_case(fp8):
    """B = 65535 rows, the grid.z limit the argument check accepts."""
    B = 65535
    return ea.make_case(fp8, 64, 3, 1, 1, np.zeros(B, np.int64), _chunk(B, 1, 1), seed=7 + fp8)


def oob_case(fp8, hd, G):
    max_len = 3 * CHUNK + 40
    pos = [5, -1, max_len - 1, max_len, 0, 1 << 40, CHUNK]
    return ea.make_case(fp8, hd, G, NKV, max_len, pos, _chunk(len(pos), NKV, max_len), seed=hd + G)


def cases():
    """Every case of this file, for the host-side tests: (name, thunk that builds it)."""
    for fp8, hd, G in GRID:
        for chunk in (64, 128):
            for max_len in MAX_LENS:
                yield (f'grid fp8={fp8} hd={hd} G={G} chunk={chunk} max_len={max_len}',
                       lambda a=(fp8, hd, G, chunk, max_len): grid_case(*a))
    for fp8 in (False, True):
        yield f'wide fp8={fp8}', lambda fp8=fp8: wide_case(fp8)
        yield f'grid.z limit fp8={fp8}', lambda fp8=fp8: zlimit_case(fp8)
        for hd, G in ((64, 4), (128, 7)):
            yield f'out of range fp8={fp8} hd={hd} G={G}', lambda a=(fp8, hd, G): oob_case(*a)
        yield f'stale workspace fp8={fp8}', lambda fp8=fp8: stale_case(fp8)


# ---- running a case ----
def _dev(c):
    def t(a):
        return torch.from_numpy(np.ascontiguousarray(a)).cuda()
    d = dict(q=t(c.q), kn=t(c.k_new), vn=t(c.v_new), pos=t(c.positions), kc=t(c.k_cache), vc=t(c.v_cache))
    if c.fp8:
        d['kc'], d['vc'] = d['kc'].view(torch.float8_e4m3fn), d['vc'].view(torch.float8_e4m3fn)
        d['ks'], d['vs'] = t(c.k_scale), t(c.v_scale)
    return d


def workspace_bytes(c):
    from quip_b200 import _lib
    B, nh, nkv, hd, max_len = c.shape
    need = C.c_size_t(0)
    _lib.check(_lib.load().quip_decode_attention_workspace_bytes(B, nh, hd, max_len, C.byref(need)))
    return max(int(need.value), 16)


def run(c, ws=None):
    """One kernel call on fresh device copies of the case -> (out (B, nh, hd) fp16 numpy, device tensors after the
    call).  ws: a uint8 workspace for a direct call through _lib; None goes through fused.decode_attention."""
    from quip_b200 import _lib, fused
    d = _dev(c)
    if ws is None:
        out = fused.decode_attention(d['q'], d['kn'], d['vn'], d['kc'], d['vc'], d['pos'], c.scale,
                                     k_scale=d.get('ks'), v_scale=d.get('vs'))
    else:
        B, nh, nkv, hd, max_len = c.shape
        lib = _lib.load()
        out = torch.empty_like(d['q'])
        kv = _lib.QuipKvCache(k=d['kc'].data_ptr(), v=d['vc'].data_ptr(), nkv=nkv, hd=hd, max_len=max_len,
                              format=_lib.QUIP_KV_E4M3 if c.fp8 else _lib.QUIP_KV_FP16)
        if c.fp8:
            kv.k_scale, kv.v_scale = d['ks'].data_ptr(), d['vs'].data_ptr()
        _lib.check(lib.quip_decode_attention(C.byref(kv), *[d[k].data_ptr() for k in ('q', 'kn', 'vn', 'pos')],
                                             out.data_ptr(), B, nh, C.c_float(c.scale), ws.data_ptr(), ws.numel(),
                                             torch.cuda.current_stream().cuda_stream))
    torch.cuda.synchronize()
    return out.cpu().numpy(), d


def _which_slot(c, b, h, row):
    """For a one-slot head: the slot (of the row, as the kernel should read it) whose V the output row equals."""
    _, V, _, vs = (a[0] for a in ea.row_slots(c, [b]))
    kv = h // c.G
    cand = (V[kv] * vs[kv][:, None]).astype(np.float16)
    hit = np.nonzero((cand.view(np.uint16) == row.view(np.uint16)).all(1))[0]
    _, Vp, _, vsp = (a[0] for a in ea.row_slots(c, [b], pre=True))
    p = int(c.positions[b])
    stale = np.array_equal((Vp[kv, p] * vsp[kv, p]).astype(np.float16).view(np.uint16), row.view(np.uint16))
    return ', '.join([f'slot {int(j)}' for j in hit] + (['the cache slot pos before the append'] if stale else [])) or 'none'


def assert_attention_bits_equal(c, got, want, what):
    """fp16 bit patterns of the valid rows equal; rows out of range are all NaN.  On a mismatch report the count, the
    first (b, h, d), the chunk, the head's selected set, and for a one-slot head the slot whose V the output equals."""
    valid = np.array([c.valid(b) for b in range(len(c.positions))])
    assert np.isnan(got[~valid].astype(np.float32)).all(), f'{what}: a row out of range is not all NaN'
    g, w = got[valid].view(np.uint16), want[valid].view(np.uint16)
    if np.array_equal(g, w):
        return
    bad = np.argwhere(g != w)
    rows = np.nonzero(valid)[0]
    b, h, d = int(rows[bad[0][0]]), int(bad[0][1]), int(bad[0][2])
    S = np.nonzero(c.sel[b, h])[0]
    msg = (f'{what}: {len(bad)} of {g.size} outputs differ from fp16(fp32(O) / fp32(L)); first at (b, h, d) = '
           f'({b}, {h}, {d}), chunk {c.chunk}, position {int(c.positions[b])}, head kind {c.kinds[b][h]}, |S| = {len(S)}: '
           f'got {got[b, h, d]!r} want {want[b, h, d]!r}')
    if len(S) == 1:
        msg += f'; S = {{{int(S[0])}}}, the output row equals the V of {_which_slot(c, b, h, got[b, h])}'
    raise AssertionError(msg)


def assert_cache_after(c, d, what):
    """Only slot positions[b] of each valid row changed: k_new / v_new for fp16, kvfp8.quantize of them for e4m3."""
    kc, vc = c.k_cache.copy(), c.v_cache.copy()
    ks = None if c.k_scale is None else c.k_scale.copy()
    vs = None if c.v_scale is None else c.v_scale.copy()
    if c.fp8:
        kq, kqs, vq, vqs = c.new_quantized()
    for b in range(len(c.positions)):
        if not c.valid(b):
            continue
        p = int(c.positions[b])
        if c.fp8:
            kc[b, :, p], vc[b, :, p], ks[b, :, p], vs[b, :, p] = kq[b], vq[b], kqs[b], vqs[b]
        else:
            kc[b, :, p], vc[b, :, p] = c.k_new[b], c.v_new[b]
    for name, want in (('kc', kc), ('vc', vc), ('ks', ks), ('vs', vs)):
        if want is None:
            continue
        got = d[name].cpu()
        got = got.view(torch.uint8) if got.dtype == torch.float8_e4m3fn else got.view(torch.int16) if got.dtype == torch.float16 else got
        want = torch.from_numpy(want)
        want = want.view(torch.int16) if want.dtype == torch.float16 else want
        if not torch.equal(got, want):
            bad = (got != want).nonzero()[0].tolist()
            raise AssertionError(f'{what}: {name} differs after the call at {bad} (positions {c.positions[bad[0]]})')


def check(c, what, ws=None):
    want, _ = ea.reference(c)
    got, d = run(c, ws)
    assert_attention_bits_equal(c, got, want, what)
    assert_cache_after(c, d, what)
    return got


# ---- every instantiation at both chunk sizes ----
@pytest.mark.parametrize('fp8,hd,G', GRID, ids=[f'{"e4m3" if f else "fp16"}-hd{hd}-G{G}' for f, hd, G in GRID])
def test_every_instantiation_bit_exact(fp8, hd, G):
    for chunk in (64, 128):
        for max_len in MAX_LENS:
            c = grid_case(fp8, hd, G, chunk, max_len)
            check(c, f'{"e4m3" if fp8 else "fp16"} hd={hd} G={G} chunk={chunk} max_len={max_len}')


# ---- wide grids ----
@pytest.mark.parametrize('fp8', [False, True], ids=['fp16', 'e4m3'])
def test_wide_grid_bit_exact(fp8):
    c = wide_case(fp8)
    assert c.chunk == CHUNK and int(c.positions.max()) // CHUNK + 1 == 32
    check(c, f'wide {"e4m3" if fp8 else "fp16"}')


@pytest.mark.parametrize('fp8', [False, True], ids=['fp16', 'e4m3'])
def test_grid_z_limit_bit_exact(fp8):
    check(zlimit_case(fp8), f'B = 65535 {"e4m3" if fp8 else "fp16"}')


# ---- positions out of range ----
@pytest.mark.parametrize('fp8,hd,G', [(f, hd, G) for f in (False, True) for hd, G in ((64, 4), (128, 7))])
def test_out_of_range_positions_give_nan_rows_and_write_nothing(fp8, hd, G):
    """Rows at -1, max_len and 2^40 come out all NaN and leave their cache bytes and scales alone (assert_cache_after);
    the valid rows equal a run without them, bit for bit."""
    c = oob_case(fp8, hd, G)
    got = check(c, f'out of range {"e4m3" if fp8 else "fp16"} hd={hd} G={G}')
    rows = np.array([b for b in range(len(c.positions)) if c.valid(b)])
    assert len(rows) < len(c.positions)
    sub = ea.AttnCase(c.fp8, _chunk(len(rows), NKV, c.shape[4]), c.scale, c.q[rows], c.k_new[rows], c.v_new[rows],
                      c.k_cache[rows], c.v_cache[rows], None if c.k_scale is None else c.k_scale[rows],
                      None if c.v_scale is None else c.v_scale[rows], c.positions[rows], c.sel[rows],
                      [c.kinds[b] for b in rows])
    alone = check(sub, 'the valid rows alone')
    assert np.array_equal(alone.view(np.uint16), got[rows].view(np.uint16))


# ---- stale workspace ----
def stale_case(fp8):
    return ea.make_case(fp8, 128, 5, NKV, 3 * CHUNK + 40, [0, 63, 64, 200, 300, 423, 1], 64, seed=5 + fp8)


@pytest.mark.parametrize('fp8', [False, True], ids=['fp16', 'e4m3'])
def test_descriptor_launch_combine_reads_only_its_own_partials(fp8):
    """A workspace of NaN bytes (0xFF), then one left by a call with every row at max_len - 1 (all chunks written):
    both give the clean result bit for bit."""
    c = stale_case(fp8)
    clean = check(c, 'clean workspace')
    nan_ws = torch.full((workspace_bytes(c),), 0xFF, dtype=torch.uint8, device='cuda')
    got = check(c, 'NaN workspace', ws=nan_ws)
    assert np.array_equal(got.view(np.uint16), clean.view(np.uint16))
    full = ea.make_case(fp8, 128, 5, NKV, c.shape[4], [c.shape[4] - 1] * len(c.positions), c.chunk, seed=99)
    used = torch.zeros((workspace_bytes(c),), dtype=torch.uint8, device='cuda')
    check(full, 'every chunk of every row', ws=used)
    got = check(c, 'workspace of an earlier call at larger positions', ws=used)
    assert np.array_equal(got.view(np.uint16), clean.view(np.uint16))
