"""Host-side logic and the C-ABI surface, CPU only (no compute calls into the CUDA library)."""
import os
import re

import numpy as np
import pytest
import torch
import torch.nn as nn

from conftest import GOLDEN, LAYER_NAMES, ROOT, load_layer, parts_to_torch
from oracle import butterfly as obf
from oracle import forward as ofw
from oracle import packing as opk
from quip_b200 import _lib
from quip_b200 import quant as Q
from quip_b200.incoherence import plan_side


def test_library_exports_every_declared_symbol_of_abi_v3():
    header = open(os.path.join(ROOT, 'include', 'quip_b200.h')).read()
    declared = set(re.findall(r'\b(quip_[a-z_0-9]+)\s*\(', header))
    assert declared, 'no declarations parsed'
    lib = _lib.load()
    for name in declared:
        assert hasattr(lib, name), f'{name} declared in include/quip_b200.h but not exported'
    assert declared == set(_lib.EXPORTS), declared ^ set(_lib.EXPORTS)
    assert lib.quip_abi_version() == _lib.ABI_VERSION == 3
    assert lib.quip_packed_words(16, 128, 2) == 128
    assert lib.quip_packed_words(16, 128, 3) == 192
    assert lib.quip_packed_words(16, 100, 2) == 0          # bad shape -> 0


def test_argument_errors_surface_as_messages():
    lib = _lib.load()
    rc = lib.quip_pack_codes(None, 16, 100, 2, None, None)   # K % 128 != 0: rejected before any CUDA call
    assert rc == 1
    assert b'multiple of 128' in lib.quip_last_error()
    with pytest.raises(_lib.QuipError):
        _lib.check(rc)
    # glue entry points: shape / alignment / null checks come before any launch
    assert lib.quip_rmsnorm(64, None, 64, None, 64, 4, 12, 1e-5, None) == 1 and b'multiple of 8' in lib.quip_last_error()
    assert lib.quip_rmsnorm(64, None, 64, 64, 64, 4, 16, 1e-5, None) == 1 and b'without a residual' in lib.quip_last_error()
    assert lib.quip_rmsnorm(64, None, 68, None, 64, 4, 16, 1e-5, None) == 1 and b'aligned' in lib.quip_last_error()
    assert lib.quip_rmsnorm(None, None, 64, None, 64, 4, 16, 1e-5, None) == 1 and b'null' in lib.quip_last_error()
    assert lib.quip_rmsnorm(64, None, 64, None, 64, 0, 16, 1e-5, None) == 0          # no rows: nothing to launch
    assert lib.quip_rope(64, 64, 64, 64, 4, 4, 4, 24, None) == 1 and b'multiple of 16' in lib.quip_last_error()
    assert lib.quip_rope(64, None, 64, 64, 4, 4, 4, 16, None) == 1 and b'head counts' in lib.quip_last_error()
    assert lib.quip_rope(64, None, 64, 64, 0, 4, 0, 16, None) == 0
    assert lib.quip_silu_mul(64, 64, 64, 12, None) == 1 and b'multiple of 8' in lib.quip_last_error()
    assert lib.quip_silu_mul(64, 64, 64, 0, None) == 0


@pytest.mark.parametrize('bits', [2, 3, 4])
def test_host_packer_matches_oracle_layout(bits):
    rng = np.random.default_rng(bits)
    codes = rng.integers(0, 1 << bits, size=(48, 384), dtype=np.uint8)
    q = Q.pack_codes(torch.from_numpy(codes), bits)
    np.testing.assert_array_equal(q.numpy(), opk.native_pack(codes, bits))
    np.testing.assert_array_equal(Q.unpack_codes(q, 48, 384, bits).numpy(), codes)
    with pytest.raises(ValueError):
        Q.packed_words(20, 384, bits)


def test_quantizer_matches_reference_outputs():
    z = np.load(os.path.join(GOLDEN, 'quantizer.npz'))
    for bits in (2, 3, 4):
        w = torch.from_numpy(z[f'w{bits}'])
        qz = Q.Quantizer()
        qz.configure(bits, perchannel=True, sym=False, qfn='a', mse=False)
        assert not qz.ready()
        qz.find_params(w, weight=True)
        assert qz.ready() and qz.enabled()
        np.testing.assert_array_equal(qz.scale.numpy(), z[f'scale{bits}'])
        np.testing.assert_array_equal(qz.zero.numpy(), z[f'zero{bits}'])
        np.testing.assert_array_equal(qz.quantize(w).numpy(), z[f'qa{bits}'])
        qb = Q.Quantizer()
        qb.configure(bits, perchannel=True, sym=False, qfn='b', mse=False)
        qb.find_params(w, weight=True)
        assert qb.scale is None                      # quant.py:138-142
        np.testing.assert_array_equal(qb.quantize(w).numpy(), z[f'qb{bits}'])
        np.testing.assert_array_equal(qb.scale.numpy(), z[f'sb{bits}'])


@pytest.mark.parametrize('name', [n for n in LAYER_NAMES if n not in ('l4b_plain', 'l3b_rescale')])
def test_side_plans_match_oracle(name):
    parts, _ = load_layer(name)
    tp = parts_to_torch(parts)
    for side, bfly, n in (('V', tp.V, tp.codes.shape[1]), ('U', tp.U, tp.codes.shape[0])):
        plan = plan_side(bfly, side)
        ref = obf.side_plan(parts[side], n, side)
        assert plan.layout == ref['layout']
        np.testing.assert_array_equal(plan.order.numpy(), ref['order'])
        want_idx = ref['io_idx'] if side == 'V' else np.argsort(ref['io_idx'])
        got_idx = np.arange(n) if plan.idx is None else plan.idx.numpy()
        np.testing.assert_array_equal(got_idx, want_idx)
        for ps, (F, p, nblk, strided) in zip(plan.passes, ref['passes']):
            assert (ps.p, ps.nblk, ps.strided) == (p, nblk, strided)
            np.testing.assert_array_equal(ps.factors.numpy(), F)


@pytest.mark.parametrize('name', LAYER_NAMES)
def test_quantlinear_pack_parts_and_state_dict(name):
    parts, z = load_layer(name)
    tp = parts_to_torch(parts)
    N, K = tp.codes.shape
    spec = Q.spec_from_parts(tp)
    ql = Q.QuantLinear(infeatures=K, outfeatures=N, **spec)
    ql.pack_parts(tp)
    # integer codes: bit-exact against the reference's, under the known layout permutation
    plan = ofw.kernel_plan(parts)
    np.testing.assert_array_equal(ql.codes().numpy(), plan['codes'])
    np.testing.assert_array_equal(ql.qweight.numpy(), opk.native_pack(plan['codes'], parts['bits']))
    assert bool(ql.meta[1]) == (parts['qfn'] == 'b')
    # state_dict round trip into a freshly constructed module
    ql2 = Q.QuantLinear(infeatures=K, outfeatures=N, **spec)
    ql2.load_state_dict(ql.state_dict())
    for k, v in ql.state_dict().items():
        assert torch.equal(v, ql2.state_dict()[k]), k
    with pytest.raises(RuntimeError):
        ql(torch.zeros(1, K, dtype=torch.float16))         # no CPU path
    with pytest.raises(ValueError):
        ql(torch.zeros(1, K + 1, dtype=torch.float16))


def test_pack_reference_contract_qfna():
    """Quant3Linear.pack contract (quant.py:185-191): grid weights + quantizer scale/zero -> codes."""
    parts, z = load_layer('l4b_plain')
    N, K = parts['codes'].shape
    lin = nn.Linear(K, N)
    lin.weight.data = torch.from_numpy(z['W_ref']).float()          # no incoherence: W_ref is the grid itself
    lin.bias.data = torch.from_numpy(parts['bias']).float()
    ql = Q.QuantLinear(4, K, N, bias=True)
    ql.pack(lin, torch.from_numpy(z['raw_scale']), torch.from_numpy(z['raw_zero']))
    np.testing.assert_array_equal(ql.codes().numpy(), parts['codes'])
    np.testing.assert_allclose(ql.zeros.numpy(), z['raw_zero'] * z['raw_scale'])
    bad = nn.Linear(K, N)
    with pytest.raises(ValueError):
        Q.QuantLinear(4, K, N, incoh='blocked').pack(bad, torch.ones(N, 1), torch.zeros(N, 1))


def test_make_quant_swaps_exactly_the_named_layers():
    class Block(nn.Module):
        def __init__(self):
            super().__init__()
            self.q_proj = nn.Linear(128, 128)
            self.fc1 = nn.Linear(128, 256, bias=False)
            self.keep = nn.Linear(128, 128)

    class Net(nn.Module):
        def __init__(self):
            super().__init__()
            self.layers = nn.ModuleList([Block(), Block()])
            self.lm_head = nn.Linear(128, 512)

    net = Net()
    names = ['layers.0.q_proj', 'layers.1.fc1']
    Q.make_quant(net, names, bits=2)
    assert isinstance(net.layers[0].q_proj, Q.QuantLinear) and net.layers[0].q_proj.bias is not None
    assert isinstance(net.layers[1].fc1, Q.QuantLinear) and net.layers[1].fc1.bias is None
    assert type(net.layers[0].fc1) is nn.Linear and type(net.layers[1].q_proj) is nn.Linear
    assert type(net.layers[0].keep) is nn.Linear and type(net.lm_head) is nn.Linear
    assert net.layers[1].fc1.infeatures == 128 and net.layers[1].fc1.outfeatures == 256
    Q.make_quant(net, names, bits=2)                           # idempotent on already-swapped modules
    Q.make_quant3(net, ['layers.0.keep'])
    assert net.layers[0].keep.bits == 3
    with pytest.raises(NotImplementedError):
        Q.QuantLinear(8, 128, 128)


def test_fragment_order_matches_the_header_formula():
    """QuipPass.factors_frag (include/quip_b200.h): word (((blk*(p/8) + nt)*(p/32) + j)*32 + lane)*4 + q holds
    F[blk][8nt + lane/4][k0], [k0+1] with k0 = 32j + 16(q/2) + 8(q%2) + 2(lane%4)."""
    import numpy as np
    import torch
    from quip_b200.quant import fragment_order
    for nblk, p in [(3, 64), (2, 32)]:
        f = torch.arange(nblk * p * p, dtype=torch.float32).reshape(nblk, p, p).half()
        frag = fragment_order(f).reshape(-1, 2).numpy()              # words of two halves
        F_ = f.numpy()
        rng = np.random.default_rng(p)
        for _ in range(200):
            blk, nt, j = rng.integers(nblk), rng.integers(p // 8), rng.integers(p // 32)
            lane, q = rng.integers(32), rng.integers(4)
            word = (((blk * (p // 8) + nt) * (p // 32) + j) * 32 + lane) * 4 + q
            k0 = 32 * j + 16 * (q // 2) + 8 * (q % 2) + 2 * (lane % 4)
            row = 8 * nt + lane // 4
            assert frag[word, 0] == F_[blk, row, k0] and frag[word, 1] == F_[blk, row, k0 + 1]


def test_abi_v3_keeps_the_optional_pointers_of_v2():
    from quip_b200 import _lib
    assert 'factors_frag' in [n for n, _ in _lib.QuipPass._fields_]
    assert 'inv_idx' in [n for n, _ in _lib.QuipSide._fields_]
    s = _lib.QuipSide()
    assert not s.inv_idx and not s.passes[0].factors_frag          # NULL by default: the C side takes the unfused routes
    hdr = open(os.path.join(ROOT, 'include', 'quip_b200.h')).read()
    assert 'QUIP_ABI_VERSION 3' in hdr and 'factors_frag' in hdr and 'inv_idx' in hdr


def test_committed_bench_line_has_the_contract_keys():
    """tests/golden/bench_line_h100.json is the JSON line bench.py printed on an H100 (80 GB HBM3, 400 W power limit):
    every key a consumer of the line reads is there."""
    import json
    path = os.path.join(ROOT, 'tests', 'golden', 'bench_line_h100.json')
    line = [l for l in open(path).read().splitlines() if l.strip().startswith('{')][-1]
    d = json.loads(line)
    for k in ('metric', 'value', 'unit', 'n_gpus', 'steps', 'warmup', 'ms_per_step', 'higher_is_better', 'scaling',
              'vs_baseline', 'dtype', 'data', 'config', 'e2e', 'gpu_launches', 'clocks', 'roofline', 'cpu_baseline'):
        assert k in d, k
    assert d['warmup'] >= 3 and d['higher_is_better'] is True and d['scaling'] == 'weak' and d['vs_baseline'] is None
    assert 'workload' in d['config'] and 'l2' in d['config'] and 'model' not in d['config']
    assert set(d['e2e']) >= {'value', 'unit', 'h2d_bytes_per_step', 'd2h_bytes_per_step'} and d['e2e']['h2d_bytes_per_step'] > 0
    r = d['roofline']
    assert r['bound'] in ('hbm', 'tensor') and abs(r['frac'] - r['achieved'] / r['peak']) < 1e-9 and 0 < r['frac'] <= 1
    assert set(d['cpu_baseline']) >= {'value', 'unit', 'cores', 'kind', 'sample'} and d['cpu_baseline']['kind'] in ('port', 'reference')
    assert d['gpu_launches'] > 0 and {'sm_mhz', 'sm_max_mhz', 'reasons'} <= set(d['clocks'])
    assert abs(d['value'] - d['n_gpus'] * d['steps'] * 2048 / (d['ms_per_step'] * d['steps'] / 1e3)) / d['value'] < 1e-6


def test_clock_sampler_summarises_only_rows_inside_the_timed_region():
    import importlib.util
    spec = importlib.util.spec_from_file_location('bench_mod', os.path.join(ROOT, 'bench.py'))
    bench = importlib.util.module_from_spec(spec)
    spec.loader.exec_module(bench)
    clk = bench.ClockSampler(0)
    row = lambda mhz, cap: [str(mhz), '1965', '700.0', 'Not Active', 'Not Active', 'Not Active', cap]
    clk.all_rows = [(1.0, row(1200, 'Not Active')), (5.0, row(1950, 'Active')), (5.2, row(1965, 'Not Active')),
                    (9.0, row(900, 'Not Active'))]
    clk.t0, clk.t1 = 4.9, 5.3
    s = clk.summary()
    assert s['samples'] == 2 and s['sm_mhz'] == 1965.0 and s['sm_max_mhz'] == 1965.0 and s['reasons'] == ['sw_power_cap']
    clk.t0, clk.t1 = 20.0, 21.0                       # nothing landed inside: fall back to the last rows, never crash
    assert clk.summary()['samples'] == 2


def test_outgrown_workspaces_stay_alive_for_captured_graphs():
    from quip_b200 import quant as Q
    dev = torch.device('cpu')
    a = Q._workspace(dev, 1000, stream_ptr=12345)
    assert a.numel() == 1 << 20 and Q._workspace(dev, 4096, stream_ptr=12345) is a          # reuse while it fits
    ptr = a.data_ptr()
    b = Q._workspace(dev, (1 << 20) + 1, stream_ptr=12345)
    assert b.numel() == 2 << 20 and b is not a
    assert any(t is a for t in Q._retired) and a.data_ptr() == ptr                           # the old block is not freed
    assert Q._workspace(dev, 10, stream_ptr=777) is not b                                    # per-stream workspaces


# ---- property tests (hypothesis): pack <-> unpack for 2/3/4 bits, the reference layouts included (SURVEY section 4) ----
from hypothesis import given, settings, strategies as st  # noqa: E402


@settings(max_examples=25, deadline=None)
@given(bits=st.sampled_from([2, 3, 4]), nb=st.integers(1, 4), kb=st.integers(1, 3), seed=st.integers(0, 2 ** 31 - 1),
       fill=st.sampled_from(['random', 'zeros', 'max', 'ramp']))
def test_pack_unpack_round_trip_property(bits, nb, kb, seed, fill):
    N, K = 16 * nb, 128 * kb
    top = (1 << bits) - 1
    if fill == 'random':
        codes = np.random.default_rng(seed).integers(0, top + 1, size=(N, K), dtype=np.uint8)
    elif fill == 'zeros':
        codes = np.zeros((N, K), np.uint8)
    elif fill == 'max':
        codes = np.full((N, K), top, np.uint8)
    else:
        codes = ((np.arange(N)[:, None] * 7 + np.arange(K)[None, :]) % (top + 1)).astype(np.uint8)
    q = Q.pack_codes(torch.from_numpy(codes), bits)
    assert q.dtype == torch.int32 and q.numel() == Q.packed_words(N, K, bits) == N * K * bits // 32
    np.testing.assert_array_equal(q.numpy(), opk.native_pack(codes, bits))                 # the oracle's layout, word for word
    np.testing.assert_array_equal(Q.unpack_codes(q, N, K, bits).numpy(), codes)
    np.testing.assert_array_equal(opk.native_unpack(q.numpy(), N, K, bits), codes)
    # every code lands in exactly `bits` bits: flipping one code changes one word (two when a 3-bit code straddles)
    c2 = codes.copy()
    c2[seed % N, seed % K] ^= 1
    changed = int((Q.pack_codes(torch.from_numpy(c2), bits) != q).sum())
    assert 1 <= changed <= 2


@settings(max_examples=15, deadline=None)
@given(bits=st.sampled_from([2, 3, 4]), nb=st.integers(1, 3), seed=st.integers(0, 2 ** 31 - 1))
def test_reference_layout_round_trip_property(bits, nb, seed):
    """The reference's own layouts, (K*bits/32, N) int32 (quant.py:192-220, zeroShot/models/quant.py:193-199), as restated
    in oracle/packing.py (pinned to the reference's words in test_oracle_golden.py): pack <-> unpack is the identity and the
    word count is what Quant3Linear / Quant4Linear register.  (quip_convert_ref, the GPU converter, is checked against the
    same functions in tests/test_gpu_kernels.py.)"""
    N, K = 16 * nb, 128
    codes = np.random.default_rng(seed).integers(0, 1 << bits, size=(N, K), dtype=np.uint8)
    pack, unpack = {2: (opk.ref_pack2, opk.ref_unpack2), 3: (opk.ref_pack3, opk.ref_unpack3),
                    4: (opk.ref_pack4, opk.ref_unpack4)}[bits]
    words = pack(codes)
    assert words.shape == (K * bits // 32, N) and words.dtype == np.int32
    np.testing.assert_array_equal(unpack(words, K), codes)
