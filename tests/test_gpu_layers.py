"""Whole-layer parity: QuantLinear.forward (C ABI, CUDA) vs the reference's dense fp16 forward
(golden y_ref from F.linear on the reference's W_ref) and vs the oracle's stage-by-stage model."""
import numpy as np
import pytest
import torch

from conftest import LAYER_NAMES, load_layer, parts_to_torch
from oracle import forward as ofw

pytestmark = pytest.mark.gpu

# north_star tolerance: 1e-3 relative (norm-wise, SURVEY section 7 "parity budget") on the fp16 layer output
TOL_REF = 1e-3
# the CUDA pipeline against its own numpy model (same fp16 rounding points): only accumulation order differs
TOL_MODEL = 2.5e-4


def _report(name, rec):
    """Append the measured errors of one case as a JSON line to the suite's parity report (parity_report.jsonl)."""
    import json
    import os
    from conftest import ROOT
    os.makedirs(os.path.join(ROOT, 'gpurun_out'), exist_ok=True)
    with open(os.path.join(ROOT, 'gpurun_out', 'parity_report.jsonl'), 'a') as f:
        f.write(json.dumps(dict(case=name, **rec)) + '\n')


def _module(parts):
    from quip_b200 import quant as Q
    tp = parts_to_torch(parts)
    N, K = tp.codes.shape
    ql = Q.QuantLinear(infeatures=K, outfeatures=N, **Q.spec_from_parts(tp))
    ql.pack_parts(tp)
    return ql.cuda()


@pytest.mark.parametrize('name', LAYER_NAMES)
def test_layer_matches_reference_output(name):
    parts, z = load_layer(name)
    ql = _module(parts)
    # bit-exact integer codes under the layout permutation
    plan = ofw.kernel_plan(parts)
    np.testing.assert_array_equal(ql.codes().cpu().numpy(), plan['codes'])
    x = torch.from_numpy(z['x']).cuda()
    y = ql(x).cpu().numpy()
    assert y.dtype == np.float16 and y.shape == z['y_ref'].shape
    e_ref = ofw.rel_err(y, z['y_ref'])
    e_model = ofw.rel_err(y, ofw.kernel_forward(z['x'], parts, fp16_points=True))
    _report(name, dict(M=int(x.shape[0]), rel_err_vs_reference=e_ref, rel_err_vs_model=e_model))
    assert e_ref < TOL_REF, (name, e_ref)
    assert e_model < TOL_MODEL * (1 if parts['V'] is None else 2), (name, e_model)


@pytest.mark.parametrize('name', ['l2b_incoh', 'l4b_plain', 'l3b_incoh'])
@pytest.mark.parametrize('M', [1, 7, 32, 33, 128, 2048])
def test_layer_token_counts(name, M):
    parts, z = load_layer(name)
    ql = _module(parts)
    K = parts['codes'].shape[1]
    rng = np.random.default_rng(M)
    x = (rng.standard_normal((M, K)) * (1 + 3 * rng.random(K))[None, :]).astype(np.float16)
    W = z['W_ref']
    want = ofw.dense_forward(x, W, parts['bias'])
    y = ql(torch.from_numpy(x).cuda()).cpu().numpy()
    err = ofw.rel_err(y, want)
    _report(name, dict(M=M, rel_err_vs_reference=err))
    assert err < TOL_REF, (name, M, err)
    # leading shape handling and dtype round trip
    y3 = ql(torch.from_numpy(x).cuda().reshape(1, M, K))
    assert y3.shape == (1, M, parts['codes'].shape[0])


def test_forward_is_linear_and_deterministic():
    """Size-independent properties at a Llama-2-7B layer shape (4096 -> 11008, 2-bit, blocked butterflies)."""
    from quip_b200.synth import synth_layer_parts
    from quip_b200 import quant as Q
    tp = synth_layer_parts(K=4096, N=11008, bits=2, incoh='blocked', rescale=True, bias=False, seed=3)
    ql = Q.QuantLinear(infeatures=4096, outfeatures=11008, **Q.spec_from_parts(tp))
    ql.pack_parts(tp)
    ql = ql.cuda()
    g = torch.Generator(device='cuda').manual_seed(0)
    for M in (4, 256):
        a = torch.randn(M, 4096, device='cuda', generator=g).half()
        b = torch.randn(M, 4096, device='cuda', generator=g).half()
        ya, yb, yab = ql(a).float(), ql(b).float(), ql((a.float() + b.float()).half()).float()
        lin = (yab - ya - yb).norm() / yab.norm()
        assert lin < 3e-3, (M, float(lin))
        assert torch.equal(ql(a), ql(a))
        assert float((ql(torch.zeros_like(a))).abs().max()) == 0.0
    # round trip of the integer codes at full size
    assert torch.equal(ql.codes().cpu(), tp.codes[plan_order(tp)[0]][:, plan_order(tp)[1]])


def plan_order(tp):
    from quip_b200.incoherence import plan_side
    return plan_side(tp.U, 'U').order, plan_side(tp.V, 'V').order


@pytest.mark.parametrize('K,N,incoh,bias', [(4096, 4096, 'blocked', False), (2048, 768, 'blocked', True),
                                             (768, 2048, 'blocked', False), (4096, 2048, 'kron', True)])
@pytest.mark.parametrize('M', [33, 37, 300, 2048])              # <= 32 tokens take the few-token kernels
def test_fused_side_kernel_equals_the_separate_kernels(K, N, incoh, bias, M):
    """One-kernel incoherence sides (gather + strided pass + contiguous pass [+ row sums], 16 token rows resident in
    shared memory) against the same steps as separate launches: same fp16 rounding points, so the outputs agree to
    the last bit except where the fp32 row sums were added in a different order."""
    from quip_b200 import _lib, quant as Q
    from quip_b200.synth import synth_layer_parts
    lib = _lib.load()
    tp = synth_layer_parts(K=K, N=N, bits=2, incoh=incoh, rescale=True, bias=bias, seed=K + N + M, qfn='a')
    ql = Q.QuantLinear(infeatures=K, outfeatures=N, **Q.spec_from_parts(tp)).cuda()
    ql.pack_parts(tp)
    x = (torch.randn(M, K, device='cuda') * (1 + 3 * torch.rand(K, device='cuda'))).half()
    try:
        lib.quip_config(b'side_fused', 0)
        y0 = ql(x).float()
        lib.quip_config(b'side_fused', 1)
        before = lib.quip_launch_count()
        y1 = ql(x).float()
        launches = lib.quip_launch_count() - before
    finally:
        lib.quip_config(b'side_fused', 1)
    torch.cuda.synchronize()
    # side, GEMM, side -- not gather + 2 passes + row sums on each side (a 768 side, 48 x 16 blocks, stays unfused)
    assert launches <= (3 if min(K, N) >= 2048 else 6), launches
    err = (y1 - y0).norm() / y0.norm()
    assert float(err) < 1e-4, float(err)               # a few last-bit flips from the re-ordered fp32 row sums
    assert float((y1 == y0).float().mean()) > 0.98


@pytest.mark.parametrize('K,N,bits,incoh', [(8192, 1024, 2, 'blocked'), (7168, 7168, 2, 'blocked'), (28672, 8192, 2, 'blocked'),
                                             (4096, 11008, 2, 'blocked'), (4096, 4096, 3, 'blocked'), (11008, 4096, 4, 'blocked'),
                                             (2048, 8192, 2, 'blocked'), (768, 3072, 4, None), (4096, 4096, 2, 'kron'),
                                             (3072, 768, 3, 'noperm')])
def test_other_model_shapes_against_torch_fp32(K, N, bits, incoh):
    """Layer shapes of the other configurations (Llama-2-70B: 8192 = 128 x 64, 28672 = 448 x 64; OPT-30b: 7168 =
    224 x 32) through every token-count route -- few-token kernels, split-K, wgmma -- against an fp32 torch
    restatement of the same pipeline built from the module's own buffers."""
    from gpu_util import torch_reference_forward
    from quip_b200 import quant as Q
    from quip_b200.synth import synth_layer_parts
    tp = synth_layer_parts(K=K, N=N, bits=bits, incoh=incoh, rescale=incoh is not None, bias=(N in (1024, 8192, 3072)),
                           seed=K + N, qfn='a')
    ql = Q.QuantLinear(infeatures=K, outfeatures=N, **Q.spec_from_parts(tp)).cuda()
    ql.pack_parts(tp)
    x = (torch.randn(40, K, device='cuda') * (1 + 3 * torch.rand(K, device='cuda'))).half()
    want = torch_reference_forward(ql, x)
    for M in (1, 5, 8, 20, 40):
        y = ql(x[:M]).float()
        err = float((y - want[:M]).norm() / want[:M].norm())
        assert err < 1.5e-3, (K, N, bits, incoh, M, err)


def test_sibling_group_overlap_is_bit_identical():
    """q/k/v-style siblings launched concurrently on side streams give exactly the serial results."""
    from quip_b200 import quant as Q
    from quip_b200.synth import synth_layer_parts
    mods = []
    for i, N in enumerate((256, 128, 384)):
        tp = synth_layer_parts(K=512, N=N, bits=2, incoh='blocked', rescale=True, bias=(i == 1), seed=20 + i)
        ql = Q.QuantLinear(infeatures=512, outfeatures=N, **Q.spec_from_parts(tp))
        ql.pack_parts(tp)
        mods.append(ql.cuda())
    g = torch.Generator(device='cuda').manual_seed(1)
    xs = [torch.randn(M, 512, device='cuda', generator=g).half() for M in (3, 300, 64)]
    serial = [[m(x).clone() for m in mods] for x in xs]
    grp = Q.SiblingGroup(mods)
    for rep in range(2):
        for x, want in zip(xs, serial):
            got = [m(x) for m in mods]                  # q, k, v order; k and v come from the side streams
            torch.cuda.synchronize()
            for a, b in zip(got, want):
                assert torch.equal(a, b)
            got_rev = [m(x.clone()) for m in reversed(mods)]   # a different first caller
            torch.cuda.synchronize()
            for a, b in zip(reversed(got_rev), want):
                assert torch.equal(a, b)
    grp.dissolve()
    assert torch.equal(mods[0](xs[0]), serial[0][0])


@pytest.mark.parametrize('K,N,bits,incoh,bias', [(4096, 4096, 2, 'blocked', False), (4096, 11008, 2, 'blocked', False),
                                                 (11008, 4096, 2, 'blocked', True), (8192, 1024, 2, 'blocked', False),
                                                 (28672, 8192, 2, 'blocked', False), (7168, 7168, 4, 'blocked', True),
                                                 (4096, 4096, 3, 'kron', False), (2048, 8192, 4, 'noperm', True),
                                                 (768, 3072, 2, 'blocked', True)])
def test_one_launch_sides_for_a_handful_of_tokens(K, N, bits, incoh, bias):
    """quip_config('side_fewtok'): for <= 8 tokens a whole incoherence side (gather, 1/s, both passes, scatter + bias) is one
    launch in which every CTA computes the first-pass rows its second-pass block consumes (rot_side_fewtok.cu) -- three
    launches per QuantLinear instead of five.  Same result as the two-pass route up to the rounding of the intermediate
    (kept in float32 here), and within the layer tolerance of the fp32 restatement."""
    from gpu_util import torch_reference_forward
    from quip_b200 import _lib, quant as Q
    from quip_b200.synth import synth_layer_parts
    lib = _lib.load()
    tp = synth_layer_parts(K=K, N=N, bits=bits, incoh=incoh, rescale=True, bias=bias, seed=K + N + bits, qfn='a')
    ql = Q.QuantLinear(infeatures=K, outfeatures=N, **Q.spec_from_parts(tp)).cuda()
    ql.pack_parts(tp)
    x = (torch.randn(8, K, device='cuda') * (1 + 3 * torch.rand(K, device='cuda'))).half()
    want = torch_reference_forward(ql, x)
    try:
        for M in (1, 2, 3, 5, 8):
            lib.quip_config(b'side_fewtok', 0)
            y0 = ql(x[:M]).float()
            lib.quip_config(b'side_fewtok', 1)
            before = lib.quip_launch_count()
            y1 = ql(x[:M]).float()
            launches = lib.quip_launch_count() - before
            assert float((y1 - want[:M]).norm() / want[:M].norm()) < 1e-3, (M, 'vs fp32 restatement')
            # the two-pass route rounds the intermediate to fp16: two results, each within 1e-3 of the restatement
            assert float((y1 - y0).norm() / y0.norm()) < 2e-3, (M, 'vs the two-pass route')
            assert torch.equal(y1, ql(x[:M]).float())
            assert launches <= 7, (M, launches)
            if max(K, N) <= 4096 or (M == 1 and max(K, N) <= 11008):   # both sides fit shared memory (tokens + factor rows)
                assert launches == 3, (M, launches)
    finally:
        lib.quip_config(b'side_fewtok', 0)                     # the library default (the one-launch route is an ablation)
