"""The e4m3 KV cache on the GPU: quip_kv_quantize_fp8 and quip_decode_attention on e4m3 caches (csrc/attn_decode.cu) against
oracle/kvfp8.py, and PromptDecoder / generate with kv_dtype=torch.float8_e4m3fn on synthetic packed models."""
import math

import pytest
import torch

from oracle import kvfp8

from test_gpu_generate import CHUNK, MODELS, _chunk, _edges, _positions, _prompts, _tiny

pytestmark = pytest.mark.gpu
FP8 = torch.float8_e4m3fn


def _bytes(t):
    return t.view(torch.uint8)


def _edge_rows(hd):
    """Vectors at the edges of the format: amax exactly 448, all zero, e4m3 subnormals after scaling, one huge element."""
    rows = torch.zeros(4, hd)
    rows[0, :3] = torch.tensor([448.0, -448.0, 1.0])
    rows[2] = torch.linspace(-1, 1, hd) * 2.0 ** -12
    rows[2, 0] = 1.0                                                  # the rest land below 2^-6 * s: subnormals
    rows[3, 5] = -60000.0
    rows[3, 6:] = torch.randn(hd - 6, generator=torch.Generator().manual_seed(3))
    return rows.half()


@pytest.mark.parametrize('hd', [64, 128])
def test_kv_quantize_is_bit_exact_and_leaves_later_slots(hd):
    from quip_b200 import fused
    B, nkv, P, max_len = 3, 2, 37, 50
    g = torch.Generator(device='cuda').manual_seed(hd)
    src = (torch.randn(B, nkv, P, hd, generator=g, device='cuda') *
           10.0 ** torch.randint(-3, 3, (B, nkv, P, 1), generator=g, device='cuda')).half()
    src[0, 0, :4] = _edge_rows(hd).cuda()
    cache = torch.randint(0, 256, (B, nkv, max_len, hd), generator=g, device='cuda', dtype=torch.uint8).view(FP8)
    scales = torch.randn(B, nkv, max_len, generator=g, device='cuda')
    c0, s0 = cache.clone(), scales.clone()
    fused.kv_quantize(src, cache, scales)
    q, s = kvfp8.quantize(src.cpu())
    assert torch.equal(_bytes(cache[:, :, :P]).cpu(), _bytes(q)) and torch.equal(scales[:, :, :P].cpu(), s)
    amax = src.float().abs().amax(-1)
    s_cuda = torch.where(amax == 0, 1.0, amax / torch.full_like(amax, 448.0))   # a scalar divisor is not IEEE on CUDA
    q_cuda = (src.float() / s_cuda[..., None]).to(FP8)                # torch CUDA's own conversion
    assert torch.equal(_bytes(cache[:, :, :P]), _bytes(q_cuda)) and torch.equal(scales[:, :, :P], s_cuda)
    assert torch.equal(_bytes(cache[:, :, P:]), _bytes(c0[:, :, P:])) and torch.equal(scales[:, :, P:], s0[:, :, P:])


def _case(B, G, hd, max_len, positions, seed=0, nkv=2):
    g = torch.Generator(device='cuda').manual_seed(seed)
    nh = G * nkv

    def r(*s):
        return torch.randn(*s, generator=g, device='cuda').half()
    q, kn, vn = r(B, nh, hd), r(B, nkv, hd), r(B, nkv, hd)
    kc, ks = kvfp8.quantize(r(B, nkv, max_len, hd) * 3)
    vc, vs = kvfp8.quantize(r(B, nkv, max_len, hd))
    pos = torch.tensor(positions, dtype=torch.long, device='cuda')
    return q, kn, vn, kc, vc, ks, vs, pos


def _attn(q, kn, vn, kc, vc, ks, vs, pos, scale):
    from quip_b200 import fused
    return fused.decode_attention(q, kn, vn, kc, vc, pos, scale, k_scale=ks, v_scale=vs)


@pytest.mark.parametrize('hd', [64, 128])
@pytest.mark.parametrize('G', [1, 4, 8])
@pytest.mark.parametrize('B', [1, 3, 32])
def test_fp8_kernel_matches_float64_attention_over_the_dequantized_cache(hd, G, B):
    max_len = 3 * CHUNK + 40
    nkv = 8 if B == 32 else 2
    edge = _edges(_chunk(B, nkv, max_len), max_len)
    scale = 1.0 / math.sqrt(hd)
    if B == 1:
        runs = [[p] for p in edge]
    elif B == 3:
        runs = [edge[i:i + 3] for i in range(0, len(edge), 3)]
        runs[-1] += _positions(3 - len(runs[-1]), max_len, B, [])
    else:
        runs = [_positions(B, max_len, B, edge)]
    for positions in runs:
        q, kn, vn, kc, vc, ks, vs, pos = _case(B, G, hd, max_len, positions, seed=hd + G + B, nkv=nkv)
        k0, v0, ks0, vs0 = kc.clone(), vc.clone(), ks.clone(), vs.clone()
        out = _attn(q, kn, vn, kc, vc, ks, vs, pos, scale)
        ref = kvfp8.attention(q, kn, vn, k0, v0, ks0, vs0, pos, scale)
        for b in range(B):
            err = float((out[b].double() - ref[b]).norm() / ref[b].norm())
            assert err < 1e-3, (positions[b], b, err)
        # the append is the oracle quantization of k_new / v_new, bytes and scale; nothing else moves
        rows = torch.arange(B, device='cuda')
        for new, c0, s0 in ((kn, k0, ks0), (vn, v0, vs0)):
            nq, ns = kvfp8.quantize(new)
            c0[rows, :, pos], s0[rows, :, pos] = nq, ns
        assert torch.equal(_bytes(kc), _bytes(k0)) and torch.equal(_bytes(vc), _bytes(v0))
        assert torch.equal(ks, ks0) and torch.equal(vs, vs0)


@pytest.mark.parametrize('hd', [64, 128])
def test_fp8_kernel_never_reads_past_the_position_and_rows_are_independent(hd):
    B, G, max_len = 6, 4, 4 * CHUNK
    c = _chunk(B, 2, max_len)
    positions = [0, c - 1, c, c + 1, 3 * CHUNK + 7, max_len - 1]
    q, kn, vn, kc, vc, ks, vs, pos = _case(B, G, hd, max_len, positions, seed=11)
    scale = 1.0 / math.sqrt(hd)

    def run(kc, vc, ks, vs):
        return _attn(q, kn, vn, kc.clone(), vc.clone(), ks.clone(), vs.clone(), pos, scale)
    clean = run(kc, vc, ks, vs)
    assert torch.equal(clean, run(kc, vc, ks, vs))                    # deterministic
    kp, vp, ksp, vsp = kc.clone(), vc.clone(), ks.clone(), vs.clone()
    for b, p in enumerate(positions):
        for t in (kp, vp):
            _bytes(t)[b, :, p:] = 0x7F                                # e4m3 NaN; slot p too: the kernel appends there
        ksp[b, :, p:] = float('nan')
        vsp[b, :, p:] = float('nan')
    poisoned = run(kp, vp, ksp, vsp)
    assert torch.isfinite(poisoned).all() and torch.equal(poisoned, clean)
    q2, kn2, vn2, kc2, vc2, ks2, vs2, _ = _case(B, G, hd, max_len, positions, seed=12)
    for t2, t in ((q2, q), (kn2, kn), (vn2, vn), (kc2, kc), (vc2, vc), (ks2, ks), (vs2, vs)):
        t2[2] = t[2]
    pos2 = torch.tensor([max_len - 1, 5, positions[2], 2 * CHUNK, 0, 77], dtype=torch.long, device='cuda')
    other = _attn(q2, kn2, vn2, kc2, vc2, ks2, vs2, pos2, scale)
    assert torch.equal(other[2], clean[2])


def _fed(n_steps, seed=9):
    return torch.randint(0, 320, (3, n_steps), generator=torch.Generator().manual_seed(seed)).cuda()


@pytest.mark.parametrize('kind', MODELS)
def test_fp8_decoder_appends_logits_and_graph_replay(kind):
    """Teacher-forced against the fp16-cache decoder: every layer-0 slot the fp8 decoder appends is the oracle
    quantization of the fp16 decoder's slot, and the logits stay within one e4m3 step (2^-4, relative norm).  A
    captured fp8 decoder replays the eager fp8 step bit for bit."""
    from quip_b200.decode import PromptDecoder
    model = _tiny(kind)
    prompts, ids = _prompts(), _fed(8)
    with torch.no_grad():
        ref = PromptDecoder(model, max_len=32, batch=3)
        eager = PromptDecoder(model, max_len=32, batch=3, kv_dtype=FP8)
        graph = PromptDecoder(model, max_len=32, batch=3, kv_dtype=FP8).capture()
        lr, le, lg = ref.prefill(prompts), eager.prefill(prompts), graph.prefill(prompts)
        assert torch.equal(lr, le) and torch.equal(le, lg)            # the first token comes from the fp16 forward
        worst = 0.0
        for i in range(ids.shape[1]):
            r, e, g = ref.step(ids[:, i]).float(), eager.step(ids[:, i]).clone(), graph.step(ids[:, i])
            assert torch.equal(e, g), i
            worst = max(worst, float((e.float() - r).norm() / r.norm()))
    for b, p in enumerate(prompts):
        slots = torch.arange(p.numel(), p.numel() + ids.shape[1])
        for cache, scales, src in ((eager.k_cache, eager.k_scale, ref.k_cache), (eager.v_cache, eager.v_scale, ref.v_cache)):
            q, s = kvfp8.quantize(src[0, b, :, slots])
            assert torch.equal(_bytes(cache[0, b, :, slots]), _bytes(q)) and torch.equal(scales[0, b, :, slots], s)
        # the prefill's slots too (quip_kv_quantize_fp8 of the same fp16 keys)
        q, s = kvfp8.quantize(ref.k_cache[:, b, :, :p.numel()])
        assert torch.equal(_bytes(eager.k_cache[:, b, :, :p.numel()]), _bytes(q))
    print(f'{kind}: fp8 vs fp16 cache logits, worst relative norm error {worst:.2e}')
    assert worst <= 2.0 ** -4, worst


def test_fp8_generate_returns_the_greedy_tokens_of_the_decoder():
    from quip_b200.decode import PromptDecoder, generate
    model = _tiny((2, 64))
    prompts = _prompts()
    out = generate(model, prompts, 20, kv_dtype=FP8)
    with torch.no_grad():
        dec = PromptDecoder(model, max_len=37, batch=3, max_new=20, kv_dtype=FP8).capture()
        dec.prefill(prompts)
        for _ in range(19):
            dec.step()
    for b in range(3):
        assert torch.equal(out[b], dec.generated[b].cpu())


def test_fp8_capture_from_a_full_cache_then_reuse_after_reset():
    from quip_b200.decode import PromptDecoder
    model = _tiny((2, 128))
    prompts = _prompts()
    with torch.no_grad():
        dec = PromptDecoder(model, max_len=19, batch=3, max_new=3, kv_dtype=FP8)
        dec.prefill(prompts)
        dec.step()
        dec.step()                                                    # row 2 at max_len, generated full
        pos, gen = dec.positions.clone(), dec.generated.clone()
        dec.capture()
        assert torch.equal(dec.positions, pos) and torch.equal(dec.generated, gen)
        dec.reset()
        assert not dec.k_scale.any() and not dec.v_scale.any()
        fresh = PromptDecoder(model, max_len=19, batch=3, max_new=3, kv_dtype=FP8).capture()
        for d in (dec, fresh):
            d.prefill([p[:6] for p in prompts])
            d.step()
            d.step()
        assert torch.equal(dec.generated, fresh.generated) and torch.equal(dec.logits, fresh.logits)
