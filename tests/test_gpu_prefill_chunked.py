"""Chunked prefill on the GPU: the append and prefill-attention kernels (csrc/attn_prefill.cu) against oracle/kvfp8.py and
float64, and PromptDecoder.prefill(chunk=C) / generate(prefill_chunk_size=C) on synthetic packed models against the HF
path, teacher-forced e4m3 decode, and in peak memory."""
import math

import pytest
import torch

from oracle import kvfp8

pytestmark = pytest.mark.gpu

BLOCK = 64           # KV slots per block of the prefill kernel (PF_BN)


def _case(B, T, G, hd, max_len, positions, counts, seed=0, nkv=2, fp8=False):
    g = torch.Generator(device='cuda').manual_seed(seed)
    nh = G * nkv

    def r(*s):
        return torch.randn(*s, generator=g, device='cuda').half()
    q, kn, vn = r(B, T, nh, hd), r(B, T, nkv, hd), r(B, T, nkv, hd)
    kc, vc = r(B, nkv, max_len, hd), r(B, nkv, max_len, hd)
    pos = torch.tensor(positions, dtype=torch.long, device='cuda')
    cnt = torch.tensor(counts, dtype=torch.long, device='cuda')
    if not fp8:
        return q, kn, vn, kc, vc, pos, cnt, None, None
    kq, ks = kvfp8.quantize(kc)
    vq, vs = kvfp8.quantize(vc)
    return q, kn, vn, kq, vq, pos, cnt, ks, vs


def _sc(ks, vs):
    return {} if ks is None else dict(k_scale=ks, v_scale=vs)


def _appended(kn, vn, kc, vc, pos, cnt, ks=None, vs=None):
    """The caches (and scales) as they must be after the append: token i < cnt[b] of row b at slot pos[b] + i."""
    kc, vc = kc.clone(), vc.clone()
    ks, vs = (None, None) if ks is None else (ks.clone(), vs.clone())
    for b in range(kn.shape[0]):
        p, n = int(pos[b]), int(cnt[b])
        if ks is None:
            kc[b, :, p:p + n], vc[b, :, p:p + n] = kn[b, :n].transpose(0, 1), vn[b, :n].transpose(0, 1)
        else:
            for x, c, s in ((kn, kc, ks), (vn, vc, vs)):
                xq, xs = kvfp8.quantize(x[b, :n].transpose(0, 1))
                c[b, :, p:p + n], s[b, :, p:p + n] = xq, xs
    return kc, vc, ks, vs


def _reference(q, kc, vc, pos, cnt, scale, ks=None, vs=None):
    """float64 causal attention of the counted tokens over the appended caches (e4m3: dequantized); other rows 0."""
    B, T, nh, hd = q.shape
    G = nh // kc.shape[1]
    out = torch.zeros(B, T, nh, hd, dtype=torch.float64, device=q.device)
    for b in range(B):
        p, n = int(pos[b]), int(cnt[b])
        if n == 0:
            continue
        end = p + n
        if ks is None:
            K, V = kc[b, :, :end].double(), vc[b, :, :end].double()
        else:
            K = kvfp8.dequantize(kc[b, :, :end], ks[b, :, :end]).double()
            V = kvfp8.dequantize(vc[b, :, :end], vs[b, :, :end]).double()
        K, V = K.repeat_interleave(G, 0), V.repeat_interleave(G, 0)
        s = torch.einsum('thd,hjd->thj', q[b, :n].double(), K) * scale
        mask = torch.arange(end, device=q.device)[None] <= (p + torch.arange(n, device=q.device))[:, None]
        s = s.masked_fill(~mask[:, None], float('-inf'))
        out[b, :n] = torch.einsum('thj,hjd->thd', torch.softmax(s, -1), V)
    return out


def _run(q, kn, vn, kc, vc, pos, cnt, scale, ks=None, vs=None):
    """append, then attend (on copies of the caches): (out, caches after)."""
    from quip_b200 import fused
    kc, vc = kc.clone(), vc.clone()
    ks, vs = (None, None) if ks is None else (ks.clone(), vs.clone())
    fused.kv_append(kn, vn, kc, vc, pos, cnt, **_sc(ks, vs))
    return fused.prefill_attention(q, kc, vc, pos, cnt, scale, **_sc(ks, vs)), (kc, vc, ks, vs)


def _same_bytes(a, b):
    return torch.equal(a.view(torch.uint8), b.view(torch.uint8))


@pytest.mark.parametrize('fp8', [False, True])
@pytest.mark.parametrize('hd', [64, 128])
def test_append_writes_exactly_the_counted_slots(hd, fp8):
    from quip_b200 import fused
    B, T, nkv, max_len = 5, 37, 4, 200
    positions, counts = [0, 63, 100, 150, 7], [37, 20, 0, 50 - 13, 1]
    q, kn, vn, kc, vc, pos, cnt, ks, vs = _case(B, T, 1, hd, max_len, positions, counts, seed=hd, nkv=nkv, fp8=fp8)
    want = _appended(kn, vn, kc, vc, pos, cnt, ks, vs)
    fused.kv_append(kn, vn, kc, vc, pos, cnt, **_sc(ks, vs))
    assert _same_bytes(kc, want[0]) and _same_bytes(vc, want[1])       # sentinels elsewhere, row 2 untouched
    if fp8:
        assert torch.equal(ks, want[2]) and torch.equal(vs, want[3])


@pytest.mark.parametrize('fp8', [False, True])
@pytest.mark.parametrize('hd', [64, 128])
@pytest.mark.parametrize('G', [1, 4, 8])
@pytest.mark.parametrize('T', [1, 7, 64, 100, 257, 512])
def test_prefill_attention_matches_float64_with_ragged_positions_and_counts(T, G, hd, fp8):
    max_len = 1000 + T + 3
    scale = 1.0 / math.sqrt(hd)
    runs = [([p], [T]) for p in (0, 37, 1000)]
    runs.append(([0, 37, 1000], [T, 0, max(1, T // 2 + 1)]))
    runs.append(([1000, 0, 37], [max(1, T - 3), T, 0]))
    for positions, counts in runs:
        B = len(positions)
        q, kn, vn, kc, vc, pos, cnt, ks, vs = _case(B, T, G, hd, max_len, positions, counts, seed=T + G + hd + B,
                                                    fp8=fp8)
        out, after = _run(q, kn, vn, kc, vc, pos, cnt, scale, ks, vs)
        want = _appended(kn, vn, kc, vc, pos, cnt, ks, vs)
        assert _same_bytes(after[0], want[0]) and _same_bytes(after[1], want[1])
        ref = _reference(q, *want[:2], pos, cnt, scale, *want[2:])
        for b in range(B):
            n = counts[b]
            assert not out[b, n:].any(), (positions[b], b)           # rows past the count are zero
            for i in range(n):
                err = float((out[b, i].double() - ref[b, i]).norm() / ref[b, i].norm())
                assert err < 1e-3, (positions[b], counts[b], b, i, err)


@pytest.mark.parametrize('fp8', [False, True])
@pytest.mark.parametrize('hd', [64, 128])
def test_prefill_attention_never_reads_past_the_count_is_deterministic_and_row_independent(hd, fp8):
    from quip_b200 import fused
    B, T, G, max_len = 5, 150, 4, 6 * BLOCK
    positions, counts = [0, BLOCK - 3, 2 * BLOCK, 3, 100], [T, 77, 1, 0, 129]
    q, kn, vn, kc, vc, pos, cnt, ks, vs = _case(B, T, G, hd, max_len, positions, counts, seed=3, fp8=fp8)
    scale = 1.0 / math.sqrt(hd)
    clean, (kc1, vc1, ks1, vs1) = _run(q, kn, vn, kc, vc, pos, cnt, scale, ks, vs)
    assert torch.isfinite(clean).all()
    again = fused.prefill_attention(q, kc1, vc1, pos, cnt, scale, **_sc(ks1, vs1))
    assert torch.equal(again, clean)                                  # deterministic
    kp, vp = kc1.clone(), vc1.clone()
    ksp, vsp = (None, None) if ks1 is None else (ks1.clone(), vs1.clone())
    for b in range(B):
        end = positions[b] + counts[b]
        for t in (kp, vp) + ((ksp, vsp) if fp8 else ()):
            t[b, :, end:] = float('nan')                              # e4m3: NaN bytes
    assert torch.equal(fused.prefill_attention(q, kp, vp, pos, cnt, scale, **_sc(ksp, vsp)), clean)
    # other rows at other positions with other counts and contents: row 4 does not move
    q2, kn2, vn2, kc2, vc2, _, _, ks2, vs2 = _case(B, T, G, hd, max_len, positions, counts, seed=4, fp8=fp8)
    for t2, t in ((q2, q), (kn2, kn), (vn2, vn), (kc2, kc), (vc2, vc)) + (((ks2, ks), (vs2, vs)) if fp8 else ()):
        t2[4] = t[4]
    pos2 = torch.tensor([7, 200, 0, 99, positions[4]], dtype=torch.long, device='cuda')
    cnt2 = torch.tensor([T, 3, 150, 17, counts[4]], dtype=torch.long, device='cuda')
    other, _ = _run(q2, kn2, vn2, kc2, vc2, pos2, cnt2, scale, ks2, vs2)
    assert torch.equal(other[4], clean[4])


@pytest.mark.parametrize('fp8', [False, True])
@pytest.mark.parametrize('G', [1, 4])
@pytest.mark.parametrize('T', [1, 3, 8])
def test_prefill_attention_agrees_with_extend_attention_at_few_tokens(T, G, fp8):
    from quip_b200 import fused
    B, hd, max_len = 4, 128, 300
    positions = [0, 60, 64, 300 - T]
    q, kn, vn, kc, vc, pos, cnt, ks, vs = _case(B, T, G, hd, max_len, positions, [T] * B, seed=5, fp8=fp8)
    a, _ = _run(q, kn, vn, kc, vc, pos, cnt, 0.1, ks, vs)
    sc = _sc(None if ks is None else ks.clone(), None if vs is None else vs.clone())
    b = fused.extend_attention(q, kn, vn, kc.clone(), vc.clone(), pos, 0.1, **sc)
    for r in range(B):
        err = float((a[r].double() - b[r].double()).norm() / b[r].double().norm())
        assert err < 2e-3, (r, err)


# ---- PromptDecoder.prefill(chunk=C) on the synthetic packed models of test_gpu_generate

def _tiny(kind):
    from test_gpu_generate import _tiny as tiny
    return tiny(kind)


def _long_prompts():
    g = torch.Generator().manual_seed(9)
    return [torch.randint(0, 320, (n,), generator=g) for n in (70, 9, 101)]


@pytest.mark.parametrize('kind', [(4, 64), (2, 64), (2, 128), 'opt'])
def test_chunked_prefill_logits_match_the_hf_forward_as_closely_as_the_hf_path(kind):
    import bench
    from quip_b200.decode import PromptDecoder
    from test_gpu_generate import _norms
    model = _tiny(kind)
    prompts = _long_prompts()
    with torch.no_grad():
        hf_path = PromptDecoder(model, max_len=120, batch=3).prefill(prompts).float()
        chunked = {C: PromptDecoder(model, max_len=120, batch=3).prefill(prompts, chunk=C).float() for C in (16, 64)}
        worst = {C: 0.0 for C in chunked}
        worst_hf = control = 0.0
        for b, p in enumerate(prompts):
            runs = []
            for flip in (False, True):
                hooks = bench._ulp_flip_hooks(_norms(model), 3e-5, seed=b) if flip else []
                try:
                    runs.append(model(p.cuda()[None]).logits[0, -1].float())
                finally:
                    for hk in hooks:
                        hk.remove()
            want, ctrl = runs
            control = max(control, float((ctrl - want).norm() / want.norm()))
            worst_hf = max(worst_hf, float((hf_path[b] - want).norm() / want.norm()))
            for C, lg in chunked.items():
                worst[C] = max(worst[C], float((lg[b] - want).norm() / want.norm()))
    for C, w in worst.items():
        assert w < max(2e-3, 3.0 * control), (C, w, control, worst_hf)


@pytest.mark.parametrize('kv_dtype', [None, torch.float8_e4m3fn])
@pytest.mark.parametrize('kind', [(4, 64), (2, 128), 'opt'])
def test_generation_with_chunked_prefill_equals_generation_away_from_near_ties(kind, kv_dtype):
    """The chunked and the HF-path prefill leave caches that differ by rounding (e4m3: also by what the prompt attends
    over), so the steps' logits differ slightly.  Up to the first position whose top-2 gap is at most twice the largest
    logit difference of the two runs, the tokens must agree.  With an e4m3 cache the two prefills compute different
    things (quantized against fp16 attention), so the logits differ more and near-ties come sooner."""
    from quip_b200.decode import PromptDecoder
    model = _tiny(kind)
    prompts, n = _long_prompts(), 16
    runs = []
    for chunk in (None, 32):
        dec = PromptDecoder(model, max_len=120, batch=3, max_new=n, kv_dtype=kv_dtype).capture()
        with torch.no_grad():
            lg = [dec.prefill(prompts, chunk=chunk).float().clone()]
            lg += [dec.step().float().clone() for _ in range(n - 1)]
        runs.append((dec.generated.cpu(), lg))
    (g0, l0), (g1, l1) = runs
    checked = 0
    for b in range(3):
        for j in range(n):                                            # l0[j] selects generated[j]
            top2 = l0[j][b].topk(2).values
            if float(top2[0] - top2[1]) <= 2 * float((l1[j][b] - l0[j][b]).abs().max()):
                break
            assert int(g0[b, j]) == int(g1[b, j]), (b, j)
            checked += 1
    assert checked >= (n if kv_dtype is None else 3), checked


@pytest.mark.parametrize('kind', [(4, 64), (2, 128), 'opt'])
def test_e4m3_chunked_prefill_matches_teacher_forced_e4m3_decode(kind):
    """Chunked e4m3 prefill attends over the quantized cache, as T = 1 decode steps fed the prompt token by token do.
    Their linears run at other token counts on other kernel routes, so keys and values differ by fp16 rounding and some
    land across an e4m3 rounding boundary; the first layer's keys and values, which no attention has touched, measure
    that rate.  The HF-path prefill has the same linear routes but attends in fp16: past the first layer its cache and
    its logits are further from the teacher-forced decode than the chunked prefill's."""
    from quip_b200.decode import PromptDecoder
    model = _tiny(kind)
    prompts = _long_prompts()
    e4 = torch.float8_e4m3fn
    with torch.no_grad():
        chunked = PromptDecoder(model, max_len=120, batch=3, kv_dtype=e4)
        hf = PromptDecoder(model, max_len=120, batch=3, kv_dtype=e4)
        logits = {'chunked': chunked.prefill(prompts, chunk=32).float(), 'hf': hf.prefill(prompts).float()}
        flips = {(k, li): 0 for k in logits for li in range(2)}
        total = 0
        err = {k: 0.0 for k in logits}
        for b, p in enumerate(prompts):
            one = PromptDecoder(model, max_len=120, batch=1, kv_dtype=e4).capture()
            for t in p.cuda():
                want = one.step(t.reshape(1))[0].float()
            n = p.numel()
            total += 2 * one.k_cache[0, 0, :, :n].numel()
            for k, dec in (('chunked', chunked), ('hf', hf)):
                for li in range(2):
                    for x, y in ((dec.k_cache, one.k_cache), (dec.v_cache, one.v_cache)):
                        flips[k, li] += int((x[li, b, :, :n].view(torch.uint8) != y[li, 0, :, :n].view(torch.uint8)).sum())
                err[k] = max(err[k], float((logits[k][b] - want).norm() / want.norm()))
    rate = {key: v / total for key, v in flips.items()}
    assert abs(rate['chunked', 0] - rate['hf', 0]) < 0.01 and rate['chunked', 0] < 0.05, rate   # layer 0: linears only
    assert rate['chunked', 1] < 0.5 * rate['hf', 1], rate
    assert err['chunked'] < 0.5 * err['hf'] and err['chunked'] < 2e-2, err


def _peak_added(fn):
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    fn()
    torch.cuda.synchronize()
    return torch.cuda.max_memory_allocated() - base


def test_chunked_prefill_memory_follows_the_chunk_not_the_prompt():
    """2 layers at Llama-2-7B widths, B = 8: the HF path holds every token's activations and an fp16 copy of the cache at
    once; chunks of 256 tokens hold 256 per row."""
    from quip_b200 import synth
    from quip_b200.decode import PromptDecoder
    cfg = synth.model_config('llama7b', num_hidden_layers=2)
    model = synth.build_synthetic_model(cfg, torch.device('cuda:0'), bits=2, seed=1, seqlen=256)
    B, C = 8, 256
    g = torch.Generator().manual_seed(0)
    peaks = {}
    for P in (1024, 2048):
        prompts = [torch.randint(0, cfg.vocab_size, (P,), generator=g) for _ in range(B)]
        dec = PromptDecoder(model, max_len=P, batch=B)
        with torch.no_grad():
            dec.prefill(prompts, chunk=C)                             # lazy workspaces outside the measurement
            peaks[P, 'chunked'] = _peak_added(lambda: dec.prefill(prompts, chunk=C))
            peaks[P, 'hf'] = _peak_added(lambda: dec.prefill(prompts))
        del dec
        torch.cuda.empty_cache()
    for P in (1024, 2048):
        assert peaks[P, 'chunked'] < 0.5 * peaks[P, 'hf'], peaks
    assert abs(peaks[2048, 'chunked'] - peaks[1024, 'chunked']) <= 0.1 * peaks[1024, 'chunked'], peaks
