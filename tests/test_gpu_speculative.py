"""Speculative generation on the GPU: the extend-attention kernel (csrc/attn_decode.cu) against float64, the draft and
accept kernels (csrc/spec.cu) against oracle/speculative.py, quip_sample_at against quip_sample, and SpecDecoder /
generate(prompt_lookup_num_tokens=...) on synthetic packed models against the eager HF forward and plain generation."""
import math

import numpy as np
import pytest
import torch

from oracle import kvfp8
from oracle import speculative as spec_oracle

pytestmark = pytest.mark.gpu

CHUNK = 64           # KV slots per CTA of the extend kernel (AX_CHUNK)


def _case(B, T, G, hd, max_len, positions, seed=0, nkv=2, fp8=False):
    g = torch.Generator(device='cuda').manual_seed(seed)
    nh = G * nkv

    def r(*s):
        return torch.randn(*s, generator=g, device='cuda').half()
    q, kn, vn = r(B, T, nh, hd), r(B, T, nkv, hd), r(B, T, nkv, hd)
    kc, vc = r(B, nkv, max_len, hd), r(B, nkv, max_len, hd)
    pos = torch.tensor(positions, dtype=torch.long, device='cuda')
    if not fp8:
        return q, kn, vn, kc, vc, pos, None, None
    kq, ks = kvfp8.quantize(kc)
    vq, vs = kvfp8.quantize(vc)
    return q, kn, vn, kq, vq, pos, ks, vs


def _attn(q, kn, vn, kc, vc, pos, scale, ks=None, vs=None):
    from quip_b200 import fused
    return fused.extend_attention(q, kn, vn, kc, vc, pos, scale, k_scale=ks, v_scale=vs)


def _appended(kn, vn, kc, vc, pos, ks=None, vs=None):
    """The caches (and scales) as they must be after the call: token i of row b at slot pos[b] + i, nothing else."""
    kc, vc = kc.clone(), vc.clone()
    ks, vs = (None, None) if ks is None else (ks.clone(), vs.clone())
    for b in range(kn.shape[0]):
        p, T = int(pos[b]), kn.shape[1]
        if ks is None:
            kc[b, :, p:p + T], vc[b, :, p:p + T] = kn[b].transpose(0, 1), vn[b].transpose(0, 1)
        else:
            for x, c, s in ((kn, kc, ks), (vn, vc, vs)):
                xq, xs = kvfp8.quantize(x[b].transpose(0, 1))
                c[b, :, p:p + T], s[b, :, p:p + T] = xq, xs
    return kc, vc, ks, vs


def _reference(q, kc, vc, pos, scale, ks=None, vs=None):
    """float64 causal attention over the caches as appended (e4m3: dequantized)."""
    B, T, nh, hd = q.shape
    G = nh // kc.shape[1]
    out = torch.empty(B, T, nh, hd, dtype=torch.float64, device=q.device)
    for b in range(B):
        n = int(pos[b]) + T
        if ks is None:
            K, V = kc[b, :, :n].double(), vc[b, :, :n].double()
        else:
            K = kvfp8.dequantize(kc[b, :, :n], ks[b, :, :n]).double()
            V = kvfp8.dequantize(vc[b, :, :n], vs[b, :, :n]).double()
        K, V = K.repeat_interleave(G, 0), V.repeat_interleave(G, 0)
        s = torch.einsum('thd,hjd->thj', q[b].double(), K) * scale
        mask = torch.arange(n, device=q.device)[None] <= (int(pos[b]) + torch.arange(T, device=q.device))[:, None]
        s = s.masked_fill(~mask[:, None], float('-inf'))
        out[b] = torch.einsum('thj,hjd->thd', torch.softmax(s, -1), V)
    return out


def _edges(T, max_len):
    """New slots straddling the 64- and 128-slot chunk edges, starting at 0, and ending exactly at max_len."""
    c = [0, CHUNK - T // 2 - 1, CHUNK - 1, CHUNK, 2 * CHUNK - (T + 1) // 2, 2 * CHUNK - 1, 2 * CHUNK - T, max_len - T]
    return [min(max(p, 0), max_len - T) for p in c]


def _same_bytes(a, b):
    return torch.equal(a.view(torch.uint8), b.view(torch.uint8))


@pytest.mark.parametrize('fp8', [False, True])
@pytest.mark.parametrize('hd', [64, 128])
@pytest.mark.parametrize('G', [1, 4, 8])
@pytest.mark.parametrize('T', [1, 2, 5, 8])
@pytest.mark.parametrize('B', [1, 3, 32])
def test_extend_matches_float64_and_appends_exactly(B, T, G, hd, fp8):
    max_len = 3 * CHUNK + 40
    nkv = 8 if B == 32 else 2
    edge = _edges(T, max_len)
    scale = 1.0 / math.sqrt(hd)
    if B == 1:
        runs = [[p] for p in edge]
    elif B == 3:
        runs = [edge[i:i + 3] + edge[:max(0, 3 - len(edge[i:i + 3]))] for i in range(0, len(edge), 3)]
    else:
        g = torch.Generator().manual_seed(T + G)
        runs = [edge + [int(torch.randint(0, max_len - T + 1, (1,), generator=g)) for _ in range(B - len(edge))]]
    for positions in runs:
        q, kn, vn, kc, vc, pos, ks, vs = _case(B, T, G, hd, max_len, positions, seed=hd + G + B + T, nkv=nkv, fp8=fp8)
        want_k, want_v, want_ks, want_vs = _appended(kn, vn, kc, vc, pos, ks, vs)
        out = _attn(q, kn, vn, kc, vc, pos, scale, ks, vs)
        ref = _reference(q, want_k, want_v, pos, scale, want_ks, want_vs)
        for b in range(B):
            for i in range(T):
                err = float((out[b, i].double() - ref[b, i]).norm() / ref[b, i].norm())
                assert err < 1e-3, (positions[b], b, i, err)
        assert _same_bytes(kc, want_k) and _same_bytes(vc, want_v)
        if fp8:
            assert torch.equal(ks, want_ks) and torch.equal(vs, want_vs)


@pytest.mark.parametrize('fp8', [False, True])
@pytest.mark.parametrize('hd', [64, 128])
def test_extend_never_reads_past_its_slots_is_causal_deterministic_and_row_independent(hd, fp8):
    B, T, G, max_len = 6, 5, 4, 4 * CHUNK
    positions = [0, CHUNK - 2, CHUNK, 2 * CHUNK - 3, 3 * CHUNK + 7, max_len - T]
    q, kn, vn, kc, vc, pos, ks, vs = _case(B, T, G, hd, max_len, positions, seed=11, fp8=fp8)
    scale = 1.0 / math.sqrt(hd)

    def run(q=q, kn=kn, vn=vn, kc=kc, vc=vc, pos=pos, ks=ks, vs=vs):
        return _attn(q, kn, vn, kc.clone(), vc.clone(), pos, scale,
                     None if ks is None else ks.clone(), None if vs is None else vs.clone())
    clean = run()
    assert torch.isfinite(clean).all()
    assert torch.equal(clean, run())                                  # deterministic
    kp, vp = kc.clone(), vc.clone()
    ksp, vsp = (None, None) if ks is None else (ks.clone(), vs.clone())
    for b, p in enumerate(positions):
        if fp8:
            kp[b, :, p:] = float('nan')                               # e4m3 NaN bytes
            vp[b, :, p:] = float('nan')
            ksp[b, :, p:] = float('nan')
            vsp[b, :, p:] = float('nan')
        else:
            kp[b, :, p:] = float('nan')
            vp[b, :, p:] = float('nan')
    assert torch.equal(run(kc=kp, vc=vp, ks=ksp, vs=vsp), clean)
    # causality: new keys / values of tokens after i do not move token i
    for i in range(T - 1):
        kn2, vn2 = kn.clone(), vn.clone()
        kn2[:, i + 1:] = torch.randn_like(kn2[:, i + 1:].float()).half()
        vn2[:, i + 1:] = torch.randn_like(vn2[:, i + 1:].float()).half()
        assert torch.equal(run(kn=kn2, vn=vn2)[:, :i + 1], clean[:, :i + 1]), i
    # other rows at other positions with other contents: row 2 does not move
    q2, kn2, vn2, kc2, vc2, _, ks2, vs2 = _case(B, T, G, hd, max_len, positions, seed=12, fp8=fp8)
    for t2, t in ((q2, q), (kn2, kn), (vn2, vn), (kc2, kc), (vc2, vc)) + (((ks2, ks), (vs2, vs)) if fp8 else ()):
        t2[2] = t[2]
    pos2 = torch.tensor([max_len - T, 5, positions[2], 2 * CHUNK, 0, 77], dtype=torch.long, device='cuda')
    other = run(q=q2, kn=kn2, vn=vn2, kc=kc2, vc=vc2, pos=pos2, ks=ks2, vs=vs2)
    assert torch.equal(other[2], clean[2])


@pytest.mark.parametrize('fp8', [False, True])
def test_extend_rows_past_the_cache_get_nan_and_write_nothing(fp8):
    B, T, G, hd, max_len = 4, 4, 2, 64, 2 * CHUNK
    positions = [max_len - T + 1, -1, max_len - T, 3]
    q, kn, vn, kc, vc, pos, ks, vs = _case(B, T, G, hd, max_len, positions, seed=3, fp8=fp8)
    k0, v0 = kc.clone(), vc.clone()
    out = _attn(q, kn, vn, kc, vc, pos, 0.125, ks, vs)
    assert torch.isnan(out[:2]).all() and torch.isfinite(out[2:]).all()
    assert _same_bytes(kc[:2], k0[:2]) and _same_bytes(vc[:2], v0[:2])


@pytest.mark.parametrize('fp8', [False, True])
def test_extend_at_one_token_agrees_with_decode_attention(fp8):
    from quip_b200 import fused
    B, G, hd, max_len = 5, 4, 128, 300
    positions = [0, 63, 64, 200, 299]
    q, kn, vn, kc, vc, pos, ks, vs = _case(B, 1, G, hd, max_len, positions, seed=4, fp8=fp8)
    sc = {} if not fp8 else dict(k_scale=ks.clone(), v_scale=vs.clone())
    a = fused.decode_attention(q[:, 0].contiguous(), kn[:, 0].contiguous(), vn[:, 0].contiguous(), kc.clone(), vc.clone(),
                               pos, 0.1, **sc)
    b = _attn(q, kn, vn, kc.clone(), vc.clone(), pos, 0.1, ks, vs)[:, 0]
    assert float((a.double() - b.double()).norm() / a.double().norm()) < 1e-3


def _histories(B, max_len, vocab, seed):
    g = np.random.default_rng(seed)
    hist = g.integers(0, vocab, (B, max_len)).astype(np.int64)
    pos = g.integers(0, max_len, B).astype(np.int64)
    for b in range(0, B, 4):                                          # periodic rows: overlapping copies
        per = 1 + b % 3
        hist[b, :] = np.tile(g.integers(0, vocab, per), max_len // per + 1)[:max_len]
    pos[1] = 0                                                        # nothing before the current token
    return hist, pos


@pytest.mark.parametrize('k,n_max', [(1, 1), (4, 3), (7, 2), (7, 5)])
def test_ngram_draft_kernel_equals_the_oracle(k, n_max):
    from quip_b200 import fused
    for vocab in (3, 12, 1000):
        hist, pos = _histories(67, 300, vocab, seed=vocab + k)
        want = spec_oracle.ngram_draft(hist, pos, k, 1, n_max)
        got = torch.zeros(67, k + 1, dtype=torch.long, device='cuda')
        fused.ngram_draft(torch.from_numpy(hist).cuda(), torch.from_numpy(pos).cuda(), got, 1, n_max)
        assert np.array_equal(got.cpu().numpy(), want), vocab


def test_spec_accept_kernel_equals_the_oracle():
    from quip_b200 import fused
    g = np.random.default_rng(5)
    B, T, max_new, max_len = 40, 6, 9, 64
    tokens = g.integers(0, 3, (B, T)).astype(np.int64)
    targets = g.integers(0, 3, (B, T)).astype(np.int64)
    targets[::3, :-1] = tokens[::3, 1:]                               # every draft right
    n_gen = g.integers(0, max_new + 2, B).astype(np.int64)            # finished rows and rows near max_new
    positions = g.integers(0, max_len - T, B).astype(np.int64)
    positions[-1] = max_len - 2                                       # history writes clipped at max_len
    gen = g.integers(0, 3, (B, max_new)).astype(np.int64)
    hist = g.integers(0, 3, (B, max_len)).astype(np.int64)
    accepted = g.integers(0, 5, B).astype(np.int64)
    cuda = [torch.from_numpy(x.copy()).cuda() for x in (tokens, targets, gen, hist, positions, n_gen, accepted)]
    spec_oracle.spec_accept(tokens, targets, gen, hist, positions, n_gen, accepted, max_new)
    fused.spec_accept(*cuda, max_new)
    for got, want in zip(cuda[2:], (gen, hist, positions, n_gen, accepted)):
        assert np.array_equal(got.cpu().numpy(), want)


def test_sample_at_equals_sample_at_each_rows_step():
    from quip_b200 import fused
    B, T, V = 5, 3, 5000
    g = torch.Generator(device='cuda').manual_seed(1)
    logits = (torch.randn(B, T, V, generator=g, device='cuda') * 3).half()
    temp = torch.tensor([1.0, 0.7, 0.0, 1.3, 0.9], device='cuda')
    top_k = torch.tensor([0, 50, 0, 1, 7], dtype=torch.int32, device='cuda')
    top_p = torch.tensor([1.0, 0.9, 1.0, 0.5, 0.95], device='cuda')
    seed = torch.tensor([1, 2, 3, -4, 5], dtype=torch.int64, device='cuda')
    steps = torch.tensor([0, 7, 3, 1 << 40, 19], dtype=torch.int64, device='cuda')
    got = fused.sample_at(logits, temp, top_k, top_p, seed, steps, torch.zeros(B, T, dtype=torch.long, device='cuda'))
    for b in range(B):
        for i in range(T):
            one = torch.zeros(1, dtype=torch.long, device='cuda')
            fused.sample(logits[b, i][None].contiguous(), temp[b:b + 1], top_k[b:b + 1], top_p[b:b + 1], seed[b:b + 1],
                         steps[b:b + 1] + i, one)
            assert int(got[b, i]) == int(one), (b, i)


# ---- SpecDecoder on the synthetic packed models of test_gpu_generate

def _tiny(kind):
    from transformers import LlamaConfig, OPTConfig
    from quip_b200.synth import build_synthetic_model
    if kind == 'opt':
        cfg = OPTConfig(hidden_size=256, ffn_dim=1024, num_hidden_layers=2, num_attention_heads=4, vocab_size=320,
                        max_position_embeddings=128, word_embed_proj_dim=256)
    else:
        nkv, hd = kind
        cfg = LlamaConfig(hidden_size=4 * hd, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                          num_key_value_heads=nkv, vocab_size=320, max_position_embeddings=128)
    return build_synthetic_model(cfg, torch.device('cuda:0'), bits=2, incoh='blocked', rescale=True, seed=5, seqlen=64)


def _prompts():
    """Prompts with repeats, so that lookup finds matches from the first step."""
    g = torch.Generator().manual_seed(7)
    base = [torch.randint(0, 320, (n,), generator=g) for n in (5, 3, 6)]
    return [torch.cat((p, p, p[:2])) for p in base]


def _run_spec(model, prompts, n, k, capture, kv_dtype=None):
    from quip_b200.decode import SpecDecoder
    dec = SpecDecoder(model, max_len=64, batch=len(prompts), max_new=n, draft_tokens=k, kv_dtype=kv_dtype)
    if capture:
        dec.capture()
    log = []
    with torch.no_grad():
        dec.prefill(prompts)
        for _ in range(n - 1):
            g0 = dec.n_gen.clone()
            logits = dec.step().float().clone()
            log.append((g0, dec.n_gen.clone(), logits))
    return dec, log


@pytest.mark.parametrize('kind', [(2, 64), 'opt'])
def test_spec_graph_replay_equals_the_eager_spec_step(kind):
    model = _tiny(kind)
    e, elog = _run_spec(model, _prompts(), 16, 4, capture=False)
    g, glog = _run_spec(model, _prompts(), 16, 4, capture=True)
    assert torch.equal(e.generated, g.generated) and torch.equal(e.accepted, g.accepted)
    for (a0, a1, la), (b0, b1, lb) in zip(elog, glog):
        assert torch.equal(a0, b0) and torch.equal(a1, b1) and torch.equal(la, lb)


def _norms(model):
    if model.config.model_type == 'opt':
        d = model.model.decoder
        return [m for layer in d.layers for m in (layer.self_attn_layer_norm, layer.final_layer_norm)] + [d.final_layer_norm]
    return [m for layer in model.model.layers for m in (layer.input_layernorm, layer.post_attention_layernorm)] + [model.model.norm]


@pytest.mark.parametrize('kv_dtype', [None, torch.float8_e4m3fn])
@pytest.mark.parametrize('kind', [(4, 64), (2, 64), (2, 128), 'opt'])
def test_spec_tokens_are_the_verify_steps_own_choice_and_its_logits_match_eager_hf(kind, kv_dtype):
    import bench
    model = _tiny(kind)
    prompts, n = _prompts(), 20
    dec, log = _run_spec(model, prompts, n, 4, capture=True, kv_dtype=kv_dtype)
    assert int(dec.accepted.sum()) > 0
    gen = dec.generated.cpu()
    assert dec.n_gen.tolist() == [n] * len(prompts)
    worst = control = 0.0
    for b, p in enumerate(prompts):
        fed = torch.cat((p, gen[b, :n - 1])).cuda()[None]
        runs = []
        for flip in (False, True):
            hooks = bench._ulp_flip_hooks(_norms(model), 3e-5, seed=b) if flip else []
            try:
                with torch.no_grad():
                    runs.append(model(fed).logits[0].float())
            finally:
                for hk in hooks:
                    hk.remove()
        want, ctrl = runs
        P = p.numel()
        for g0, g1, logits in log:
            s, e = int(g0[b]), int(g1[b])
            for i in range(e - s):
                # token i of the step predicts generated[s + i]; its input sits at position P + s - 1 + i
                assert int(logits[b, i].argmax()) == int(gen[b, s + i]), (b, s, i)
                w = want[P + s - 1 + i]
                worst = max(worst, float((logits[b, i] - w).norm() / w.norm()))
                control = max(control, float((ctrl[P + s - 1 + i] - w).norm() / w.norm()))
    if kv_dtype is None:
        assert worst < max(2e-3, 3.0 * control), (worst, control)
    else:                                                             # one e4m3 rounding of every cached key and value
        assert worst < 0.1, (worst, control)


@pytest.mark.parametrize('kv_dtype', [None, torch.float8_e4m3fn])
@pytest.mark.parametrize('kind', [(4, 64), (2, 128), 'opt'])
def test_spec_generation_equals_plain_generation_away_from_near_ties(kind, kv_dtype):
    """Plain and speculative steps run the linears at other token counts, so their logits differ by rounding.  A token
    can differ only where the plain run's top-2 gap is at most twice the largest logit difference of the two runs at that
    position; up to the first such position the tokens must agree."""
    from quip_b200.decode import PromptDecoder
    model = _tiny(kind)
    prompts, n = _prompts(), 20
    dec, log = _run_spec(model, prompts, n, 4, capture=True, kv_dtype=kv_dtype)
    assert int(dec.accepted.sum()) > 0
    plain = PromptDecoder(model, max_len=64, batch=len(prompts), max_new=n, kv_dtype=kv_dtype).capture()
    with torch.no_grad():
        plogits = [plain.prefill(prompts).float().clone()]
        plogits += [plain.step().float().clone() for _ in range(n - 1)]
    spec_gen, plain_gen = dec.generated.cpu(), plain.generated.cpu()
    checked = 0
    for b in range(len(prompts)):
        slog = {}
        for g0, g1, logits in log:
            for i in range(int(g1[b]) - int(g0[b])):
                slog[int(g0[b]) + i] = logits[b, i]
        for j in range(1, n):                                         # plogits[j] predicts generated[j]
            top2 = plogits[j][b].topk(2).values
            diff = float((slog[j] - plogits[j][b]).abs().max())
            if float(top2[0] - top2[1]) <= 2 * diff:
                break
            assert int(spec_gen[b, j]) == int(plain_gen[b, j]), (b, j)
            checked += 1
        assert int(spec_gen[b, 0]) == int(plain_gen[b, 0])
    assert checked >= n // 2, checked


def test_generate_speculative_sampled_and_greedy_run_and_count_acceptance():
    from quip_b200.decode import generate
    model = _tiny((2, 64))
    prompts = _prompts()
    stats = {}
    out = generate(model, prompts, 24, prompt_lookup_num_tokens=4, spec_stats=stats)
    assert [o.numel() for o in out] == [24] * 3 and sum(stats['accepted']) > 0
    a = generate(model, prompts, 24, prompt_lookup_num_tokens=4, do_sample=True, seed=[1, 2, 3], top_k=20)
    b = generate(model, prompts, 24, prompt_lookup_num_tokens=4, do_sample=True, seed=[1, 2, 3], top_k=20)
    assert all(torch.equal(x, y) for x, y in zip(a, b))
