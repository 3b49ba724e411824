"""The decode-attention kernel (csrc/attn_decode.cu) against float64 torch, and generation from prompts
(quip_b200/decode.py: PromptDecoder, generate) on synthetic packed models against the eager HF decode."""
import math

import pytest
import torch

pytestmark = pytest.mark.gpu

CHUNK = 128          # KV slots per CTA of the kernel (AD_CHUNK) ...


def _chunk(B, nkv, max_len):
    """... or 64 when that grid would hold fewer than 2 * 132 CTAs (csrc/attn_decode.cu)."""
    return 64 if B * nkv * -(-max_len // CHUNK) < 2 * 132 else CHUNK


def _attn(q, k_new, v_new, kc, vc, pos, scale):
    from quip_b200 import fused
    return fused.decode_attention(q, k_new, v_new, kc, vc, pos, scale)


def _case(B, G, hd, max_len, positions, seed=0, nkv=2):
    g = torch.Generator(device='cuda').manual_seed(seed)
    nh = G * nkv

    def r(*s):
        return torch.randn(*s, generator=g, device='cuda').half()
    q, kn, vn = r(B, nh, hd), r(B, nkv, hd), r(B, nkv, hd)
    kc, vc = r(B, nkv, max_len, hd), r(B, nkv, max_len, hd)
    pos = torch.tensor(positions, dtype=torch.long, device='cuda')
    return q, kn, vn, kc, vc, pos


def _reference(q, kn, vn, kc, vc, pos, scale):
    """float64, with the new key / value at slot pos[b] and slots 0 .. pos[b] only."""
    B, nh, hd = q.shape
    G = nh // kn.shape[1]
    out = torch.empty(B, nh, hd, dtype=torch.float64, device=q.device)
    for b in range(B):
        p = int(pos[b])
        K, V = kc[b, :, :p + 1].double().clone(), vc[b, :, :p + 1].double().clone()
        K[:, p], V[:, p] = kn[b].double(), vn[b].double()
        K, V = K.repeat_interleave(G, 0), V.repeat_interleave(G, 0)
        s = torch.einsum('hd,hjd->hj', q[b].double(), K) * scale
        out[b] = torch.einsum('hj,hjd->hd', torch.softmax(s, -1), V)
    return out


def _edges(chunk, max_len):
    return [0, chunk - 1, chunk, chunk + 1, 2 * chunk - 1, 2 * chunk, 2 * chunk + 1, max_len - 1]


def _positions(B, max_len, seed, edge):
    g = torch.Generator().manual_seed(seed)
    return [edge[b] if b < len(edge) else int(torch.randint(0, max_len, (1,), generator=g)) for b in range(B)]


@pytest.mark.parametrize('hd', [64, 128])
@pytest.mark.parametrize('G', [1, 4, 8])
@pytest.mark.parametrize('B', [1, 3, 32])
def test_kernel_matches_float64_attention_on_ragged_positions(hd, G, B):
    max_len = 3 * CHUNK + 40
    nkv = 8 if B == 32 else 2                                         # 32 rows: 128-slot chunks, fewer: 64-slot chunks
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
        q, kn, vn, kc, vc, pos = _case(B, G, hd, max_len, positions, seed=hd + G + B, nkv=nkv)
        k0, v0 = kc.clone(), vc.clone()
        out = _attn(q, kn, vn, kc, vc, pos, scale)
        ref = _reference(q, kn, vn, k0, v0, pos, scale)
        for b in range(B):
            err = float((out[b].double() - ref[b]).norm() / ref[b].norm())
            assert err < 1e-3, (positions[b], b, err)
        # append is exact: slot pos[b] holds k_new / v_new bit for bit, every other byte is unchanged
        rows = torch.arange(B, device='cuda')
        k0[rows, :, pos], v0[rows, :, pos] = kn, vn
        assert torch.equal(kc, k0) and torch.equal(vc, v0)


@pytest.mark.parametrize('hd', [64, 128])
def test_kernel_never_reads_past_the_position_and_rows_are_independent(hd):
    B, G, max_len = 6, 4, 4 * CHUNK
    c = _chunk(B, 2, max_len)
    positions = [0, c - 1, c, c + 1, 3 * CHUNK + 7, max_len - 1]
    q, kn, vn, kc, vc, pos = _case(B, G, hd, max_len, positions, seed=11)
    scale = 1.0 / math.sqrt(hd)
    clean = _attn(q, kn, vn, kc.clone(), vc.clone(), pos, scale)
    again = _attn(q, kn, vn, kc.clone(), vc.clone(), pos, scale)
    assert torch.equal(clean, again)                                  # deterministic
    kp, vp = kc.clone(), vc.clone()
    for b, p in enumerate(positions):
        kp[b, :, p:] = float('nan')                                   # slot p too: the kernel takes k_new / v_new there
        vp[b, :, p:] = float('nan')
    poisoned = _attn(q, kn, vn, kp, vp, pos, scale)
    assert torch.isfinite(poisoned).all() and torch.equal(poisoned, clean)
    # other rows at other positions, with other contents: row 2's result does not move
    q2, kn2, vn2, kc2, vc2, _ = _case(B, G, hd, max_len, positions, seed=12)
    for t2, t in ((q2, q), (kn2, kn), (vn2, vn), (kc2, kc), (vc2, vc)):
        t2[2] = t[2]
    pos2 = torch.tensor([max_len - 1, 5, positions[2], 2 * CHUNK, 0, 77], dtype=torch.long, device='cuda')
    other = _attn(q2, kn2, vn2, kc2, vc2, pos2, scale)
    assert torch.equal(other[2], clean[2])


def _tiny(kind):
    from transformers import LlamaConfig, OPTConfig
    from quip_b200.synth import build_synthetic_model
    if kind == 'opt':
        cfg = OPTConfig(hidden_size=256, ffn_dim=1024, num_hidden_layers=2, num_attention_heads=4, vocab_size=320,
                        max_position_embeddings=128, word_embed_proj_dim=256)
    else:
        nkv, hd = kind
        hidden = 4 * hd
        cfg = LlamaConfig(hidden_size=hidden, intermediate_size=512, num_hidden_layers=2, num_attention_heads=4,
                          num_key_value_heads=nkv, vocab_size=320, max_position_embeddings=128)
    return build_synthetic_model(cfg, torch.device('cuda:0'), bits=2, incoh='blocked', rescale=True, seed=5, seqlen=64)


MODELS = [(4, 64), (2, 64), (2, 128), 'opt']


def _norms(model):
    if model.config.model_type == 'opt':
        d = model.model.decoder
        return [m for layer in d.layers for m in (layer.self_attn_layer_norm, layer.final_layer_norm)] + [d.final_layer_norm]
    return [m for layer in model.model.layers for m in (layer.input_layernorm, layer.post_attention_layernorm)] + [model.model.norm]


def _prompts():
    g = torch.Generator().manual_seed(7)
    return [torch.randint(0, 320, (n,), generator=g) for n in (9, 4, 17)]


@pytest.mark.parametrize('kind', MODELS)
def test_generation_matches_eager_hf_decode_and_batch_one(kind):
    import bench
    from quip_b200.decode import PromptDecoder
    model = _tiny(kind)
    prompts, n = _prompts(), 12
    with torch.no_grad():
        dec = PromptDecoder(model, max_len=40, batch=3, max_new=n).capture()
        got = [dec.prefill(prompts).float().clone()]
        got += [dec.step().float().clone() for _ in range(n - 1)]
        tokens = dec.generated.cpu()
    worst = control = 0.0
    for b, p in enumerate(prompts):
        fed = torch.cat((p, tokens[b, :n - 1])).cuda()
        runs = []
        for flip in (False, True):
            past, res = None, []
            with torch.no_grad():
                for i in range(p.numel() - 1, fed.numel()):
                    hooks = bench._ulp_flip_hooks(_norms(model), 3e-5, seed=i) if flip else []
                    try:
                        x = fed[None, :i + 1] if past is None else fed[None, i:i + 1]
                        out = model(x, past_key_values=past, use_cache=True)
                    finally:
                        for hk in hooks:
                            hk.remove()
                    past = out.past_key_values
                    res.append(out.logits[0, -1].float())
            runs.append(res)
        want, ctrl = runs
        for i in range(n):
            w = want[i]
            worst = max(worst, float((got[i][b] - w).norm() / w.norm()))
            control = max(control, float((ctrl[i] - w).norm() / w.norm()))
    assert worst < max(2e-3, 3.0 * control), (worst, control)
    # each prompt alone, fed the same tokens: other token counts take other few-token routes
    for b, p in enumerate(prompts):
        with torch.no_grad():
            one = PromptDecoder(model, max_len=40, batch=1).capture()
            first = one.prefill([p]).float()
            assert float((first[0] - got[0][b]).norm() / got[0][b].norm()) < 5e-3
            for i in range(n - 1):
                lg = one.step(tokens[b, i:i + 1].cuda())[0].float()
                err = float((lg - got[i + 1][b]).norm() / got[i + 1][b].norm())
                assert err < 5e-3, (b, i, err)


def test_generate_returns_the_greedy_tokens_of_the_decoder():
    from quip_b200.decode import PromptDecoder, generate
    model = _tiny((2, 64))
    prompts = _prompts()
    out = generate(model, prompts, 20)
    with torch.no_grad():
        dec = PromptDecoder(model, max_len=37, batch=3, max_new=20).capture()
        dec.prefill(prompts)
        for _ in range(19):
            dec.step()
    for b in range(3):
        assert torch.equal(out[b], dec.generated[b].cpu())


@pytest.mark.parametrize('kind', [(2, 64), 'opt'])
def test_graph_replay_equals_the_eager_prompt_decoder_step(kind):
    from quip_b200.decode import PromptDecoder
    model = _tiny(kind)
    prompts = _prompts()
    ids = torch.randint(0, 320, (3, 6), generator=torch.Generator().manual_seed(9)).cuda()
    with torch.no_grad():
        eager = PromptDecoder(model, max_len=32, batch=3)
        eager.prefill(prompts)
        e = [eager.step(ids[:, i]).clone() for i in range(ids.shape[1])]
        graph = PromptDecoder(model, max_len=32, batch=3).capture()
        graph.prefill(prompts)
        g = [graph.step(ids[:, i]).clone() for i in range(ids.shape[1])]
    for i, (a, b) in enumerate(zip(e, g)):
        assert torch.equal(a, b), i


@pytest.mark.parametrize('kind', [(4, 64), (2, 128), 'opt'])
def test_uniform_positions_agree_with_graph_decoder(kind):
    from quip_b200.decode import GraphDecoder, PromptDecoder
    model = _tiny(kind)
    ids = torch.randint(0, 320, (3, 10), generator=torch.Generator().manual_seed(8)).cuda()
    with torch.no_grad():
        g = GraphDecoder(model, max_len=16, batch=3).capture()
        p = PromptDecoder(model, max_len=16, batch=3).capture()
        for i in range(ids.shape[1]):
            a, b = g.step(ids[:, i]).float(), p.step(ids[:, i]).float()
            err = float((a - b).norm() / a.norm())
            assert err < 2e-3, (i, err)


def test_generate_one_token_and_capture_from_a_full_cache():
    """max_new_tokens = 1 needs no decode step.  A decoder captured with a row's cache full and its generated buffer full
    warms up in range and leaves its state as it was; after reset() its graph generates what a fresh decoder's does."""
    from quip_b200.decode import PromptDecoder, generate
    model = _tiny((2, 64))
    prompts = _prompts()
    one = generate(model, prompts, 1)
    with torch.no_grad():
        first = PromptDecoder(model, max_len=18, batch=3).prefill(prompts).argmax(-1).cpu()
        assert [t.tolist() for t in one] == [[int(t)] for t in first]
        dec = PromptDecoder(model, max_len=19, batch=3, max_new=3)
        dec.prefill(prompts)
        dec.step()
        dec.step()                                                    # row 2 at max_len, generated full
        pos, gen = dec.positions.clone(), dec.generated.clone()
        dec.capture()
        assert torch.equal(dec.positions, pos) and torch.equal(dec.generated, gen)
        dec.reset()
        fresh = PromptDecoder(model, max_len=19, batch=3, max_new=3).capture()
        for d in (dec, fresh):
            d.prefill([p[:6] for p in prompts])
            d.step()
            d.step()
        assert torch.equal(dec.generated, fresh.generated) and torch.equal(dec.logits, fresh.logits)
