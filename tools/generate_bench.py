"""Generation from prompts on Llama-2-7B / 70B shapes (synthetic 2-bit packed weights, quip_b200.synth): prefill
tokens/s, decode step time of GraphDecoder (uniform positions, SDPA over the whole static cache, repeat_interleave for
GQA) against PromptDecoder (per-row positions, csrc/attn_decode.cu), and the decode-attention kernel alone against the
HBM bandwidth of the H100 SXM data sheet (3.35 TB/s).  Needs a CUDA device.

    python tools/generate_bench.py --out DIR [--models llama7b,llama70b] [--layers70b 80] [--steps 16]

Prints one line per measurement and writes DIR/generate_bench.json.  The decode steps of both decoders run at the same
positions on one shared cache, alternating in the same process, and their logits are compared.  A decode configuration
whose cache (twice over: GraphDecoder.capture keeps a copy) does not fit the free device memory is skipped and listed.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

HBM_BPS = 3.35e12                     # H100 SXM data sheet


def card():
    info = dict(name=torch.cuda.get_device_name(0))
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30)
        info['nvidia_smi'] = r.stdout.strip().splitlines()[0] if r.stdout.strip() else r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info['nvidia_smi'] = f'unavailable: {e}'
    return info


def events_ms(fn, reps, warm=3):
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def attn_bytes(positions, nkv, hd):
    """HBM bytes the kernel must read: the valid prefix of K and V of every row (fp16)."""
    return sum(2 * nkv * (int(p) + 1) * hd * 2 for p in positions)


def kernel_alone(nh, nkv, hd, B, ctx, reps):
    """quip_decode_attention at every row's position ctx-1 of a cache of ctx slots, and the torch attention GraphDecoder
    runs for the same step (index_copy_ of k / v, repeat_interleave for GQA, SDPA over the cache under the mask)."""
    from quip_b200 import fused
    g = torch.Generator(device='cuda').manual_seed(0)
    kc = torch.randn(B, nkv, ctx, hd, generator=g, device='cuda').half()
    vc = torch.randn(B, nkv, ctx, hd, generator=g, device='cuda').half()
    q = torch.randn(B, nh, hd, generator=g, device='cuda').half()
    kn, vn = kc[:, :, -1].clone(), vc[:, :, -1].clone()
    pos = torch.full((B,), ctx - 1, dtype=torch.long, device='cuda')
    scale = hd ** -0.5
    ms = events_ms(lambda: fused.decode_attention(q, kn, vn, kc, vc, pos, scale), reps)
    nbytes = attn_bytes(pos.tolist(), nkv, hd)
    p1 = pos[:1]
    mask = (torch.arange(ctx, device='cuda') <= p1)[None, None, None, :]

    def torch_step():
        kc.index_copy_(2, p1, kn[:, :, None])
        vc.index_copy_(2, p1, vn[:, :, None])
        kk, vv = kc, vc
        if nkv != nh:
            kk, vv = kk.repeat_interleave(nh // nkv, dim=1), vv.repeat_interleave(nh // nkv, dim=1)
        return torch.nn.functional.scaled_dot_product_attention(q[:, :, None], kk, vv, attn_mask=mask, scale=scale)
    ms_torch = events_ms(torch_step, max(reps // 4, 5))
    ref = torch_step()[:, :, 0].float()
    got = fused.decode_attention(q, kn, vn, kc, vc, pos, scale).float()
    err = float((got - ref).norm() / ref.norm())
    del kc, vc
    torch.cuda.empty_cache()
    return dict(nh=nh, nkv=nkv, hd=hd, B=B, context=ctx, kernel_ms=ms, bytes=nbytes, bytes_per_s=nbytes / ms * 1e3,
                share_of_3_35_TBps=nbytes / ms * 1e3 / HBM_BPS, torch_attention_ms=ms_torch, rel_err_vs_torch=err)


def rel(a, b):
    return float((a.float() - b.float()).norm() / b.float().norm())


def decode_steps(model, B, ctx, steps, trials=3):
    """Per-step ms of GraphDecoder and PromptDecoder, both captured, at every row's position ctx .. ctx+steps-1."""
    from quip_b200.decode import GraphDecoder, PromptDecoder
    max_len = ctx + steps
    gd = GraphDecoder(model, max_len=max_len, batch=B)
    gd.k_cache.normal_(0.0, 0.5)
    gd.v_cache.normal_(0.0, 0.5)
    gd.capture()
    pd = PromptDecoder(model, max_len=max_len, batch=B)
    pd.k_cache, pd.v_cache = gd.k_cache, gd.v_cache                  # one cache: same contents for both
    torch.cuda.empty_cache()
    pd.capture()
    ids = torch.randint(0, model.config.vocab_size, (steps, B), generator=torch.Generator().manual_seed(1)).cuda()

    def run(dec):
        if dec is gd:
            gd.position.fill_(ctx)
            gd._pos_host = ctx
        else:
            pd.positions.fill_(ctx)
            pd._pos_host = [ctx] * B
        first = dec.step(ids[0]).clone()
        for i in range(1, steps):
            dec.step(ids[i])
        return first

    res = {'graph': [], 'prompt': []}
    err = 0.0
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for t in range(trials + 1):
        firsts = {}
        for name, dec in (('graph', gd), ('prompt', pd)):
            torch.cuda.synchronize()
            e0.record()
            firsts[name] = run(dec)
            e1.record()
            torch.cuda.synchronize()
            if t:                                                      # trial 0 warms up
                res[name].append(e0.elapsed_time(e1) / steps)
        err = max(err, rel(firsts['prompt'], firsts['graph']))
    gms, pms = sorted(res['graph'])[trials // 2], sorted(res['prompt'])[trials // 2]
    del gd, pd
    torch.cuda.empty_cache()
    return dict(B=B, context=ctx, graph_decoder_ms=gms, prompt_decoder_ms=pms, graph_decoder_tok_s=B * 1e3 / gms,
                prompt_decoder_tok_s=B * 1e3 / pms, logits_rel_err=err, trials_ms=res)


def prefill_rate(model, B, P, reps=3):
    from quip_b200.decode import PromptDecoder
    g = torch.Generator().manual_seed(2)
    prompts = [torch.randint(0, model.config.vocab_size, (P,), generator=g) for _ in range(B)]
    dec = PromptDecoder(model, max_len=P + 1, batch=B)
    ms = events_ms(lambda: dec.prefill(prompts), reps, warm=1)
    del dec
    torch.cuda.empty_cache()
    return dict(B=B, P=P, ms=ms, tokens_per_s=B * P * 1e3 / ms)


def cache_bytes(cfg, layers, B, max_len):
    nkv = getattr(cfg, 'num_key_value_heads', None) or cfg.num_attention_heads
    return 2 * layers * B * nkv * max_len * (cfg.hidden_size // cfg.num_attention_heads) * 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--models', default='llama7b,llama70b')
    ap.add_argument('--layers70b', type=int, default=80, help='decoder layers of the 70B shape to build (of 80)')
    ap.add_argument('--steps', type=int, default=16)
    ap.add_argument('--kernel-reps', type=int, default=100)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('generate_bench needs a CUDA device')
    from quip_b200.synth import build_synthetic_model, model_config
    os.makedirs(a.out, exist_ok=True)
    out = dict(card=card(), glue='QUIP_FUSED_LAYER=' + os.environ.get('QUIP_FUSED_LAYER', 'unset'), models={})
    print(json.dumps(out['card']), flush=True)
    for name in a.models.split(','):
        layers = a.layers70b if name == 'llama70b' else None
        cfg = model_config(name, **({'num_hidden_layers': layers} if layers else {}))
        nh, hd = cfg.num_attention_heads, cfg.hidden_size // cfg.num_attention_heads
        nkv = cfg.num_key_value_heads
        rec = dict(layers=cfg.num_hidden_layers, nh=nh, nkv=nkv, hd=hd, kernel=[], decode=[], prefill=[], skipped=[])
        out['models'][name] = rec
        for B in (1, 8, 32):
            for ctx in (128, 2048, 4096):
                r = kernel_alone(nh, nkv, hd, B, ctx, a.kernel_reps)
                rec['kernel'].append(r)
                print(f'{name} kernel B={B} ctx={ctx}: {r["kernel_ms"]:.4f} ms, {r["bytes_per_s"] / 1e12:.2f} TB/s '
                      f'({100 * r["share_of_3_35_TBps"]:.0f}% of 3.35), torch attention {r["torch_attention_ms"]:.4f} ms, '
                      f'rel err {r["rel_err_vs_torch"]:.1e}', flush=True)
        model = build_synthetic_model(cfg, torch.device('cuda:0'), bits=2, seed=0, seqlen=4096)
        for B, P in ((1, 2048), (8, 512)):
            r = prefill_rate(model, B, P)
            rec['prefill'].append(r)
            print(f'{name} prefill {B}x{P}: {r["ms"]:.1f} ms, {r["tokens_per_s"]:.0f} tokens/s', flush=True)
        for B in (1, 8, 32):
            for ctx in (128, 2048, 4096):
                free = torch.cuda.mem_get_info()[0]
                need = 2 * cache_bytes(cfg, cfg.num_hidden_layers, B, ctx + a.steps) + (4 << 30)
                if need > free:
                    rec['skipped'].append(dict(B=B, context=ctx, need_bytes=need, free_bytes=free))
                    print(f'{name} decode B={B} ctx={ctx}: skipped, needs {need / 2**30:.1f} GiB of {free / 2**30:.1f}', flush=True)
                    continue
                r = decode_steps(model, B, ctx, a.steps)
                rec['decode'].append(r)
                print(f'{name} decode B={B} ctx={ctx}: GraphDecoder {r["graph_decoder_ms"]:.3f} ms/step '
                      f'({r["graph_decoder_tok_s"]:.0f} tok/s), PromptDecoder {r["prompt_decoder_ms"]:.3f} ms/step '
                      f'({r["prompt_decoder_tok_s"]:.0f} tok/s), logits rel err {r["logits_rel_err"]:.1e}', flush=True)
        del model
        torch.cuda.empty_cache()
    with open(os.path.join(a.out, 'generate_bench.json'), 'w') as f:
        json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
