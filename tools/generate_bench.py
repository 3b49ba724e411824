"""Generation from prompts on Llama-2-7B / 70B shapes (synthetic 2-bit packed weights, quip_b200.synth): prefill
tokens/s, decode step time of GraphDecoder (uniform positions, SDPA over the whole static cache, repeat_interleave for
GQA) against PromptDecoder (per-row positions, csrc/attn_decode.cu), and the decode-attention kernel alone against the
HBM bandwidth of the H100 SXM data sheet (3.35 TB/s).  Needs a CUDA device.

    python tools/generate_bench.py --out DIR [--models llama7b,llama70b] [--layers70b 80] [--steps 16]
                                   [--sections kernel,prefill,decode,fp8]      (fp8kernel: the fp8 kernel rows only;
                                                                                sample: the sampling rows)

Section fp8 measures the e4m3 KV cache (PromptDecoder(kv_dtype=torch.float8_e4m3fn)): the fp8 kernel alone next to the
fp16 one (bytes: hd per cached K / V vector plus its 4-byte scale), PromptDecoder steps fp16 against fp8 at B = 32 and
contexts 2048 / 4096 (alternating in one process, one decoder allocated at a time, both caches filled from the same
values; logits compared), and configurations whose fp16 cache does not fit the card, run with fp8 or listed with the
bytes they need.

Section sample times quip_sample (csrc/sample.cu) alone for B in {1, 32, 128} x V in {32000, 50272, 128256} at
T = 0.7, k = 50, p = 0.9 and at k = 0, p = 0.9, next to torch.argmax and the torch warper chain (temperature, top-k, sort,
softmax, cumsum, top-p mask, multinomial) on the same rows, and a 7B PromptDecoder step at B = 32, context 2048, greedy
against sampling, alternated over three trials.

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


def attn_bytes(positions, nkv, hd, fp8=False):
    """HBM bytes the kernel must read: the valid prefix of K and V of every row (fp16, or e4m3 plus a 4-byte scale per
    vector)."""
    per = hd + 4 if fp8 else hd * 2
    return sum(2 * nkv * (int(p) + 1) * per for p in positions)


def kernel_alone_fp8(nh, nkv, hd, B, ctx, reps):
    """quip_decode_attention_fp8 at every row's position ctx-1 of an e4m3 cache of ctx slots; rel err against the fp16
    kernel on the unquantized cache."""
    from quip_b200 import fused
    g = torch.Generator(device='cuda').manual_seed(0)
    k16 = torch.randn(B, nkv, ctx, hd, generator=g, device='cuda').half()
    v16 = torch.randn(B, nkv, ctx, hd, generator=g, device='cuda').half()
    q = torch.randn(B, nh, hd, generator=g, device='cuda').half()
    kn, vn = k16[:, :, -1].clone(), v16[:, :, -1].clone()
    pos = torch.full((B,), ctx - 1, dtype=torch.long, device='cuda')
    scale = hd ** -0.5
    ref = fused.decode_attention(q, kn, vn, k16, v16, pos, scale).float()
    kc = torch.empty(B, nkv, ctx, hd, dtype=torch.float8_e4m3fn, device='cuda')
    vc = torch.empty_like(kc)
    ks = torch.empty(B, nkv, ctx, device='cuda')
    vs = torch.empty_like(ks)
    fused.kv_quantize(k16, kc, ks)
    fused.kv_quantize(v16, vc, vs)
    del k16, v16
    ms = events_ms(lambda: fused.decode_attention(q, kn, vn, kc, vc, pos, scale, k_scale=ks, v_scale=vs), reps)
    nbytes = attn_bytes(pos.tolist(), nkv, hd, fp8=True)
    err = rel(fused.decode_attention(q, kn, vn, kc, vc, pos, scale, k_scale=ks, v_scale=vs), ref)
    del kc, vc
    torch.cuda.empty_cache()
    return dict(kv='fp8', nh=nh, nkv=nkv, hd=hd, B=B, context=ctx, kernel_ms=ms, bytes=nbytes,
                bytes_per_s=nbytes / ms * 1e3, share_of_3_35_TBps=nbytes / ms * 1e3 / HBM_BPS, rel_err_vs_fp16=err)


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


def cache_bytes(cfg, layers, B, max_len, fp8=False):
    """K and V cache bytes: fp16, or e4m3 plus one fp32 scale per cached vector."""
    nkv = getattr(cfg, 'num_key_value_heads', None) or cfg.num_attention_heads
    hd = cfg.hidden_size // cfg.num_attention_heads
    return 2 * layers * B * nkv * max_len * (hd + 4 if fp8 else hd * 2)


def _filled_prompt_decoder(model, B, ctx, max_len, fp8):
    """A captured PromptDecoder whose rows sit at position ctx over a cache filled from seeded fp16 values (the same
    values for either dtype: stored as they are, or quantized with quip_kv_quantize_fp8)."""
    from quip_b200 import fused
    from quip_b200.decode import PromptDecoder
    dec = PromptDecoder(model, max_len=max_len, batch=B, kv_dtype=torch.float8_e4m3fn if fp8 else None)
    L, nkv, hd = len(dec.layers), dec.nkv, dec.hd
    for li in range(L):
        for i, (cache, scales) in enumerate(((dec.k_cache, dec.k_scale), (dec.v_cache, dec.v_scale))):
            g = torch.Generator(device='cuda').manual_seed(2 * li + i)
            src = (torch.randn(B, nkv, ctx, hd, generator=g, device='cuda') * 0.5).half()
            if fp8:
                fused.kv_quantize(src, cache[li], scales[li])
            else:
                cache[li, :, :, :ctx].copy_(src)
            del src
    torch.cuda.empty_cache()
    dec.capture()
    return dec


def decode_steps_fp8(model, B, ctx, steps, trials=2, kinds=('fp16', 'fp8')):
    """Per-step ms of captured PromptDecoders with an fp16 and an e4m3 cache at every row's position ctx .. ctx+steps-1,
    alternating trial by trial in this process; one decoder is allocated at a time, so each kind needs 1x its cache."""
    max_len = ctx + steps
    ids = torch.randint(0, model.config.vocab_size, (steps, B), generator=torch.Generator().manual_seed(1)).cuda()
    res = {k: [] for k in kinds}
    firsts = {}
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    for t in range(trials + 1):
        for kind in kinds:
            dec = _filled_prompt_decoder(model, B, ctx, max_len, kind == 'fp8')
            with torch.no_grad():
                for rep in range(2):                                  # the first pass warms up
                    dec.positions.fill_(ctx)
                    dec._pos_host = [ctx] * B
                    torch.cuda.synchronize()
                    e0.record()
                    first = dec.step(ids[0]).clone()
                    for i in range(1, steps):
                        dec.step(ids[i])
                    e1.record()
                    torch.cuda.synchronize()
                    if rep and t:                                     # trial 0 warms up
                        res[kind].append(e0.elapsed_time(e1) / steps)
            firsts[kind] = first
            del dec
            torch.cuda.empty_cache()
    out = dict(B=B, context=ctx, trials_ms=res)
    for kind in kinds:
        ms = sorted(res[kind])[len(res[kind]) // 2]
        out[f'{kind}_ms'] = ms
        out[f'{kind}_tok_s'] = B * 1e3 / ms
    if len(kinds) == 2:
        out['logits_rel_err_fp8_vs_fp16'] = rel(firsts['fp8'], firsts['fp16'])
    return out


def torch_warpers(x, T, k, p):
    """HF-style sampling chain in torch ops: temperature, top-k, top-p over a descending sort, multinomial."""
    z = x.float() / T
    if k:
        kth = torch.topk(z, k, dim=-1).values[:, -1:]
        z = z.masked_fill(z < kth, float('-inf'))
    s, idx = torch.sort(z, descending=True, dim=-1)
    cs = torch.softmax(s, -1).cumsum(-1)
    drop = (cs - torch.softmax(s, -1)) >= p                             # mass ranked strictly above is >= p
    s = s.masked_fill(drop, float('-inf'))
    pick = torch.multinomial(torch.softmax(s, -1), 1)
    return idx.gather(-1, pick)[:, 0]


def sample_alone(B, V, k, p, reps):
    from quip_b200 import fused
    g = torch.Generator(device='cuda').manual_seed(0)
    x = (torch.randn(B, V, generator=g, device='cuda') * 3).half()
    T = torch.full((B,), 0.7, device='cuda')
    kk = torch.full((B,), k, dtype=torch.int32, device='cuda')
    pp = torch.full((B,), p, device='cuda')
    sd = torch.arange(B, dtype=torch.int64, device='cuda')
    step = torch.zeros(1, dtype=torch.int64, device='cuda')
    out = torch.empty(B, dtype=torch.int64, device='cuda')
    ms = events_ms(lambda: fused.sample(x, T, kk, pp, sd, step, out), reps)
    ms_argmax = events_ms(lambda: x.argmax(-1), reps)
    ms_chain = events_ms(lambda: torch_warpers(x, 0.7, k, p), max(reps // 4, 5))
    return dict(B=B, V=V, T=0.7, top_k=k, top_p=p, kernel_ms=ms, torch_argmax_ms=ms_argmax, torch_warpers_ms=ms_chain)


def sample_steps(model, B, ctx, steps, trials=3):
    """Per-step ms of a captured PromptDecoder generating greedily and one sampling (T 0.7, k 50, p 0.9) at every row's
    position ctx .. ctx+steps-1, alternating trial by trial."""
    from quip_b200.decode import PromptDecoder
    max_len = ctx + steps + 1
    res = {'greedy': [], 'sampling': []}
    for t in range(trials + 1):
        for kind in ('greedy', 'sampling'):
            dec = PromptDecoder(model, max_len=max_len, batch=B, max_new=steps + 1, sampling=kind == 'sampling')
            if kind == 'sampling':
                dec.set_sampling(temperature=0.7, top_k=50, top_p=0.9, seed=list(range(B)))
            dec.k_cache.normal_(0.0, 0.5)
            dec.v_cache.normal_(0.0, 0.5)
            dec.capture()
            with torch.no_grad():
                for rep in range(2):
                    dec.positions.fill_(ctx)
                    dec._pos_host = [ctx] * B
                    dec._t.fill_(1)
                    dec._t_host = 1
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(steps):
                        dec.step()
                    e1.record()
                    torch.cuda.synchronize()
                    if rep and t:
                        res[kind].append(e0.elapsed_time(e1) / steps)
            del dec
            torch.cuda.empty_cache()
    out = dict(B=B, context=ctx, trials_ms=res)
    for kind in res:
        out[f'{kind}_ms'] = sorted(res[kind])[len(res[kind]) // 2]
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--models', default='llama7b,llama70b')
    ap.add_argument('--layers70b', type=int, default=80, help='decoder layers of the 70B shape to build (of 80)')
    ap.add_argument('--steps', type=int, default=16)
    ap.add_argument('--kernel-reps', type=int, default=100)
    ap.add_argument('--sections', default='kernel,prefill,decode,fp8')
    a = ap.parse_args()
    sections = set(a.sections.split(','))
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
        rec = dict(layers=cfg.num_hidden_layers, nh=nh, nkv=nkv, hd=hd, kernel=[], decode=[], prefill=[], skipped=[],
                   kernel_fp8=[], decode_fp8=[], capacity_fp8=[])
        out['models'][name] = rec
        for B in (1, 8, 32) if 'kernel' in sections else ():
            for ctx in (128, 2048, 4096):
                r = kernel_alone(nh, nkv, hd, B, ctx, a.kernel_reps)
                rec['kernel'].append(r)
                print(f'{name} kernel B={B} ctx={ctx}: {r["kernel_ms"]:.4f} ms, {r["bytes_per_s"] / 1e12:.2f} TB/s '
                      f'({100 * r["share_of_3_35_TBps"]:.0f}% of 3.35), torch attention {r["torch_attention_ms"]:.4f} ms, '
                      f'rel err {r["rel_err_vs_torch"]:.1e}', flush=True)
                if sections & {'fp8', 'fp8kernel'}:
                    r = kernel_alone_fp8(nh, nkv, hd, B, ctx, a.kernel_reps)
                    rec['kernel_fp8'].append(r)
                    print(f'{name} fp8 kernel B={B} ctx={ctx}: {r["kernel_ms"]:.4f} ms, {r["bytes_per_s"] / 1e12:.2f} TB/s '
                          f'({100 * r["share_of_3_35_TBps"]:.0f}% of 3.35), rel err vs fp16 kernel {r["rel_err_vs_fp16"]:.1e}',
                          flush=True)
        if 'sample' in sections and name == 'llama7b':
            rec['sample'] = []
            for B in (1, 32, 128):
                for V in (32000, 50272, 128256):
                    for k, p in ((50, 0.9), (0, 0.9)):
                        r = sample_alone(B, V, k, p, a.kernel_reps)
                        rec['sample'].append(r)
                        print(f'sample B={B} V={V} k={k} p={p}: kernel {1e3 * r["kernel_ms"]:.1f} us, torch argmax '
                              f'{1e3 * r["torch_argmax_ms"]:.1f} us, torch warpers {1e3 * r["torch_warpers_ms"]:.1f} us',
                              flush=True)
        if not sections & {'prefill', 'decode', 'fp8', 'sample'}:
            continue
        model = build_synthetic_model(cfg, torch.device('cuda:0'), bits=2, seed=0, seqlen=4096)
        for B, P in ((1, 2048), (8, 512)) if 'prefill' in sections else ():
            r = prefill_rate(model, B, P)
            rec['prefill'].append(r)
            print(f'{name} prefill {B}x{P}: {r["ms"]:.1f} ms, {r["tokens_per_s"]:.0f} tokens/s', flush=True)
        for B in (1, 8, 32) if 'decode' in sections else ():
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
        if 'sample' in sections and name == 'llama7b':
            r = sample_steps(model, 32, 2048, a.steps)
            rec['sample_decode'] = r
            print(f'{name} PromptDecoder B=32 ctx=2048: greedy {r["greedy_ms"]:.3f} ms/step, sampling '
                  f'{r["sampling_ms"]:.3f} ms/step', flush=True)
        # fp16 against fp8 at B = 32, then the configurations only an e4m3 cache fits (7B 48 x 4096, 70B 64 x 4096)
        runs = [(32, 2048, ('fp16', 'fp8')), (32, 4096, ('fp16', 'fp8'))] if 'fp8' in sections else []
        if 'fp8' in sections:
            runs.append((48 if name == 'llama7b' else 64, 4096, ('fp8',)))
        for B, ctx, kinds in runs:
            free = torch.cuda.mem_get_info()[0]
            need = {k: cache_bytes(cfg, cfg.num_hidden_layers, B, ctx + a.steps, fp8=k == 'fp8') + (4 << 30) for k in kinds}
            need16 = cache_bytes(cfg, cfg.num_hidden_layers, B, ctx + a.steps) + (4 << 30)
            if max(need.values()) > free:
                rec['skipped'].append(dict(kv=list(kinds), B=B, context=ctx, need_bytes=need, free_bytes=free))
                print(f'{name} fp8 decode B={B} ctx={ctx}: skipped, needs {max(need.values()) / 2**30:.1f} GiB of '
                      f'{free / 2**30:.1f}', flush=True)
                continue
            r = decode_steps_fp8(model, B, ctx, a.steps, kinds=kinds)
            r.update(need_bytes=need, fp16_need_bytes=need16, free_bytes=free)
            if len(kinds) == 2:
                rec['decode_fp8'].append(r)
                print(f'{name} PromptDecoder B={B} ctx={ctx}: fp16 cache {r["fp16_ms"]:.3f} ms/step ({r["fp16_tok_s"]:.0f} '
                      f'tok/s), fp8 cache {r["fp8_ms"]:.3f} ms/step ({r["fp8_tok_s"]:.0f} tok/s), logits rel err '
                      f'{r["logits_rel_err_fp8_vs_fp16"]:.1e}', flush=True)
            else:
                rec['capacity_fp8'].append(r)
                print(f'{name} PromptDecoder B={B} ctx={ctx} fp8 cache ({need["fp8"] / 2**30:.1f} GiB with margin; fp16 '
                      f'would need {need16 / 2**30:.1f} of {free / 2**30:.1f} free): {r["fp8_ms"]:.3f} ms/step '
                      f'({r["fp8_tok_s"]:.0f} tok/s)', flush=True)
        del model
        torch.cuda.empty_cache()
    with open(os.path.join(a.out, 'generate_bench.json'), 'w') as f:
        json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
