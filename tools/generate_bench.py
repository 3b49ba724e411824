"""Generation from prompts on Llama-2-7B / 70B shapes (synthetic 2-bit packed weights, quip_b200.synth): prefill
tokens/s, decode step time of GraphDecoder (uniform positions, SDPA over the whole static cache, repeat_interleave for
GQA) against PromptDecoder (per-row positions, csrc/attn_decode.cu), and the decode-attention kernel alone against the
HBM bandwidth of the H100 SXM data sheet (3.35 TB/s).  Needs a CUDA device.

    python tools/generate_bench.py --out DIR [--models llama7b,llama70b] [--layers70b 80] [--steps 16]
                                   [--sections kernel,prefill,decode,fp8]      (fp8kernel: the fp8 kernel rows only;
                                                                                sample: the sampling rows;
                                                                                spec: speculative generation)

Section fp8 measures the e4m3 KV cache (PromptDecoder(kv_dtype=torch.float8_e4m3fn)): the fp8 kernel alone next to the
fp16 one (bytes: hd per cached K / V vector plus its 4-byte scale), PromptDecoder steps fp16 against fp8 at B = 32 and
contexts 2048 / 4096 (alternating in one process, one decoder allocated at a time, both caches filled from the same
values; logits compared), and configurations whose fp16 cache does not fit the card, run with fp8 or listed with the
bytes they need.

Section sample times quip_sample (csrc/sample.cu) alone for B in {1, 32, 128} x V in {32000, 50272, 128256} at
T = 0.7, k = 50, p = 0.9 and at k = 0, p = 0.9, next to torch.argmax and the torch warper chain (temperature, top-k, sort,
softmax, cumsum, top-p mask, multinomial) on the same rows, and a 7B PromptDecoder step at B = 32, context 2048, greedy
against sampling, alternated over three trials.

Section spec measures speculative generation: quip_extend_attention(_fp8) alone next to quip_decode_attention(_fp8)
(B in {1, 8}, T in {1, 4, 8}, contexts 2048 / 4096, every row's new slots ending at the context); the captured
SpecDecoder step at T in {2, 4, 5, 6, 8} against the PromptDecoder step on the 7B shape at B in {1, 4}, context 2048
(t_T / t_1 is the break-even number of tokens a step must yield); and generate() end to end, plain against
prompt_lookup_num_tokens=4, on a prompt that repeats itself, with the measured acceptance (synthetic weights: the
acceptance says nothing about real text).

Section chunked measures chunked prefill (PromptDecoder.prefill(chunk=C), csrc/attn_prefill.cu): the prefill-attention
kernel alone in causal TFLOP/s against F.scaled_dot_product_attention(is_causal=True) on the same fp16 q / k / v (B in
{1, 8}, T in {512, 2048} at position 0, fp16 and e4m3 caches), the extend kernel against append + prefill at T = 8; on the
7B shape, tokens/s and peak allocation of the HF-path prefill against chunks of 256 .. 2048 tokens, and an e4m3 cache of
48 x 4096 filled from 4000-token prompts in chunks of 512 followed by decode steps, with the fp16 cache bytes the HF path
would have added.

Section paged measures the paged KV cache (include/quip_b200.h; PromptDecoder(n_pages=...)): the decode kernel, the
extend kernel at T = 5 and the prefill kernel (a 512-token chunk ending at the context) paged against contiguous on the
same bytes, the pool scattered into shuffled pages (B in {1, 8, 32}, contexts 2048 / 4096, 7B and 70B shapes; the two
launches alternate and each is timed three times), and on the 7B shape the generation of 128 tokens from a 2048-token
prompt with 8 samples (num_return_sequences) and from 32 prompts sharing a 1536-token preamble, shared against unshared:
prefill time, cache bytes, decode step time and tokens/s.

Section score (llama7b) measures continuation scoring: quip_token_logprobs alone (logits bytes read per second against
3.35 TB/s, next to torch's log_softmax + gather + argmax) and, on an ARC-like synthetic set (--score-docs documents of 4
choices), the reference harness's recipe against decode.score unshared, shared and shared with an e4m3 cache:
requests/s, prefilled tokens, peak allocation and the largest per-request difference against the recipe.

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


def extend_alone(nh, nkv, hd, B, T, ctx, fp8, reps):
    """quip_extend_attention(_fp8) with every row's T new slots ending at slot ctx - 1, and quip_decode_attention(_fp8)
    at position ctx - 1 on the same cache."""
    from quip_b200 import fused
    g = torch.Generator(device='cuda').manual_seed(0)
    k16 = torch.randn(B, nkv, ctx, hd, generator=g, device='cuda').half()
    v16 = torch.randn(B, nkv, ctx, hd, generator=g, device='cuda').half()
    q = torch.randn(B, T, nh, hd, generator=g, device='cuda').half()
    kn = torch.randn(B, T, nkv, hd, generator=g, device='cuda').half()
    vn = torch.randn(B, T, nkv, hd, generator=g, device='cuda').half()
    sc = {}
    if fp8:
        kc = torch.empty(B, nkv, ctx, hd, dtype=torch.float8_e4m3fn, device='cuda')
        vc = torch.empty_like(kc)
        sc = dict(k_scale=torch.empty(B, nkv, ctx, device='cuda'), v_scale=torch.empty(B, nkv, ctx, device='cuda'))
        fused.kv_quantize(k16, kc, sc['k_scale'])
        fused.kv_quantize(v16, vc, sc['v_scale'])
        del k16, v16
    else:
        kc, vc = k16, v16
    pos = torch.full((B,), ctx - T, dtype=torch.long, device='cuda')
    scale = hd ** -0.5
    ms = events_ms(lambda: fused.extend_attention(q, kn, vn, kc, vc, pos, scale, **sc), reps)
    pos1 = torch.full((B,), ctx - 1, dtype=torch.long, device='cuda')
    q1, kn1, vn1 = q[:, 0].contiguous(), kn[:, 0].contiguous(), vn[:, 0].contiguous()
    ms_dec = events_ms(lambda: fused.decode_attention(q1, kn1, vn1, kc, vc, pos1, scale, **sc), reps)
    nbytes = attn_bytes([ctx - 1] * B, nkv, hd, fp8=fp8)
    del kc, vc
    torch.cuda.empty_cache()
    return dict(kv='fp8' if fp8 else 'fp16', nh=nh, nkv=nkv, hd=hd, B=B, T=T, context=ctx, extend_ms=ms,
                decode_ms=ms_dec, bytes=nbytes, extend_bytes_per_s=nbytes / ms * 1e3, decode_bytes_per_s=nbytes / ms_dec * 1e3)


def spec_steps(model, B, ctx, Ts, steps, trials=3):
    """Per-step ms of a captured PromptDecoder (T = 1) and SpecDecoders of T tokens per row, every row starting at
    position ctx of a cache filled with random values, alternating trial by trial."""
    from quip_b200.decode import PromptDecoder, SpecDecoder
    res = {T: [] for T in (1,) + tuple(Ts)}
    for t in range(trials + 1):
        for T in res:
            max_new = steps * T + 2
            max_len = ctx + max_new + T
            if T == 1:
                dec = PromptDecoder(model, max_len=max_len, batch=B, max_new=max_new)
            else:
                dec = SpecDecoder(model, max_len=max_len, batch=B, max_new=max_new, draft_tokens=T - 1)
                dec.hist.random_(0, model.config.vocab_size)
            dec.k_cache.normal_(0.0, 0.5)
            dec.v_cache.normal_(0.0, 0.5)
            dec.capture()
            with torch.no_grad():
                for r in range(2):
                    dec.positions.fill_(ctx)
                    dec._pos_host = [ctx] * B
                    dec._t.fill_(1)
                    dec._t_host = 1
                    if T > 1:
                        dec.n_gen.fill_(1)
                        dec._steps_host = 0
                    torch.cuda.synchronize()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(steps):
                        dec.step()
                    e1.record()
                    torch.cuda.synchronize()
                    if r and t:
                        res[T].append(e0.elapsed_time(e1) / steps)
            del dec
            torch.cuda.empty_cache()
    med = {T: sorted(v)[len(v) // 2] for T, v in res.items()}
    return dict(B=B, context=ctx, trials_ms={str(k): v for k, v in res.items()}, step_ms={str(k): v for k, v in med.items()},
                break_even_tokens_per_step={str(T): med[T] / med[1] for T in Ts})


def spec_generate(model, B, n_new, k, seg=64, reps=2):
    """generate() wall time (prefill, capture and the host loop included), plain and with prompt_lookup_num_tokens=k,
    on prompts made of a random segment repeated 8 times."""
    import time

    from quip_b200.decode import generate
    g = torch.Generator().manual_seed(3)
    prompts = [torch.randint(0, model.config.vocab_size, (seg,), generator=g).repeat(8) for _ in range(B)]
    out = dict(B=B, prompt=8 * seg, new_tokens=n_new, k=k)
    for name, kw in (('plain', {}), ('spec', dict(prompt_lookup_num_tokens=k))):
        times = []
        for _ in range(reps + 1):
            stats = {}
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            toks = generate(model, prompts, n_new, spec_stats=stats, **kw) if kw else generate(model, prompts, n_new)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        s = sorted(times[1:])[len(times[1:]) // 2]
        out[f'{name}_s'] = s
        out[f'{name}_tok_s'] = sum(int(t.numel()) for t in toks) / s
        if kw:
            out['accepted'] = stats['accepted']
            out['steps'] = stats['steps']
            out['tokens_per_step'] = n_new / (stats['steps'] + 1)
        else:
            plain = toks
    out['same_tokens'] = all(torch.equal(a, b) for a, b in zip(plain, toks))
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


def causal_flops(nh, hd, B, pos, T):
    """Q.K^T and P.V flops of causal attention: sum_i 4 * (pos + i + 1) * hd per query head."""
    return B * nh * 4 * hd * (T * (pos + 1) + T * (T - 1) // 2)


def prefill_kernel_alone(nh, nkv, hd, B, T, fp8, reps):
    """quip_prefill_attention(_fp8) of T tokens per row at position 0 (the cache already appended), in causal TFLOP/s,
    next to F.scaled_dot_product_attention(is_causal=True) on the same fp16 q / k / v (GQA expanded outside the
    timing)."""
    from quip_b200 import fused
    g = torch.Generator(device='cuda').manual_seed(0)
    q = torch.randn(B, T, nh, hd, generator=g, device='cuda').half()
    kn = torch.randn(B, T, nkv, hd, generator=g, device='cuda').half()
    vn = torch.randn(B, T, nkv, hd, generator=g, device='cuda').half()
    pos = torch.zeros(B, dtype=torch.long, device='cuda')
    cnt = torch.full((B,), T, dtype=torch.long, device='cuda')
    if fp8:
        kc = torch.zeros(B, nkv, T, hd, dtype=torch.float8_e4m3fn, device='cuda')
        sc = dict(k_scale=torch.zeros(B, nkv, T, device='cuda'), v_scale=torch.zeros(B, nkv, T, device='cuda'))
    else:
        kc, sc = torch.zeros(B, nkv, T, hd, dtype=torch.float16, device='cuda'), {}
    vc = torch.zeros_like(kc)
    fused.kv_append(kn, vn, kc, vc, pos, cnt, **sc)
    scale = hd ** -0.5
    ms = events_ms(lambda: fused.prefill_attention(q, kc, vc, pos, cnt, scale, **sc), reps)
    got = fused.prefill_attention(q, kc, vc, pos, cnt, scale, **sc)
    qt = q.transpose(1, 2).contiguous()
    kt = kn.transpose(1, 2).repeat_interleave(nh // nkv, dim=1).contiguous()
    vt = vn.transpose(1, 2).repeat_interleave(nh // nkv, dim=1).contiguous()
    sdpa = torch.nn.functional.scaled_dot_product_attention
    ms_sdpa = events_ms(lambda: sdpa(qt, kt, vt, is_causal=True, scale=scale), reps)
    ref = sdpa(qt, kt, vt, is_causal=True, scale=scale).transpose(1, 2)
    fl = causal_flops(nh, hd, B, 0, T)
    del kc, vc, kt, vt
    torch.cuda.empty_cache()
    return dict(kv='fp8' if fp8 else 'fp16', nh=nh, nkv=nkv, hd=hd, B=B, T=T, pos=0, kernel_ms=ms,
                kernel_tflops=fl / ms / 1e9, sdpa_ms=ms_sdpa, sdpa_tflops=fl / ms_sdpa / 1e9, rel_err_vs_sdpa=rel(got, ref))


def extend_vs_prefill(nh, nkv, hd, B, ctx, reps, T=8):
    """A step of T new tokens per row ending at slot ctx - 1: quip_extend_attention (append included) against
    quip_kv_append + quip_prefill_attention on the same fp16 cache."""
    from quip_b200 import fused
    g = torch.Generator(device='cuda').manual_seed(0)
    kc = torch.randn(B, nkv, ctx, hd, generator=g, device='cuda').half()
    vc = torch.randn(B, nkv, ctx, hd, generator=g, device='cuda').half()
    q = torch.randn(B, T, nh, hd, generator=g, device='cuda').half()
    kn = torch.randn(B, T, nkv, hd, generator=g, device='cuda').half()
    vn = torch.randn(B, T, nkv, hd, generator=g, device='cuda').half()
    pos = torch.full((B,), ctx - T, dtype=torch.long, device='cuda')
    cnt = torch.full((B,), T, dtype=torch.long, device='cuda')
    scale = hd ** -0.5
    ms_ext = events_ms(lambda: fused.extend_attention(q, kn, vn, kc, vc, pos, scale), reps)

    def pair():
        fused.kv_append(kn, vn, kc, vc, pos, cnt)
        return fused.prefill_attention(q, kc, vc, pos, cnt, scale)
    ms_pf = events_ms(pair, reps)
    err = rel(pair(), fused.extend_attention(q, kn, vn, kc, vc, pos, scale))
    del kc, vc
    torch.cuda.empty_cache()
    return dict(nh=nh, nkv=nkv, hd=hd, B=B, T=T, context=ctx, extend_ms=ms_ext, append_prefill_ms=ms_pf,
                rel_err=err)


def _peak(fn):
    """(ms, peak bytes allocated above the start) of one call of fn."""
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1), torch.cuda.max_memory_allocated() - base


def chunked_prefill_rates(model, B, P, chunks, reps=2):
    """Tokens/s and peak allocation above the static cache of the HF-path prefill and of chunked prefills (fp16 cache);
    each timed call follows one warm-up call of the same kind."""
    from quip_b200.decode import PromptDecoder
    g = torch.Generator().manual_seed(3)
    prompts = [torch.randint(0, model.config.vocab_size, (P,), generator=g) for _ in range(B)]
    dec = PromptDecoder(model, max_len=P, batch=B)
    rows = []
    with torch.no_grad():
        for C in (None,) + tuple(c for c in chunks if c <= P):
            dec.prefill(prompts, chunk=C)
            res = [_peak(lambda: dec.prefill(prompts, chunk=C)) for _ in range(reps)]
            ms = sorted(r[0] for r in res)[len(res) // 2]
            rows.append(dict(B=B, P=P, chunk=C, ms=ms, tokens_per_s=B * P * 1e3 / ms, peak_bytes=max(r[1] for r in res)))
    del dec
    torch.cuda.empty_cache()
    return rows


def chunked_capacity(model, cfg, B, P, max_len, C, steps):
    """The configuration the HF path cannot run: an e4m3 cache of B x max_len, prompts of P tokens prefilled in chunks
    of C, then `steps` captured decode steps; with the bytes the HF path would have needed on top of the static cache."""
    from quip_b200.decode import PromptDecoder
    g = torch.Generator().manual_seed(4)
    prompts = [torch.randint(0, cfg.vocab_size, (P,), generator=g) for _ in range(B)]
    L = cfg.num_hidden_layers
    hf_cache = cache_bytes(cfg, L, B, P)                              # the HF DynamicCache of the padded prompts (fp16)
    free = torch.cuda.mem_get_info()[0]
    dec = PromptDecoder(model, max_len=max_len, batch=B, max_new=steps + 1, kv_dtype=torch.float8_e4m3fn).capture()
    static = cache_bytes(cfg, L, B, max_len, fp8=True)
    with torch.no_grad():
        ms_prefill, peak = _peak(lambda: dec.prefill(prompts, chunk=C))
        torch.cuda.synchronize()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(steps):
            dec.step()
        e1.record()
        torch.cuda.synchronize()
    out = dict(kv='fp8', B=B, P=P, max_len=max_len, chunk=C, prefill_ms=ms_prefill, prefill_tokens_per_s=B * P * 1e3 / ms_prefill,
               prefill_peak_bytes_above_cache=peak, decode_steps=steps, decode_ms_per_step=e0.elapsed_time(e1) / steps,
               static_cache_bytes=static, hf_path_fp16_cache_bytes=hf_cache, free_bytes_before=free,
               positions=sorted(set(dec.positions.tolist())), tokens_finite=bool(torch.isfinite(dec.logits.float()).all()))
    del dec
    torch.cuda.empty_cache()
    return out


def _scatter_pages(x, table):
    """Pool (n_pages, nkv, 64, ...) holding slot j of row b of x (B, nkv, ctx, ...) at slot j % 64 of page
    table[b, j // 64]."""
    B, nkv, ctx = x.shape[:3]
    pool = torch.empty((int(table.max()) + 1, nkv, 64) + tuple(x.shape[3:]), dtype=x.dtype, device=x.device)
    pool[table.long().reshape(-1)] = x.view(B, nkv, ctx // 64, 64, *x.shape[3:]).transpose(1, 2).reshape(
        B * (ctx // 64), nkv, 64, *x.shape[3:])
    return pool


def paged_kernels(nh, nkv, hd, B, ctx, reps):
    """Decode, extend (T = 5) and prefill (T = 512) kernels at every row's context ctx: contiguous against paged over the
    same bytes on shuffled pages.  Returns the median of three alternating timings of each and whether the outputs are
    bit-identical."""
    from quip_b200 import fused
    g = torch.Generator(device='cuda').manual_seed(0)
    kc = torch.randn(B, nkv, ctx, hd, generator=g, device='cuda').half()
    vc = torch.randn(B, nkv, ctx, hd, generator=g, device='cuda').half()
    table = torch.randperm(B * (ctx // 64), generator=torch.Generator().manual_seed(1)).to(torch.int32)
    table = table.view(B, ctx // 64).cuda()
    kp, vp = _scatter_pages(kc, table), _scatter_pages(vc, table)
    scale = hd ** -0.5
    out = dict(nh=nh, nkv=nkv, hd=hd, B=B, context=ctx)
    T5, T512 = 5, 512
    q1 = torch.randn(B, nh, hd, generator=g, device='cuda').half()
    kn1, vn1 = kc[:, :, -1].clone(), vc[:, :, -1].clone()
    q5 = torch.randn(B, T5, nh, hd, generator=g, device='cuda').half()
    kn5, vn5 = kc[:, :, -T5:].transpose(1, 2).contiguous(), vc[:, :, -T5:].transpose(1, 2).contiguous()
    qp = torch.randn(B, T512, nh, hd, generator=g, device='cuda').half()
    pos1 = torch.full((B,), ctx - 1, dtype=torch.long, device='cuda')
    pos5 = torch.full((B,), ctx - T5, dtype=torch.long, device='cuda')
    posp = torch.full((B,), ctx - T512, dtype=torch.long, device='cuda')
    cnt = torch.full((B,), T512, dtype=torch.long, device='cuda')
    kinds = dict(
        decode=(lambda k, v, **kw: fused.decode_attention(q1, kn1, vn1, k, v, pos1, scale, **kw), reps),
        extend=(lambda k, v, **kw: fused.extend_attention(q5, kn5, vn5, k, v, pos5, scale, **kw), reps),
        prefill=(lambda k, v, **kw: fused.prefill_attention(qp, k, v, posp, cnt, scale, **kw), max(reps // 10, 10)))
    for name, (fn, n) in kinds.items():
        ms = {'contiguous': [], 'paged': []}
        for _ in range(3):
            ms['contiguous'].append(events_ms(lambda: fn(kc, vc), n))
            ms['paged'].append(events_ms(lambda: fn(kp, vp, page_table=table), n))
        a, b = (sorted(v)[1] for v in ms.values())
        same = torch.equal(fn(kc, vc).view(torch.int16), fn(kp, vp, page_table=table).view(torch.int16))
        out[name] = dict(contiguous_ms=a, paged_ms=b, paged_over_contiguous=b / a, bit_identical=same)
    del kc, vc, kp, vp
    torch.cuda.empty_cache()
    return out


def paged_generate(model, prompts, n_new, share, chunk=512, sample=False):
    """What generate() does (capture, chunked prefill, captured steps), timed: prefill ms, decode ms per step, cache
    bytes and tokens/s, unshared (contiguous cache) or with shared prefix pages (plan_prefix_pages).  Returns the
    stats and the generated tokens."""
    from quip_b200.decode import KV_PAGE, PromptDecoder, plan_prefix_pages
    B = len(prompts)
    max_len = max(len(p) for p in prompts) + n_new
    pages, starts = {}, None
    if share:
        table, n_pages, starts = plan_prefix_pages(prompts, [len(p) + n_new for p in prompts],
                                                   max_pages=-(-max_len // KV_PAGE))
        pages = dict(page_table=table, n_pages=n_pages)
    torch.cuda.synchronize()
    dec = PromptDecoder(model, max_len=max_len, batch=B, max_new=n_new, sampling=sample, **pages)
    if sample:
        dec.set_sampling(temperature=0.8, seed=list(range(B)))
    dec.capture()
    cache = dec.k_cache.numel() * dec.k_cache.element_size() * 2
    with torch.no_grad():
        prefill_ms, _ = _peak(lambda: dec.prefill(prompts, chunk=chunk, starts=starts))
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(n_new - 1):
            dec.step()
        e1.record()
        torch.cuda.synchronize()
    step_ms = e0.elapsed_time(e1) / (n_new - 1)
    fed = sum(len(p) - s for p, s in zip(prompts, starts or [0] * B))
    r = dict(B=B, shared=share, prefill_ms=prefill_ms, prefilled_tokens=fed, cache_bytes=cache, decode_ms_per_step=step_ms,
             tokens_per_s=B * n_new * 1e3 / (prefill_ms + step_ms * (n_new - 1)),
             n_pages=pages.get('n_pages'), max_pages=-(-max_len // KV_PAGE))
    gen = dec.generated.cpu()
    del dec
    torch.cuda.empty_cache()
    return r, gen


def score_kernel_alone(R, V, reps):
    """quip_token_logprobs on fp16 logits (R, V): logits bytes read per second against 3.35 TB/s, next to torch's
    log_softmax(x.float()).gather plus argmax on the same tensor."""
    from quip_b200 import fused
    g = torch.Generator(device='cuda').manual_seed(R + V)
    x = torch.randn(R, V, generator=g, device='cuda').half()
    t = torch.randint(0, V, (R,), generator=g, device='cuda')
    lp = torch.empty(R, device='cuda')
    gr = torch.empty(R, dtype=torch.uint8, device='cuda')
    ms = events_ms(lambda: fused.token_logprobs(x, t, lp, gr), reps)

    def torch_way():
        y = torch.log_softmax(x.float(), -1).gather(-1, t[:, None])[:, 0]
        return y, x.argmax(-1) == t
    tms = events_ms(torch_way, max(reps // 4, 5))
    y, tg = torch_way()
    nbytes = R * V * 2
    return dict(R=R, V=V, kernel_ms=ms, bytes_per_s=nbytes / ms * 1e3, share_of_3_35_TBps=nbytes / ms * 1e3 / HBM_BPS,
                torch_ms=tms, max_abs_diff=float((lp - y).abs().max()), greedy_equal=bool(torch.equal(gr.bool(), tg)))


def score_workload(V, docs, seed=0):
    """ARC-like synthetic requests: docs documents of 4 choices, a context of 64-512 random tokens shared within a
    document, continuations of 1-16 tokens."""
    g = torch.Generator().manual_seed(seed)
    ctxs, conts = [], []
    for _ in range(docs):
        ctx = torch.randint(0, V, (int(torch.randint(64, 513, (1,), generator=g)),), generator=g).tolist()
        for _ in range(4):
            ctxs.append(ctx)
            conts.append(torch.randint(0, V, (int(torch.randint(1, 17, (1,), generator=g)),), generator=g).tolist())
    return ctxs, conts


def score_reference_recipe(model, ctxs, conts, batch_size, max_length):
    """The reference harness's recipe on the packed model: each batch right-padded to its longest request through
    model(ids), fp32 log_softmax of the whole (B, S, V) logits, gather, argmax."""
    from quip_b200.decode import score_windows
    reqs = score_windows(ctxs, conts, max_length)
    res, tokens = [None] * len(ctxs), 0
    for s in range(0, len(reqs), batch_size):
        part = reqs[s:s + batch_size]
        P = len(part[0][0])
        tokens += P * len(part)
        ids = torch.zeros(len(part), P, dtype=torch.long)
        for b, (inp, _, _) in enumerate(part):
            ids[b, :len(inp)] = torch.tensor(inp)
        with torch.no_grad():
            lsm = torch.log_softmax(model(ids.cuda()).logits.float(), -1)
        for b, (inp, cont, idx) in enumerate(part):
            n = len(cont)
            x = lsm[b, len(inp) - n:len(inp)]
            c = torch.tensor(cont, device='cuda')
            ans = (float(x.gather(-1, c[:, None]).double().sum()), bool((x.argmax(-1) == c).all()))
            for i in idx:
                res[i] = ans
        del lsm
    return res, tokens


def score_arms(model, docs, batch_size, chunk):
    """requests/s, prefilled tokens, peak allocation and the largest per-request difference against the reference recipe
    for (a) the recipe, (b) score unshared, (c) score shared, (d) score shared with an e4m3 cache."""
    import time

    from quip_b200.decode import plan_prefix_pages, score, score_windows
    V, L = model.config.vocab_size, 2048
    ctxs, conts = score_workload(V, docs)
    reqs = score_windows(ctxs, conts, L)

    def prefilled(share):
        n = 0
        for s in range(0, len(reqs), batch_size):
            part = reqs[s:s + batch_size]
            if not share:
                n += sum(len(r[0]) for r in part)
                continue
            heads = [torch.tensor(r[0][:len(r[0]) - len(r[1]) + 1]) for r in part]
            starts = plan_prefix_pages(heads, [len(r[0]) for r in part])[2]
            n += sum(len(r[0]) - st for r, st in zip(part, starts))
        return n

    arms = dict(recipe=lambda: score_reference_recipe(model, ctxs, conts, batch_size, L),
                unshared=lambda: (score(model, ctxs, conts, batch_size=batch_size, max_length=L, prefill_chunk_size=chunk,
                                        share_prompt_prefixes=False), prefilled(False)),
                shared=lambda: (score(model, ctxs, conts, batch_size=batch_size, max_length=L, prefill_chunk_size=chunk),
                                prefilled(True)),
                shared_e4m3=lambda: (score(model, ctxs, conts, batch_size=batch_size, max_length=L,
                                           prefill_chunk_size=chunk, kv_dtype=torch.float8_e4m3fn), prefilled(True)))
    out, base = {}, None
    for name, fn in arms.items():
        fn()                                                         # warm-up: lazy set-up, workspaces
        torch.cuda.synchronize()
        torch.cuda.reset_peak_memory_stats()
        m0 = torch.cuda.memory_allocated()
        t0 = time.perf_counter()
        res, tokens = fn()
        torch.cuda.synchronize()
        dt = time.perf_counter() - t0
        base = res if base is None else base
        out[name] = dict(seconds=dt, requests_per_s=len(ctxs) / dt, prefilled_tokens=tokens,
                         peak_bytes_above_model=torch.cuda.max_memory_allocated() - m0,
                         max_abs_diff_vs_recipe=max(abs(a[0] - b[0]) for a, b in zip(res, base)),
                         is_greedy_agreement=sum(a[1] == b[1] for a, b in zip(res, base)) / len(res))
    out.update(docs=docs, requests=len(ctxs), batch_size=batch_size, chunk=chunk)
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--models', default='llama7b,llama70b')
    ap.add_argument('--layers70b', type=int, default=80, help='decoder layers of the 70B shape to build (of 80)')
    ap.add_argument('--steps', type=int, default=16)
    ap.add_argument('--kernel-reps', type=int, default=100)
    ap.add_argument('--sections', default='kernel,prefill,decode,fp8')    # also: fp8kernel, sample, spec, chunked, paged,
    #                                                                         score
    ap.add_argument('--score-docs', type=int, default=512, help='documents of 4 choices in the score section')
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
        if 'spec' in sections:
            rec['extend_kernel'] = []
            for B in (1, 8):
                for T in (1, 4, 8):
                    for ctx in (2048, 4096):
                        for fp8 in (False, True):
                            r = extend_alone(nh, nkv, hd, B, T, ctx, fp8, a.kernel_reps)
                            rec['extend_kernel'].append(r)
                            print(f'{name} extend kernel {r["kv"]} B={B} T={T} ctx={ctx}: {1e3 * r["extend_ms"]:.1f} us '
                                  f'({r["extend_bytes_per_s"] / 1e12:.2f} TB/s), decode kernel {1e3 * r["decode_ms"]:.1f} us '
                                  f'({r["decode_bytes_per_s"] / 1e12:.2f} TB/s)', flush=True)
        if 'chunked' in sections:
            rec['prefill_kernel'], rec['extend_vs_prefill'] = [], []
            for fp8 in (False, True):
                for B in (1, 8):
                    for T in (512, 2048):
                        r = prefill_kernel_alone(nh, nkv, hd, B, T, fp8, max(a.kernel_reps // 10, 10))
                        rec['prefill_kernel'].append(r)
                        print(f'{name} prefill kernel {r["kv"]} B={B} T={T}: {r["kernel_ms"]:.3f} ms '
                              f'({r["kernel_tflops"]:.0f} TFLOP/s), SDPA causal {r["sdpa_ms"]:.3f} ms '
                              f'({r["sdpa_tflops"]:.0f} TFLOP/s), rel err {r["rel_err_vs_sdpa"]:.1e}', flush=True)
            for B in (1, 8):
                r = extend_vs_prefill(nh, nkv, hd, B, 2048, a.kernel_reps)
                rec['extend_vs_prefill'].append(r)
                print(f'{name} T=8 B={B} ctx=2048: extend {1e3 * r["extend_ms"]:.1f} us, append + prefill '
                      f'{1e3 * r["append_prefill_ms"]:.1f} us, rel err {r["rel_err"]:.1e}', flush=True)
        if 'paged' in sections:
            rec['paged_kernel'] = []
            for B in (1, 8, 32):
                for ctx in (2048, 4096):
                    r = paged_kernels(nh, nkv, hd, B, ctx, a.kernel_reps)
                    rec['paged_kernel'].append(r)
                    print(f'{name} paged kernels B={B} ctx={ctx}: ' + ', '.join(
                        f'{k} {1e3 * r[k]["contiguous_ms"]:.1f} -> {1e3 * r[k]["paged_ms"]:.1f} us '
                        f'({r[k]["paged_over_contiguous"]:.3f}x, same bits {r[k]["bit_identical"]})'
                        for k in ('decode', 'extend', 'prefill')), flush=True)
        if 'score' in sections and name == 'llama7b':
            rec['score_kernel'] = []
            for R in (64, 1024, 8192):
                for V in (32000, 50272, 128256):
                    r = score_kernel_alone(R, V, a.kernel_reps)
                    rec['score_kernel'].append(r)
                    print(f'score kernel R={R} V={V}: {1e3 * r["kernel_ms"]:.1f} us, {r["bytes_per_s"] / 1e12:.2f} TB/s '
                          f'({100 * r["share_of_3_35_TBps"]:.0f}% of 3.35), torch log_softmax+gather+argmax '
                          f'{1e3 * r["torch_ms"]:.1f} us, max diff {r["max_abs_diff"]:.1e}, greedy equal '
                          f'{r["greedy_equal"]}', flush=True)
                    torch.cuda.empty_cache()
        if not sections & {'prefill', 'decode', 'fp8', 'sample', 'spec'} and not (
                sections & {'chunked', 'paged', 'score'} and name == 'llama7b'):
            continue
        model = build_synthetic_model(cfg, torch.device('cuda:0'), bits=2, seed=0, seqlen=4096)
        if 'score' in sections and name == 'llama7b':
            r = score_arms(model, a.score_docs, 32, 512)
            rec['score'] = r
            for arm in ('recipe', 'unshared', 'shared', 'shared_e4m3'):
                x = r[arm]
                print(f'{name} score {arm}: {x["requests_per_s"]:.1f} requests/s, {x["prefilled_tokens"]} prefilled '
                      f'tokens, peak {x["peak_bytes_above_model"] / 2**30:.2f} GiB, max |diff| vs recipe '
                      f'{x["max_abs_diff_vs_recipe"]:.2e}, is_greedy agreement {x["is_greedy_agreement"]:.3f}', flush=True)
        if 'chunked' in sections and name == 'llama7b':
            rec['chunked_prefill'] = []
            for B, P in ((1, 2048), (8, 512), (8, 2048)):
                for r in chunked_prefill_rates(model, B, P, (256, 512, 1024, 2048)):
                    rec['chunked_prefill'].append(r)
                    print(f'{name} prefill {B}x{P} chunk={r["chunk"]}: {r["ms"]:.1f} ms, {r["tokens_per_s"]:.0f} '
                          f'tokens/s, peak {r["peak_bytes"] / 2**30:.2f} GiB above the cache', flush=True)
            r = chunked_capacity(model, cfg, 48, 4000, 4096, 512, a.steps)
            rec['chunked_capacity'] = r
            print(f'{name} e4m3 B=48 P=4000 chunk=512: prefill {r["prefill_ms"] / 1e3:.1f} s '
                  f'({r["prefill_tokens_per_s"]:.0f} tokens/s, peak {r["prefill_peak_bytes_above_cache"] / 2**30:.2f} GiB '
                  f'above the {r["static_cache_bytes"] / 2**30:.1f} GiB cache), {r["decode_ms_per_step"]:.2f} ms/step; the '
                  f'HF path would add {r["hf_path_fp16_cache_bytes"] / 2**30:.1f} GiB of fp16 cache', flush=True)
        if 'paged' in sections and name == 'llama7b':
            g = torch.Generator().manual_seed(5)
            V = cfg.vocab_size
            one = torch.randint(0, V, (2048,), generator=g)
            pre = torch.randint(0, V, (1536,), generator=g)
            cases = dict(n8=([one] * 8, True),
                         preamble32=([torch.cat((pre, torch.randint(0, V, (256,), generator=g))) for _ in range(32)],
                                     False))
            rec['paged_generate'] = {}
            for case, (prompts, sample) in cases.items():
                runs = {}
                for share in (False, True):
                    runs[share] = paged_generate(model, prompts, 128, share, sample=sample)
                same = float((runs[False][1] == runs[True][1]).float().mean())
                rec['paged_generate'][case] = dict(unshared=runs[False][0], shared=runs[True][0],
                                                   same_token_share=same)
                u, s_ = runs[False][0], runs[True][0]
                print(f'{name} generate {case}: prefill {u["prefill_ms"]:.0f} -> {s_["prefill_ms"]:.0f} ms '
                      f'({u["prefilled_tokens"]} -> {s_["prefilled_tokens"]} tokens), cache {u["cache_bytes"] / 2**30:.2f} '
                      f'-> {s_["cache_bytes"] / 2**30:.2f} GiB, step {u["decode_ms_per_step"]:.2f} -> '
                      f'{s_["decode_ms_per_step"]:.2f} ms, {u["tokens_per_s"]:.0f} -> {s_["tokens_per_s"]:.0f} tok/s, '
                      f'same tokens {same:.3f}', flush=True)
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
        if 'spec' in sections and name == 'llama7b':
            rec['spec_steps'] = []
            for B in (1, 4):
                r = spec_steps(model, B, 2048, (2, 4, 5, 6, 8), a.steps)
                rec['spec_steps'].append(r)
                print(f'{name} step cost B={B} ctx=2048: ' + ', '.join(f'T={T} {ms:.3f} ms' for T, ms in r['step_ms'].items()),
                      flush=True)
            rec['spec_generate'] = []
            for B in (1, 4):
                r = spec_generate(model, B, 128, 4)
                rec['spec_generate'].append(r)
                print(f'{name} generate B={B} 128 tokens: plain {r["plain_tok_s"]:.0f} tok/s, k=4 {r["spec_tok_s"]:.0f} '
                      f'tok/s, {r["tokens_per_step"]:.2f} tokens per step, same tokens {r["same_tokens"]}', flush=True)
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
