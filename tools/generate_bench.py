"""Generation from prompts on Llama-2-7B / 70B shapes (synthetic 2-bit packed weights, quip_b200.synth): prefill
tokens/s, decode step time of GraphDecoder (uniform positions, SDPA over the whole static cache, repeat_interleave for
GQA) against PromptDecoder (per-row positions, csrc/attn_decode.cu), and the decode-attention kernel alone against the
HBM bandwidth of the H100 SXM data sheet (3.35 TB/s).  Needs a CUDA device.

    python tools/generate_bench.py --out DIR [--models llama7b,llama70b] [--layers70b 80] [--steps 16]
                                   [--sections kernel,prefill,decode,fp8]      (fp8kernel: the fp8 kernel rows only;
                                                                                sample: the sampling rows;
                                                                                spec: speculative generation;
                                                                                assisted: assisted generation)

Section fp8 measures the e4m3 KV cache (PromptDecoder(kv_dtype=torch.float8_e4m3fn)): the fp8 kernel alone next to the
fp16 one (bytes: hd per cached K / V vector plus its 4-byte scale), PromptDecoder steps fp16 against fp8 at B = 32 and
contexts 2048 / 4096 (alternating in one process, one decoder allocated at a time, both caches filled from the same
values; logits compared), and configurations whose fp16 cache does not fit the card, run with fp8 or listed with the
bytes they need.

Section sample times quip_sample (csrc/sample.cu) alone for B in {1, 32, 128} x V in {32000, 50272, 128256} at
T = 0.7, k = 50, p = 0.9 and at k = 0, p = 0.9, next to torch.argmax and the torch warper chain (temperature, top-k, sort,
softmax, cumsum, top-p mask, multinomial) on the same rows, and a 7B PromptDecoder step at B = 32, context 2048, greedy
against sampling, alternated over three trials.

Section spec measures speculative generation: quip_extend_attention alone next to quip_decode_attention (fp16 and e4m3)
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

Section continuous (llama7b) measures continuous batching (generate(..., max_batch_size=32), ContinuousDecoder): 256
requests with prompt lengths uniform in [32, 1536] and budgets uniform in [16, 512] from a fixed seed, fp16 cache, greedy,
no EOS.  The static arm runs consecutive groups of 32 through generate() (prefill_chunk_size=512, per-prompt budgets);
the continuous arm runs generate()'s continuous loop (32 rows, chunks of 512 prompt tokens), instrumented with CUDA
events per step.  Reported: output tokens/s end to end, the GEMM tokens each arm's prefill feeds (padded rows included,
counted from shapes), mean and p99 time between a request's tokens, the time in graph steps and in mixed steps, the host
time per mixed step, and how many requests' tokens agree exactly.  Also ragged against padded chunked prefill alone on
8 prompts of 64 .. 2048 tokens.

Section prefix (llama7b) measures the prefix cache of continuous batching (generate(..., max_batch_size=32,
prefix_cache=True)): 256 requests, each one of 8 shared 1024-token preambles plus a unique tail of 32 .. 512 tokens,
budgets 16 .. 256 (fixed seed), fp16 cache, greedy, no EOS, and a variant of 32 such prompts each repeated 8 times.  The
cache-off and cache-on arms run the instrumented continuous loop of section continuous (32 rows, chunks of 512) one after
the other in the same process.  Reported per arm: output tokens/s and wall time, the prompt tokens the schedule fed,
the time in mixed and in graph steps, mean and p99 time between a request's tokens; and how many requests' tokens agree
exactly between the arms.

Section logits (llama7b) measures the logits processors (quip_logits_process, csrc/logits_process.cu): the kernel alone
at B in {1, 32, 128}, V in {32000, 128256} and histories of 512 and 4096 tokens with every processor on (n-gram size 3,
16 bad words), and the captured PromptDecoder step with and without processors at B in {1, 32}, 512-token prompts and
128 new tokens, alternated over three trials.

Section logprobs (llama7b) measures the log-probabilities of generation (quip_token_topk_logprobs,
csrc/topk_logprobs.cu): the kernel alone on R in {1, 8, 32, 256} rows of V = 32000 fp16 logits with n in {0, 5, 20}
(time, and one pass over the logits per second), and the captured PromptDecoder step at B in {1, 8, 32} (256-token
prompts, 64 new tokens, greedy) with logprobs off, n = 0 and n = 20, with the logits processors off and on, the three
decoders alternating over three trials.

Section assisted measures assisted generation (AssistedDecoder, generate(..., assistant_model=...)) at B in {1, 8},
k in {2, 4, 7}, every row at position 512 of random caches: the assistant's captured T = 1 and T = 2 steps alone, the
captured round, the target's captured PromptDecoder step, and the break-even yield round / plain step (the tokens a
round must yield to win).  The 7B-shape target runs with 2-bit synthetic assistants of the 7B shape cut to 2, 4 and 8
layers, the 70B shape (--layers70b) with the whole 32-layer 7B shape.  On the 7B shape the target is also its own
assistant, which accepts every draft away from ties: the round's cost at full acceptance, as a captured round and as
generate() end to end (128 tokens, k = 4, wall time with prefill and capture) against plain generate().  Acceptance on synthetic weights says nothing about real text.  The rows and their cache sizes are printed
from shapes before any device work.

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
    """quip_decode_attention on an e4m3 cache at every row's position ctx-1 of an e4m3 cache of ctx slots; rel err against the fp16
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
    """quip_extend_attention with every row's T new slots ending at slot ctx - 1, and quip_decode_attention
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


ASSIST_B, ASSIST_K, ASSIST_CTX = (1, 8), (2, 4, 7), 512


def assisted_plan(layers70b):
    """The rows of the assisted section from shapes alone: (target, its config, {assistant layers: config})."""
    from quip_b200.synth import model_config
    t7, t70 = model_config('llama7b'), model_config('llama70b', num_hidden_layers=layers70b)
    return [('llama7b', t7, {L: model_config('llama7b', num_hidden_layers=L) for L in (2, 4, 8)}),
            ('llama70b', t70, {32: model_config('llama7b')})]


def _graph_ms(fn, reps):
    """ms per replay of fn captured alone in a CUDA graph (two eager warm-up calls first)."""
    side = torch.cuda.Stream()
    side.wait_stream(torch.cuda.current_stream())
    with torch.no_grad(), torch.cuda.stream(side):
        for _ in range(2):
            fn()
        g = torch.cuda.CUDAGraph()
        with torch.cuda.graph(g, stream=side, capture_error_mode='thread_local'):
            fn()
    torch.cuda.current_stream().wait_stream(side)
    return events_ms(g.replay, reps)


def _timed_steps(dec, ctx, steps, assisted):
    """ms per captured step of dec, every row starting at position ctx (assisted: a round, n_gen = 1)."""
    B = dec.batch
    dec.positions.fill_(ctx)
    dec._pos_host = [ctx] * B
    dec._t.fill_(1)
    dec._t_host = 1
    if assisted:
        dec.n_gen.fill_(1)
        dec._steps_host = 0
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    with torch.no_grad():
        for _ in range(steps):
            dec.step()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / steps


def assisted_rows(model, assistant, B, ks, ctx, steps, reps, trials=3):
    """The assistant's captured T = 1 and T = 2 steps alone, the captured AssistedDecoder round for each k and the
    captured PromptDecoder step of the target, every row at position ctx of caches filled with random values; the
    round and the plain step alternate trial by trial.  break_even_yield[k] = round / plain: the tokens a round must
    yield to beat plain decoding."""
    from quip_b200.decode import AssistedDecoder, PromptDecoder
    max_new = steps * (max(ks) + 1) + 2
    max_len = ctx + max_new + max(ks) + 1

    def filled(dec):
        for d in (dec, getattr(dec, 'assistant', None)):
            if d is not None:
                d.k_cache.normal_(0.0, 0.5)
                d.v_cache.normal_(0.0, 0.5)
        return dec
    plain = filled(PromptDecoder(model, max_len=max_len, batch=B, max_new=max_new)).capture()
    decs = {}
    for k in ks:
        d = filled(AssistedDecoder(model, assistant, max_len=max_len, batch=B, max_new=max_new, draft_tokens=k))
        d.hist.random_(0, model.config.vocab_size)
        decs[k] = d.capture()
    d, a = decs[ks[0]], decs[ks[0]].assistant
    pair, one = d.hist[:, ctx - 1:ctx + 1].clone(), d.hist[:, ctx].clone()
    a.positions.fill_(ctx - 1)
    t2 = _graph_ms(lambda: d._assist(pair), reps)
    a.positions.fill_(ctx)
    t1 = _graph_ms(lambda: d._assist(one), reps)
    res = {'plain': []} | {k: [] for k in ks}
    for t in range(trials + 1):
        for key in res:
            ms = _timed_steps(plain if key == 'plain' else decs[key], ctx, steps, key != 'plain')
            if t:
                res[key].append(ms)
    med = {key: sorted(v)[len(v) // 2] for key, v in res.items()}
    del plain, decs, d, a
    torch.cuda.empty_cache()
    return dict(B=B, context=ctx, assistant_layers=assistant.config.num_hidden_layers, assistant_t1_ms=t1,
                assistant_t2_ms=t2, plain_step_ms=med['plain'], round_ms={str(k): med[k] for k in ks},
                break_even_yield={str(k): med[k] / med['plain'] for k in ks},
                trials_ms={str(k): v for k, v in res.items()})


def assisted_generate_self(model, B, n_new, k, P=128, reps=2):
    """generate() wall time (prefill, capture and the host loop included), plain and with the target as its own
    assistant: away from ties every draft is accepted, so this is the round's cost at full acceptance."""
    import time

    from quip_b200.decode import generate
    g = torch.Generator().manual_seed(4)
    prompts = [torch.randint(0, model.config.vocab_size, (P,), generator=g) for _ in range(B)]
    out = dict(B=B, prompt=P, new_tokens=n_new, k=k)
    toks = {}
    for name, kw in (('plain', {}), ('assisted', dict(assistant_model=model, num_assistant_tokens=k))):
        times = []
        for _ in range(reps + 1):
            stats = {}
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            toks[name] = generate(model, prompts, n_new, spec_stats=stats, **kw) if kw else generate(model, prompts, n_new)
            torch.cuda.synchronize()
            times.append(time.perf_counter() - t0)
        s = sorted(times[1:])[len(times[1:]) // 2]
        out[f'{name}_s'] = s
        out[f'{name}_tok_s'] = sum(int(t.numel()) for t in toks[name]) / s
        if kw:
            out['accepted'] = stats['accepted']
            out['replays'] = stats['steps']
            # a row's n_new - 1 tokens after the prefill's took n_new - 1 - accepted rounds (the replays past the
            # last row's last round, until the every-16-steps check, yield nothing)
            out['tokens_per_round'] = [(n_new - 1) / (n_new - 1 - acc) for acc in stats['accepted']]
    out['same_tokens'] = all(torch.equal(a, b) for a, b in zip(toks['plain'], toks['assisted']))
    out['agreeing_prefix'] = [int((a != b).nonzero()[0]) if not torch.equal(a, b) else a.numel()
                              for a, b in zip(toks['plain'], toks['assisted'])]
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
    """quip_prefill_attention of T tokens per row at position 0 (the cache already appended), in causal TFLOP/s,
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


def continuous_workload(V, n=256, seed=0):
    g = torch.Generator().manual_seed(seed)
    lens = torch.randint(32, 1537, (n,), generator=g).tolist()
    budgets = torch.randint(16, 513, (n,), generator=g).tolist()
    return [torch.randint(0, V, (k,), generator=g) for k in lens], budgets


def continuous_static(model, prompts, budgets, rows, chunk):
    """Consecutive groups of `rows` prompts through generate(): seconds, outputs and the GEMM tokens of the chunked
    prefill (each chunk runs rows x its width)."""
    import time
    from quip_b200.decode import generate
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    outs, gemm = [], 0
    for s in range(0, len(prompts), rows):
        ps = prompts[s:s + rows]
        outs += generate(model, ps, budgets[s:s + rows], prefill_chunk_size=chunk)
        P = max(p.numel() for p in ps)
        gemm += sum(len(ps) * min(chunk, P - c0) for c0 in range(0, P, chunk))
    torch.cuda.synchronize()
    return time.perf_counter() - t0, outs, gemm


def continuous_serve(model, prompts, budgets, rows, chunk, prefix_cache=False, stats=None):
    """generate()'s continuous loop (decode._generate_continuous), with a CUDA event after every step: seconds, outputs,
    per-step (kind, device ms, host ms, prompt tokens, decode tokens) and each request's token times.  prefix_cache:
    the schedule shares prompt pages (generate(..., prefix_cache=True)); stats: a dict that receives the schedule's
    prefilled prompt tokens and shared pages per request."""
    import time
    from quip_b200.decode import EOS_CHECK_EVERY, KV_PAGE, ContinuousDecoder, ContinuousSchedule
    lens = [p.numel() for p in prompts]
    need = max(-(-(n + m) // KV_PAGE) for n, m in zip(lens, budgets))
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    sched = ContinuousSchedule(lens, budgets, rows, rows * need, chunk, prompts=prompts if prefix_cache else None)
    dec = ContinuousDecoder(model, max(n + m for n, m in zip(lens, budgets)), rows, rows * need, max(budgets))
    dec.capture()
    out = [None] * len(prompts)
    steps, log = 0, []
    start = torch.cuda.Event(enable_timing=True)
    start.record()
    with torch.no_grad():
        while True:
            if sched.queue or steps % EOS_CHECK_EVERY == 0:
                done = dec.done.cpu()
                for r, i in enumerate(sched.req):
                    if i is not None and done[r]:
                        out[sched.retire(r)] = dec.generated[r, :int(dec.n_gen[r])].cpu()
                        dec.retire(r)
                for r, i, pages in sched.admit():
                    dec.admit(r, pages, budgets[i], start=KV_PAGE * sched.shared[i])
            if sched.finished:
                break
            decoding, pieces = sched.plan()
            holders = list(sched.req)
            h0 = time.perf_counter()
            if pieces:
                ends = [r for r, lo, n in pieces if lo + n == lens[sched.req[r]]]
                dec.mixed_step(decoding, [(r, prompts[sched.req[r]][lo:lo + n], lo, r in ends) for r, lo, n in pieces])
                made = [holders[r] for r in list(decoding) + ends]
            else:
                dec.decode_step()
                made = [i for i in holders if i is not None]
            host_ms = 1e3 * (time.perf_counter() - h0)
            ev = torch.cuda.Event(enable_timing=True)
            ev.record()
            log.append(('mixed' if pieces else 'graph', ev, host_ms, sum(n for _, _, n in pieces), len(decoding), made))
            steps += 1
    torch.cuda.synchronize()
    secs = time.perf_counter() - t0
    times, prev = {i: [] for i in range(len(prompts))}, 0.0
    split = dict(graph=[0.0, 0], mixed=[0.0, 0])
    for kind, ev, host_ms, pt, dt, made in log:
        t = start.elapsed_time(ev)
        split[kind][0] += t - prev
        split[kind][1] += 1
        prev = t
        for i in made:
            if len(times[i]) < out[i].numel():               # a request's first n tokens come from its first n steps
                times[i].append(t)
    if stats is not None:
        stats.update(prefilled=sched.prefilled, shared=list(sched.shared))
    del dec
    torch.cuda.empty_cache()
    return secs, out, log, times, split


def prefix_workload(V, copies=1, n=256, heads=8, head_len=1024, seed=0):
    """n requests: `heads` shared preambles of head_len tokens, each prompt one of them plus a unique tail of 32 .. 512
    tokens, budgets 16 .. 256; with copies > 1, n / copies such prompts each repeated `copies` times in a row."""
    g = torch.Generator().manual_seed(seed)
    pre = [torch.randint(0, V, (head_len,), generator=g) for _ in range(heads)]
    m = n // copies
    which = torch.randint(0, heads, (m,), generator=g).tolist()
    tails = torch.randint(32, 513, (m,), generator=g).tolist()
    prompts = [torch.cat((pre[h], torch.randint(0, V, (t,), generator=g))) for h, t in zip(which, tails)]
    budgets = torch.randint(16, 257, (m,), generator=g).tolist()
    return [p for p in prompts for _ in range(copies)], [b for b in budgets for _ in range(copies)]


def prefix_arms(model, prompts, budgets, rows=32, chunk=512):
    """continuous_serve with the prefix cache off, then on: per arm seconds, output tokens/s, prefilled prompt tokens,
    graph and mixed time, token gaps; and how many requests' tokens agree between the arms."""
    import numpy as np
    res, outs = {}, {}
    for arm, on in (('off', False), ('on', True)):
        st = {}
        secs, out, log, times, split = continuous_serve(model, prompts, budgets, rows, chunk, prefix_cache=on, stats=st)
        gaps = np.concatenate([np.diff(t) for t in times.values() if len(t) > 1])
        n_out = sum(o.numel() for o in out)
        res[arm] = dict(seconds=secs, tokens_per_s=n_out / secs, output_tokens=n_out, prefilled=st['prefilled'],
                        prompt_tokens=sum(p.numel() for p in prompts), shared_pages=sum(st['shared']),
                        graph_ms=split['graph'][0], graph_steps=split['graph'][1], mixed_ms=split['mixed'][0],
                        mixed_steps=split['mixed'][1], token_gap_ms_mean=float(gaps.mean()),
                        token_gap_ms_p99=float(np.percentile(gaps, 99)))
        outs[arm] = out
    res['same_requests'] = sum(torch.equal(a, b) for a, b in zip(outs['off'], outs['on']))
    res['requests'] = len(prompts)
    return res


def ragged_vs_padded_prefill(model, V, chunk=512, reps=3, seed=1):
    """8 prompts of 64 .. 2048 tokens prefilled in chunks of `chunk`: the paged PromptDecoder (every row through every
    chunk, padding included) against ContinuousDecoder mixed steps (packed prompt tokens only), ms each (median)."""
    from quip_b200.decode import KV_PAGE, ContinuousDecoder, ContinuousSchedule, PromptDecoder
    g = torch.Generator().manual_seed(seed)
    lens = [64, 128, 256, 512, 768, 1024, 1536, 2048]
    prompts = [torch.randint(0, V, (n,), generator=g) for n in lens]
    max_len = max(lens) + 1
    mp = -(-max_len // KV_PAGE)
    table = torch.arange(len(lens) * mp, dtype=torch.int32).view(len(lens), mp)
    pad = PromptDecoder(model, max_len=max_len, batch=len(lens), n_pages=len(lens) * mp, page_table=table)
    rag = ContinuousDecoder(model, max_len, len(lens), len(lens) * mp, 1)

    def padded():
        pad.prefill(prompts, chunk=chunk)

    def ragged():
        s = ContinuousSchedule(lens, [1] * len(lens), len(lens), len(lens) * mp, chunk)
        for r, i, pages in s.admit():
            rag.admit(r, pages, 1)
        while s.filling:
            _, pieces = s.plan()
            rag.mixed_step([], [(r, prompts[s.req[r]][lo:lo + n], lo, lo + n == lens[s.req[r]]) for r, lo, n in pieces])
        for r in range(len(lens)):
            rag.retire(r)
    res = {}
    with torch.no_grad():
        for name, fn in (('padded', padded), ('ragged', ragged)) * 2:           # the first round warms up
            ts = []
            for _ in range(reps):
                torch.cuda.synchronize()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                fn()
                e1.record()
                torch.cuda.synchronize()
                ts.append(e0.elapsed_time(e1))
            res[name] = sorted(ts)[len(ts) // 2]
    P = max(lens)
    res.update(lens=lens, padded_gemm_tokens=sum(len(lens) * min(chunk, P - c0) for c0 in range(0, P, chunk)),
               ragged_gemm_tokens=sum(lens))
    del pad, rag
    torch.cuda.empty_cache()
    return res


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


def beam_arms(model, cfg, B, K, fp8, P=512, n_new=128, steps=32, reps=50, seed=0):
    """Beam search on the synthetic model: B prompts of P tokens, K beams, no EOS.  The captured beam step (layers, head,
    candidates, select, fork) against a plain PromptDecoder step at B * K rows over the same prompts, then each beam
    kernel alone on the run's buffers (CUDA events): candidates over the step's logits, select at mid-run, and the fork
    with every row taking another row of its prompt as parent at a full current span (the most it copies)."""
    from quip_b200 import fused
    from quip_b200.decode import KV_PAGE, BeamDecoder, PromptDecoder, plan_prefix_pages
    kv = torch.float8_e4m3fn if fp8 else None
    g = torch.Generator().manual_seed(seed)
    prompts = [torch.randint(0, cfg.vocab_size, (P,), generator=g) for _ in range(B)]
    rows = [p for p in prompts for _ in range(K)]
    max_len = P + n_new
    table, n_plan, starts = plan_prefix_pages(rows, [max_len] * (B * K), max_pages=-(-max_len // KV_PAGE))
    bound = B * ((P - 1) // KV_PAGE + K * (-(-max_len // KV_PAGE) - (P - 1) // KV_PAGE)) + B * K
    dec = BeamDecoder(model, max_len, B, K, n_new, table, n_plan, [n_new] * B, kv_dtype=kv).capture()
    dec.prefill(rows, chunk=512, starts=starts)
    for _ in range(4):
        dec.step()
    torch.cuda.synchronize()
    beam_ms = events_ms(dec.graph.replay, steps, warm=0)
    base = PromptDecoder(model, max_len=max_len, batch=B * K, max_new=n_new, kv_dtype=kv).capture()
    base.prefill(rows, chunk=512)
    for _ in range(4):
        base.step()
    plain_ms = events_ms(base.graph.replay, steps, warm=0)
    del base
    torch.cuda.empty_cache()
    st, R, V = dec.beam, B * K, dec.V
    logits = dec.logits
    cand_ms = events_ms(lambda: fused.beam_candidates(logits, st['score'], K, dec.C, dec.cand_s, dec.cand_i), reps)
    st['done'].zero_()
    st['heur'].fill_(1)
    t_mid = torch.tensor([n_new // 2], device=logits.device)
    sel_ms = events_ms(lambda: fused.beam_select(dec.cand_s, dec.cand_i, dec.eos, dec.budget, t_mid, dec.pen, st, K, V,
                                                 False, False), reps)
    parents = torch.tensor([(r // K) * K + (r % K + 1) % K for r in range(R)], device=logits.device)
    lens = torch.full((R,), (P // KV_PAGE + 1) * KV_PAGE, dtype=torch.long, device=logits.device)   # 64 slots to copy
    kw = dict(k_scale=dec.k_scale, v_scale=dec.v_scale) if fp8 else {}
    fork_ms = events_ms(lambda: fused.kv_beam_fork(dec.k_cache, dec.v_cache, dec.page_table, dec.table_tmp, parents,
                                                   lens, dec.scratch0, **kw), reps)
    L, _, nkv, _, hd = dec.k_cache.shape
    forked = R if K > 1 else 0                          # K = 1: every parent is the row itself, nothing moves
    moved = forked * 2 * L * nkv * KV_PAGE * (hd * dec.k_cache.element_size() + (4 if fp8 else 0))
    r = dict(B=B, K=K, kv='e4m3' if fp8 else 'fp16', beam_step_ms=beam_ms, plain_step_ms=plain_ms,
             candidates_ms=cand_ms, select_ms=sel_ms, fork_ms=fork_ms,
             kernels_share_of_step=(cand_ms + sel_ms + fork_ms) / beam_ms,
             candidates_bytes_per_s=2 * V * R / (cand_ms * 1e-3),
             fork_copied_bytes=moved, fork_copied_bytes_per_s=moved / (fork_ms * 1e-3) if moved else 0.0,
             pool_pages=dec.n_pages, pool_bound=bound)
    del dec
    torch.cuda.empty_cache()
    return r


def logits_kernel_alone(B, V, hist_len, reps, n=3, n_bad=16, seed=0):
    """quip_logits_process alone on B fp16 rows of V logits: every processor on (penalty 1.2, n-gram size n, n_bad
    bad words of 1 .. 4 ids, min_new_tokens due with one EOS id), histories of hist_len ids drawn from 64 tokens so that
    n-grams repeat.  Timed as 20 launches captured in one CUDA graph (CUDA events around the replays).  Bytes: each
    row's history (int64) and one pass over its logits (the -0 pass of the bad words)."""
    from quip_b200 import fused
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(B, V, generator=g) * 3).half().to(dev)
    hist = torch.randint(0, 64, (B, hist_len), generator=g).to(dev)
    last = torch.full((B,), hist_len - 1, dtype=torch.long, device=dev)
    bad = torch.zeros(n_bad, 16, dtype=torch.long)
    bad_len = torch.tensor([1 + j % 4 for j in range(n_bad)], dtype=torch.int32)
    for j in range(n_bad):
        bad[j, :int(bad_len[j])] = torch.randint(0, 64, (int(bad_len[j]),), generator=g)
    args = (x, 1, hist, last, last - 8, torch.full((B,), 1.2, device=dev), torch.full((B,), n, dtype=torch.int32,
            device=dev), torch.full((B,), 16, dtype=torch.int32, device=dev), torch.tensor([2], device=dev),
            bad.to(dev), bad_len.to(dev))
    fused.logits_process(*args)
    graph, per = torch.cuda.CUDAGraph(), 20               # in a graph, as in a decode step: no host time between launches
    with torch.cuda.graph(graph):
        for _ in range(per):
            fused.logits_process(*args)
    ms = events_ms(graph.replay, max(reps // per, 5)) / per
    read = B * (hist_len * 8 + V * 2)
    return dict(B=B, V=V, hist_len=hist_len, n=n, bad_words=n_bad, kernel_ms=ms, bytes_per_s=read / (ms * 1e-3))


def logits_decode(model, cfg, B, P=512, n_new=128, trials=3, seed=0):
    """Decode with and without the logits processors on the synthetic model: B prompts of P tokens, greedy, the
    captured PromptDecoder step replayed for the n_new - 1 steps after the prefill (CUDA events), the two decoders
    alternating over `trials`.  Processors: repetition_penalty 1.2, no_repeat_ngram_size 3, 16 bad words, min_new_tokens
    16 with one EOS id."""
    from quip_b200.decode import PromptDecoder
    g = torch.Generator().manual_seed(seed)
    prompts = [torch.randint(0, cfg.vocab_size, (P,), generator=g) for _ in range(B)]
    bad = [torch.randint(0, cfg.vocab_size, (1 + j % 4,), generator=g).tolist() for j in range(16)]
    decs = {}
    for proc in (False, True):
        d = PromptDecoder(model, max_len=P + n_new, batch=B, max_new=n_new, processing=proc)
        if proc:
            d.set_processing(1.2, 3, 16, bad, [2])
        decs[proc] = d.capture()
    ms = {False: [], True: []}
    for _ in range(trials):
        for proc, d in decs.items():
            d.prefill(prompts, chunk=512)
            torch.cuda.synchronize()
            ms[proc].append(events_ms(d.graph.replay, n_new - 1, warm=0))
    same = float((decs[False].generated == decs[True].generated).float().mean())
    r = dict(B=B, P=P, n_new=n_new, plain_ms=min(ms[False]), processed_ms=min(ms[True]), trials_ms=ms,
             same_token_share_with_processors=same)
    r['plain_tok_s'], r['processed_tok_s'] = B * 1e3 / r['plain_ms'], B * 1e3 / r['processed_ms']
    r['slowdown'] = r['processed_ms'] / r['plain_ms'] - 1
    del decs
    torch.cuda.empty_cache()
    return r


def logprobs_kernel_alone(R, V, n, reps, seed=0):
    """quip_token_topk_logprobs alone on R fp16 rows of V logits (randn * 3), one output column per row, top n.  Timed
    as 20 launches captured in one CUDA graph (CUDA events around the replays).  Bytes: one pass over the logits (the
    kernel reads each row once for the lse and, with n > 0, three more times, mostly from L2)."""
    from quip_b200 import fused
    dev = torch.device('cuda:0')
    g = torch.Generator().manual_seed(seed)
    x = (torch.randn(R, V, generator=g) * 3).half().to(dev)
    tok = torch.randint(0, V, (R,), generator=g).to(dev)
    cols = torch.zeros(R, dtype=torch.long, device=dev)
    lp = torch.empty(R, 1, device=dev)
    ids = torch.empty(R, 1, n, dtype=torch.long, device=dev) if n else None
    top = torch.empty(R, 1, n, device=dev) if n else None
    fused.token_topk_logprobs(x, tok, cols, lp, ids, top)
    graph, per = torch.cuda.CUDAGraph(), 20
    with torch.cuda.graph(graph):
        for _ in range(per):
            fused.token_topk_logprobs(x, tok, cols, lp, ids, top)
    ms = events_ms(graph.replay, max(reps // per, 5)) / per
    return dict(R=R, V=V, n=n, kernel_ms=ms, bytes_per_s=R * V * 2 / (ms * 1e-3))


def logprobs_decode(model, cfg, B, proc, P=256, n_new=64, trials=3, seed=0):
    """The captured PromptDecoder step with logprobs off, n = 0 and n = 20: B prompts of P tokens, greedy, the step
    replayed for the n_new - 1 steps after the prefill (CUDA events), the three decoders alternating over `trials`.
    proc: the logits processors on (repetition_penalty 1.2, no_repeat_ngram_size 3, 16 bad words), so the step also
    copies its raw logits."""
    from quip_b200.decode import PromptDecoder
    g = torch.Generator().manual_seed(seed)
    prompts = [torch.randint(0, cfg.vocab_size, (P,), generator=g) for _ in range(B)]
    bad = [torch.randint(0, cfg.vocab_size, (1 + j % 4,), generator=g).tolist() for j in range(16)]
    decs = {}
    for n in (None, 0, 20):
        d = PromptDecoder(model, max_len=P + n_new, batch=B, max_new=n_new, processing=proc, logprobs=n)
        if proc:
            d.set_processing(1.2, 3, 0, bad, [2])
        decs[n] = d.capture()
    ms = {n: [] for n in decs}
    for _ in range(trials):
        for n, d in decs.items():
            d.prefill(prompts, chunk=256)
            torch.cuda.synchronize()
            ms[n].append(events_ms(d.graph.replay, n_new - 1, warm=0))
    same = all(torch.equal(decs[None].generated, d.generated) for d in decs.values())
    r = dict(B=B, P=P, n_new=n_new, processing=proc, off_ms=min(ms[None]), n0_ms=min(ms[0]), n20_ms=min(ms[20]),
             trials_ms={str(k): v for k, v in ms.items()}, tokens_identical=same)
    r['n0_overhead'], r['n20_overhead'] = r['n0_ms'] / r['off_ms'] - 1, r['n20_ms'] / r['off_ms'] - 1
    del decs
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', required=True)
    ap.add_argument('--models', default='llama7b,llama70b')
    ap.add_argument('--layers70b', type=int, default=80, help='decoder layers of the 70B shape to build (of 80)')
    ap.add_argument('--steps', type=int, default=16)
    ap.add_argument('--kernel-reps', type=int, default=100)
    ap.add_argument('--sections', default='kernel,prefill,decode,fp8')    # also: fp8kernel, sample, spec, chunked, paged,
    #                                                                         score, continuous, prefix, beam, logits,
    #                                                                         logprobs, assisted
    ap.add_argument('--score-docs', type=int, default=512, help='documents of 4 choices in the score section')
    a = ap.parse_args()
    sections = set(a.sections.split(','))
    if 'assisted' in sections:                         # the rows from shapes alone, before any device work
        from quip_b200.synth import MODELS
        unknown = set(a.models.split(',')) - set(MODELS)
        if unknown:
            raise SystemExit(f'unknown models {sorted(unknown)}')
        for name, tcfg, acfgs in assisted_plan(a.layers70b):
            if name not in a.models.split(','):
                continue
            for L, acfg in acfgs.items():
                for B in ASSIST_B:
                    max_len = ASSIST_CTX + a.steps * (max(ASSIST_K) + 1) + 2 + max(ASSIST_K) + 1
                    print(f'assisted plan {name} ({tcfg.num_hidden_layers} layers) + {L}-layer 7B-shape assistant '
                          f'B={B} k={ASSIST_K} ctx={ASSIST_CTX} max_len={max_len}: target cache '
                          f'{cache_bytes(tcfg, tcfg.num_hidden_layers, B, max_len) / 2**30:.2f} GiB, assistant cache '
                          f'{cache_bytes(acfg, L, B, max_len) / 2**30:.2f} GiB per decoder', flush=True)
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
        if 'logits' in sections and name == 'llama7b':
            rec['logits_kernel'] = []
            for B in (1, 32, 128):
                for V in (32000, 128256):
                    for hist_len in (512, 4096):
                        r = logits_kernel_alone(B, V, hist_len, a.kernel_reps)
                        rec['logits_kernel'].append(r)
                        print(f'logits process B={B} V={V} history={hist_len}: {1e3 * r["kernel_ms"]:.1f} us '
                              f'({r["bytes_per_s"] / 1e12:.2f} TB/s of history and logits)', flush=True)
        if 'logprobs' in sections and name == 'llama7b':
            rec['logprobs_kernel'] = []
            for R in (1, 8, 32, 256):
                for n in (0, 5, 20):
                    r = logprobs_kernel_alone(R, 32000, n, a.kernel_reps)
                    rec['logprobs_kernel'].append(r)
                    print(f'logprobs kernel R={R} V=32000 n={n}: {1e3 * r["kernel_ms"]:.1f} us '
                          f'({r["bytes_per_s"] / 1e12:.2f} TB/s of logits)', flush=True)
        if not sections & {'prefill', 'decode', 'fp8', 'sample', 'spec', 'assisted'} and not (
                sections & {'chunked', 'paged', 'score', 'continuous', 'prefix', 'beam', 'logits', 'logprobs'} and
                name == 'llama7b'):
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
        if 'continuous' in sections and name == 'llama7b':
            import numpy as np
            r = ragged_vs_padded_prefill(model, cfg.vocab_size)
            print(f'{name} prefill of 8 prompts 64..2048 in chunks of 512: padded {r["padded"]:.0f} ms '
                  f'({r["padded_gemm_tokens"]} GEMM tokens), ragged {r["ragged"]:.0f} ms ({r["ragged_gemm_tokens"]})',
                  flush=True)
            prompts, budgets = continuous_workload(cfg.vocab_size)
            s_secs, s_out, s_gemm = continuous_static(model, prompts, budgets, 32, 512)
            c_secs, c_out, log, times, split = continuous_serve(model, prompts, budgets, 32, 512)
            gaps = np.concatenate([np.diff(t) for t in times.values() if len(t) > 1])
            n_out = sum(budgets)
            mixed_host = [h for kind, _, h, *_ in log if kind == 'mixed']
            same = sum(torch.equal(a_, b_) for a_, b_ in zip(s_out, c_out))
            agree = [int((a_ != b_).nonzero()[0]) if not torch.equal(a_, b_) else a_.numel()
                     for a_, b_ in zip(s_out, c_out)]
            rec['continuous'] = dict(
                prefill_alone=r, requests=len(prompts), output_tokens=n_out,
                static=dict(seconds=s_secs, tokens_per_s=n_out / s_secs, prefill_gemm_tokens=s_gemm),
                continuous=dict(seconds=c_secs, tokens_per_s=n_out / c_secs,
                                prefill_gemm_tokens=sum(pt + dt for kind, _, _, pt, dt, _ in log if kind == 'mixed'),
                                prompt_tokens=sum(p.numel() for p in prompts),
                                token_gap_ms_mean=float(gaps.mean()), token_gap_ms_p99=float(np.percentile(gaps, 99)),
                                graph_ms=split['graph'][0], graph_steps=split['graph'][1], mixed_ms=split['mixed'][0],
                                mixed_steps=split['mixed'][1], mixed_host_ms_mean=float(np.mean(mixed_host))),
                same_requests=same, mean_agreeing_prefix=float(np.mean(agree)))
            c = rec['continuous']['continuous']
            print(f'{name} continuous 256 requests: static {n_out / s_secs:.0f} tok/s ({s_secs:.1f} s, prefill GEMM '
                  f'tokens {s_gemm}), continuous {c["tokens_per_s"]:.0f} tok/s ({c_secs:.1f} s, mixed-step GEMM tokens '
                  f'{c["prefill_gemm_tokens"]} of which {c["prompt_tokens"]} prompt); token gap mean '
                  f'{c["token_gap_ms_mean"]:.1f} ms p99 {c["token_gap_ms_p99"]:.1f} ms; graph {c["graph_ms"] / 1e3:.1f} s '
                  f'({c["graph_steps"]} steps), mixed {c["mixed_ms"] / 1e3:.1f} s ({c["mixed_steps"]} steps, host '
                  f'{c["mixed_host_ms_mean"]:.1f} ms each); identical requests {same} / {len(prompts)}, mean agreeing '
                  f'prefix {np.mean(agree):.1f} tokens', flush=True)
        if 'prefix' in sections and name == 'llama7b':
            rec['prefix'] = {}
            for case, copies in (('preambles', 1), ('preambles_x8', 8)):
                prompts, budgets = prefix_workload(cfg.vocab_size, copies)
                r = prefix_arms(model, prompts, budgets)
                rec['prefix'][case] = r
                for arm in ('off', 'on'):
                    x = r[arm]
                    print(f'{name} prefix {case} cache {arm}: {x["tokens_per_s"]:.0f} tok/s ({x["seconds"]:.1f} s), '
                          f'prefilled {x["prefilled"]} of {x["prompt_tokens"]} prompt tokens, graph '
                          f'{x["graph_ms"] / 1e3:.1f} s ({x["graph_steps"]} steps), mixed {x["mixed_ms"] / 1e3:.1f} s '
                          f'({x["mixed_steps"]} steps), token gap mean {x["token_gap_ms_mean"]:.1f} ms p99 '
                          f'{x["token_gap_ms_p99"]:.1f} ms', flush=True)
                print(f'{name} prefix {case}: identical requests {r["same_requests"]} / {r["requests"]}', flush=True)
        if 'beam' in sections and name == 'llama7b':
            rec['beam'] = []
            for fp8 in (False, True):
                for B in (1, 8):
                    for K in (1, 2, 4, 8):
                        r = beam_arms(model, cfg, B, K, fp8)
                        rec['beam'].append(r)
                        print(f'{name} beam {r["kv"]} B={B} K={K}: step {r["beam_step_ms"]:.3f} ms (plain '
                              f'{r["plain_step_ms"]:.3f} ms at {B * K} rows); candidates {1e3 * r["candidates_ms"]:.1f} us '
                              f'({r["candidates_bytes_per_s"] / 1e12:.2f} TB/s), select {1e3 * r["select_ms"]:.1f} us, '
                              f'fork {1e3 * r["fork_ms"]:.1f} us ({r["fork_copied_bytes_per_s"] / 1e12:.2f} TB/s copied); '
                              f'kernels {100 * r["kernels_share_of_step"]:.1f}% of the step; pool {r["pool_pages"]} pages '
                              f'(bound {r["pool_bound"]})', flush=True)
        if 'logits' in sections and name == 'llama7b':
            rec['logits_decode'] = []
            for B in (1, 32):
                r = logits_decode(model, cfg, B)
                rec['logits_decode'].append(r)
                print(f'{name} decode B={B} P=512, 128 new: plain {r["plain_ms"]:.3f} ms/step ({r["plain_tok_s"]:.0f} '
                      f'tok/s), with processors {r["processed_ms"]:.3f} ms/step ({r["processed_tok_s"]:.0f} tok/s), '
                      f'{100 * r["slowdown"]:+.2f}%; trials {r["trials_ms"]}', flush=True)
        if 'logprobs' in sections and name == 'llama7b':
            rec['logprobs_decode'] = []
            for proc in (False, True):
                for B in (1, 8, 32):
                    r = logprobs_decode(model, cfg, B, proc)
                    rec['logprobs_decode'].append(r)
                    print(f'{name} decode B={B} P=256 processors={proc}: off {r["off_ms"]:.3f} ms/step, n=0 '
                          f'{r["n0_ms"]:.3f} ({100 * r["n0_overhead"]:+.2f}%), n=20 {r["n20_ms"]:.3f} '
                          f'({100 * r["n20_overhead"]:+.2f}%); tokens identical {r["tokens_identical"]}; trials '
                          f'{r["trials_ms"]}', flush=True)
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
        if 'assisted' in sections:
            rec['assisted'] = []
            plan = {n: acfgs for n, _, acfgs in assisted_plan(a.layers70b)}
            for L, acfg in plan[name].items():
                assistant = build_synthetic_model(acfg, torch.device('cuda:0'), bits=2, seed=1, seqlen=4096)
                for B in ASSIST_B:
                    r = assisted_rows(model, assistant, B, ASSIST_K, ASSIST_CTX, a.steps, a.kernel_reps)
                    rec['assisted'].append(r)
                    print(f'{name} assisted B={B} ctx={ASSIST_CTX} assistant {L} layers: T=1 {r["assistant_t1_ms"]:.3f} '
                          f'ms, T=2 {r["assistant_t2_ms"]:.3f} ms, plain step {r["plain_step_ms"]:.3f} ms, rounds ' +
                          ', '.join(f'k={k} {ms:.3f} ms (break-even {r["break_even_yield"][k]:.2f} tokens)'
                                    for k, ms in r['round_ms'].items()), flush=True)
                del assistant
                torch.cuda.empty_cache()
            if name == 'llama7b':
                rec['assisted_self'], rec['assisted_self_generate'] = [], []
                for B in ASSIST_B:
                    r = assisted_rows(model, model, B, ASSIST_K, ASSIST_CTX, a.steps, a.kernel_reps)
                    rec['assisted_self'].append(r)
                    print(f'{name} assisted B={B} ctx={ASSIST_CTX} assistant = target: T=1 {r["assistant_t1_ms"]:.3f} '
                          f'ms, T=2 {r["assistant_t2_ms"]:.3f} ms, plain step {r["plain_step_ms"]:.3f} ms, rounds ' +
                          ', '.join(f'k={k} {ms:.3f} ms (break-even {r["break_even_yield"][k]:.2f} tokens)'
                                    for k, ms in r['round_ms'].items()), flush=True)
                    r = assisted_generate_self(model, B, 128, 4)
                    rec['assisted_self_generate'].append(r)
                    print(f'{name} generate B={B} 128 tokens, assistant = target, k=4: plain {r["plain_tok_s"]:.0f} '
                          f'tok/s, assisted {r["assisted_tok_s"]:.0f} tok/s, tokens per round {r["tokens_per_round"]}, '
                          f'same tokens {r["same_tokens"]}, agreeing prefix {r["agreeing_prefix"]}', flush=True)
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
