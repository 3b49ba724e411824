"""Token-by-token decode of a packed Llama or OPT model from one CUDA graph.

The reference's `benchmark()` (opt.py:431-482, llama.py via the same code) times an eager HF forward per
token with a growing KV cache; with the few-token kernels of this package one token's GPU work is a few
milliseconds while the eager Python path around it costs more than that in launch overhead.  `GraphDecoder`
is the same computation with everything a CUDA graph needs made static:

  * a KV cache of fixed length `max_len` per layer, written at the current position with `index_copy_`;
  * the position as a device tensor (advanced inside the graph), rotary cos/sin gathered from a table;
  * attention over the whole cache under a mask `arange(max_len) <= position`.

The decoder layers' own modules are reused (input_layernorm, the seven QuantLinear / nn.Linear projections,
post_attention_layernorm, final norm, lm_head): same weights, same kernels as `model(...)`; only the glue
between them is restated.  Llama (MHA or GQA; torch glue or the kernels of csrc/glue.cu) and OPT (the model benchmark() is
written for, opt.py:431-482: learned positions, LayerNorm with bias, ReLU MLP; torch glue).

`PromptDecoder` is the same step with one position per row and the attention of csrc/attn_decode.cu, filled from a batch
of prompts by the model's own many-token forward; `generate` runs it greedily from a CUDA graph.  With
kv_dtype=torch.float8_e4m3fn its cache holds e4m3 keys and values with one fp32 scale per cached head vector (hd + 4
bytes per vector instead of 2 * hd; the format is in include/quip_b200.h): twice the rows or context in the same memory,
half the cache bytes a step reads, at the cost of one e4m3 rounding of every cached key and value.  With sampling=True
its step selects by temperature, top-k and top-p with a per-row seed (quip_sample, csrc/sample.cu; the rule is in
include/quip_b200.h) instead of argmax, from settings held in device buffers, so one captured graph serves any settings.
`SpecDecoder` (generate(..., prompt_lookup_num_tokens=k)) verifies k prompt-lookup drafts per row in each captured step:
T = k + 1 tokens per row through the same layer loops, attention by csrc/attn_decode.cu's extend kernel, drafting and
acceptance by csrc/spec.cu.
"""
import math

import torch
import torch.nn.functional as F


def _rotate_half(x):
    h = x.shape[-1] // 2
    return torch.cat((-x[..., h:], x[..., :h]), dim=-1)


class GraphDecoder:
    def __init__(self, model, max_len=256, batch=1, ops=None, layer_range=None, first=True, last=True, kv_dtype=None):
        """kv_dtype: None, torch.float16 or the model's dtype: the cache in the model's dtype (the only cache this
        class keeps; PromptDecoder also takes torch.float8_e4m3fn).

        ops: provider of the fused glue kernels (quip_b200.fused.CudaGlue; picked up automatically when
        QUIP_FUSED_LAYER=1 on a CUDA device), None for the torch glue.

        layer_range=(lo, hi), first, last: one STAGE of a layer pipeline (the reference's opt_multigpu / llama_multigpu
        placement, opt.py:384-428) -- decoder layers lo..hi-1 with their own KV cache; a stage that is not the first reads
        the hidden state of the token from `h_in`, one that is not the last leaves it in `h_out` (static buffers, so the
        stage is still one graph); quip_b200.pipeline.PipelinedDecoder moves them between ranks."""
        cfg = model.config
        assert cfg.model_type in ('llama', 'opt'), 'GraphDecoder covers the Llama and OPT families'
        self.family = cfg.model_type
        self.model, self.max_len, self.batch = model, int(max_len), int(batch)
        self.dev = next(iter(model.parameters())).device
        self.nh = cfg.num_attention_heads
        dt = model.get_input_embeddings().weight.dtype     # fp16 on the GPU path; fp32 in the CPU tests
        self.first, self.last = bool(first), bool(last)
        self.T = 1                                         # tokens per row in a step (SpecDecoder: 1 + drafts)
        if self.family == 'llama':
            self.layers = list(model.model.layers)
            self.nkv = getattr(cfg, 'num_key_value_heads', None) or self.nh
            self.hd = getattr(cfg, 'head_dim', None) or cfg.hidden_size // self.nh
            # rotary table with the model's own module (HF default rope: positions 0 .. max_len-1)
            pos = torch.arange(self.max_len, device=self.dev)[None, :]
            with torch.no_grad():
                cos, sin = model.model.rotary_emb(torch.zeros(1, 1, cfg.hidden_size, device=self.dev, dtype=dt), pos)
            self.cos, self.sin = cos[0].to(dt).contiguous(), sin[0].to(dt).contiguous()        # (max_len, head_dim)
        else:
            dec = model.model.decoder
            assert self.max_len <= cfg.max_position_embeddings, 'OPT has learned positions: max_len beyond the table'
            self.layers = list(dec.layers)
            self.nkv = self.nh
            self.hd = cfg.hidden_size // self.nh
        lo, hi = layer_range or (0, len(self.layers))
        assert 0 <= lo < hi <= len(self.layers), (lo, hi)
        self.layers = self.layers[lo:hi]
        L, B = len(self.layers), self.batch
        self.h_in = None if self.first else torch.zeros(B, 1, cfg.hidden_size, dtype=dt, device=self.dev)
        self.h_out = None if self.last else torch.zeros(B, 1, cfg.hidden_size, dtype=dt, device=self.dev)
        self._alloc_cache((L, B, self.nkv, self.max_len, self.hd), dt, kv_dtype)
        self.position = torch.zeros(1, dtype=torch.long, device=self.dev)
        self.tokens = torch.zeros(B, dtype=torch.long, device=self.dev)
        self.logits = None
        self.graph = None
        self._arange = torch.arange(self.max_len, device=self.dev)
        self._pos_host = 0
        # q/k/v and gate/up read the same input: their chains of few-token kernels run on parallel branches
        self._side = [torch.cuda.Stream(device=self.dev) for _ in range(2)] if self.dev.type == 'cuda' else None
        if self.family != 'llama':
            ops = None                                     # the fused glue kernels are the Llama layer's
        elif ops is None and self.dev.type == 'cuda':
            from . import fused
            if fused.enabled() and getattr(cfg, 'hidden_act', 'silu') == 'silu' and self.hd % 16 == 0:
                ops = fused.CudaGlue()
        self.ops = ops

    def _alloc_cache(self, shape, dt, kv_dtype):
        """k_cache / v_cache of `shape` in the model's dtype dt."""
        if not (kv_dtype is None or kv_dtype == dt or kv_dtype == torch.float16):
            raise ValueError(f'{type(self).__name__} keeps its KV cache in the model dtype {dt}: kv_dtype {kv_dtype} '
                             'is not supported' + (' (PromptDecoder takes float8_e4m3fn)'
                                                   if kv_dtype == torch.float8_e4m3fn else ''))
        self.kv_dtype = dt
        self.k_cache = torch.zeros(shape, dtype=dt, device=self.dev)
        self.v_cache = torch.zeros_like(self.k_cache)

    def _parallel(self, x, mods):
        """[m(x) for m in mods] with every module after the first on its own stream (graph branches when capturing)."""
        if self._side is None:
            return [m(x) for m in mods]
        main = torch.cuda.current_stream(self.dev)
        outs = [None] * len(mods)
        for i, m in enumerate(mods[1:], 1):
            st = self._side[i - 1]
            st.wait_stream(main)
            with torch.cuda.stream(st):
                outs[i] = m(x)
        outs[0] = mods[0](x)
        for i in range(1, len(mods)):
            main.wait_stream(self._side[i - 1])
        return outs

    def reset(self):
        self._pos_host = 0
        self.position.zero_()
        self.k_cache.zero_()
        self.v_cache.zero_()

    # ---- the two seams of a step: which positions it is at, and appending k / v then attending.  This class keeps every
    # row at one position; PromptDecoder gives each row its own.

    def _step_positions(self):
        """Position of the step: (1,) (every row at the same position) or (B,); indexes the rotary rows and OPT's
        learned position table."""
        return self.position

    def _attn_mask(self, pos):
        """Boolean mask over the cache slots for _attend, broadcast over rows and heads."""
        return (self._arange <= pos)[None, None, None, :]                                  # (1, 1, 1, max_len)

    def _attend(self, li, q, k, v, mask, scale):
        """Append k, v (B, nkv, 1, hd) at the step's position of layer li's cache, attend q (B, nh, 1, hd) over the cache
        under mask: (B, 1, nh * hd)."""
        B, nh, nkv, hd = self.batch, self.nh, self.nkv, self.hd
        pos = self.position
        self.k_cache[li].index_copy_(2, pos, k)
        self.v_cache[li].index_copy_(2, pos, v)
        kk, vv = self.k_cache[li], self.v_cache[li]
        if nkv != nh:
            kk = kk.repeat_interleave(nh // nkv, dim=1)
            vv = vv.repeat_interleave(nh // nkv, dim=1)
        o = F.scaled_dot_product_attention(q, kk, vv, attn_mask=mask, scale=scale)
        return o.transpose(1, 2).reshape(B, 1, nh * hd)

    def _rope_rows(self, pos):
        """Rotary cos / sin rows of the step's tokens: (1 or B, hd) at T = 1; (B * T, hd), token i of row b at position
        pos[b] + i, otherwise."""
        if self.T > 1:
            pos = (pos[:, None] + self._tarange).reshape(-1)
        return self.cos.index_select(0, pos), self.sin.index_select(0, pos)

    def _advance(self):
        self.position.add_(1)

    # ---- the layers of the stage, three kinds of glue.  Each takes the hidden state entering the stage and returns
    # (h, pend): the residual stream and a branch output still to be added to it (None when already added).

    # csrc/glue.cu: 4 launches per layer instead of ~30 (at one token every torch elementwise op is a launch-latency-bound
    # graph node); the residual add of a branch rides on the next RMSNorm
    def _layers_fused(self, h):
        ops = self.ops
        B, T, nh, nkv, hd = self.batch, self.T, self.nh, self.nkv, self.hd
        pos = self._step_positions()
        h = h.contiguous()
        cos, sin = self._rope_rows(pos)
        cos = cos.expand(B * T, hd).contiguous()                                          # one row per token
        sin = sin.expand(B * T, hd).contiguous()
        mask = self._attn_mask(pos)
        pend = None
        for li, layer in enumerate(self.layers):
            a, mlp = layer.self_attn, layer.mlp
            n1, n2 = layer.input_layernorm, layer.post_attention_layernorm
            if pend is None:
                x = ops.rmsnorm(h, n1.weight, n1.variance_epsilon)
            else:
                h, x = ops.rmsnorm(h, n1.weight, n1.variance_epsilon, residual=pend)
            q, k, v = self._parallel(x, [a.q_proj, a.k_proj, a.v_proj])
            ops.rope_(q, k, cos, sin, hd)
            o = self._attend(li, q.view(B, T, nh, hd).transpose(1, 2), k.view(B, T, nkv, hd).transpose(1, 2),
                             v.view(B, T, nkv, hd).transpose(1, 2), mask, 1.0 / math.sqrt(hd))
            h, x = ops.rmsnorm(h, n2.weight, n2.variance_epsilon, residual=a.o_proj(o))
            gate, up = self._parallel(x, [mlp.gate_proj, mlp.up_proj])
            pend = mlp.down_proj(ops.silu_mul(gate, up))
        return h, pend

    def _layers_llama(self, h):
        B, T, nh, nkv, hd = self.batch, self.T, self.nh, self.nkv, self.hd
        pos = self._step_positions()
        cos, sin = self._rope_rows(pos)
        if T == 1:
            cos, sin = cos[:, None, None], sin[:, None, None]                              # (1 or B, 1, 1, hd)
        else:
            cos, sin = cos.view(B, 1, T, hd), sin.view(B, 1, T, hd)
        mask = self._attn_mask(pos)
        for li, layer in enumerate(self.layers):
            a = layer.self_attn
            x = layer.input_layernorm(h)
            q, k, v = self._parallel(x, [a.q_proj, a.k_proj, a.v_proj])
            q = q.view(B, T, nh, hd).transpose(1, 2)                                       # (B, nh, T, hd)
            k = k.view(B, T, nkv, hd).transpose(1, 2)
            v = v.view(B, T, nkv, hd).transpose(1, 2)
            q = q * cos + _rotate_half(q) * sin
            k = k * cos + _rotate_half(k) * sin
            o = self._attend(li, q, k, v, mask, 1.0 / math.sqrt(hd))
            h = h + a.o_proj(o)
            x = layer.post_attention_layernorm(h)
            mlp = layer.mlp
            gate, up = self._parallel(x, [mlp.gate_proj, mlp.up_proj])
            h = h + mlp.down_proj(F.silu(gate) * up)
        return h, None

    # OPT (modeling_opt.OPTDecoderLayer): pre- or post-LayerNorm, q scaled before the dot product, ReLU between fc1 and fc2;
    # biases live inside the (Quant)Linear modules
    def _layers_opt(self, h):
        B, T, nh, hd = self.batch, self.T, self.nh, self.hd
        mask = self._attn_mask(self._step_positions())
        for li, layer in enumerate(self.layers):
            a, before = layer.self_attn, layer.do_layer_norm_before
            x = layer.self_attn_layer_norm(h) if before else h
            q, k, v = self._parallel(x, [a.q_proj, a.k_proj, a.v_proj])
            q = (q * a.scaling).view(B, T, nh, hd).transpose(1, 2)                         # scaled first, as the HF module does
            o = self._attend(li, q, k.view(B, T, nh, hd).transpose(1, 2), v.view(B, T, nh, hd).transpose(1, 2), mask, 1.0)
            h = h + a.out_proj(o)
            if not before:
                h = layer.self_attn_layer_norm(h)
            x = layer.final_layer_norm(h) if before else h
            h = h + layer.fc2(layer.activation_fn(layer.fc1(x)))
            if not before:
                h = layer.final_layer_norm(h)
        return h, None

    def _embed(self):
        """Token (and, for OPT, learned position: index position + 2) embeddings of the step: (B, T, hidden); tokens is
        (B,) at T = 1 and (B, T) otherwise."""
        multi = self.T > 1
        if self.family == 'llama':
            return self.model.model.embed_tokens(self.tokens) if multi else self.model.model.embed_tokens(self.tokens)[:, None, :]
        d = self.model.model.decoder
        h = d.embed_tokens(self.tokens) if multi else d.embed_tokens(self.tokens)[:, None, :]
        if d.project_in is not None:
            h = d.project_in(h)
        pos = self._step_positions()
        if multi:
            return h + F.embedding(pos[:, None] + self._tarange + d.embed_positions.offset, d.embed_positions.weight)
        return h + F.embedding(pos + d.embed_positions.offset, d.embed_positions.weight)[:, None]

    def _head(self, h, pend):
        """Final norm (fused with the pending residual add on the glue-kernel path) -> lm_head: logits (B, vocab), or
        (B, T, vocab) for a step of T > 1 tokens per row."""
        if self.family == 'llama':
            fn = self.model.model.norm
            if self.ops is not None:
                _, h = self.ops.rmsnorm(h, fn.weight, fn.variance_epsilon, residual=pend)
            else:
                h = fn(h)
        else:
            d = self.model.model.decoder
            if d.final_layer_norm is not None:
                h = d.final_layer_norm(h)
            if d.project_out is not None:
                h = d.project_out(h)
        logits = self.model.lm_head(h)
        return logits if self.T > 1 else logits[:, 0, :]

    # one decode step of the stage on the static buffers (what the graph records)
    def _step(self):
        h = self._embed() if self.first else self.h_in
        if self.family == 'opt':
            h, pend = self._layers_opt(h)
        elif self.ops is not None:
            h, pend = self._layers_fused(h)
        else:
            h, pend = self._layers_llama(h)
        if self.last:
            self.logits = self._head(h, pend)
        else:
            self.h_out.copy_(h if pend is None else h + pend)   # fp16 add: the rounding the fused residual add performs
        self._advance()

    def capture(self):
        """Record one step.  The cache and position are restored afterwards, so capture is side-effect free."""
        from .quant import QuantLinear
        for mod in self.model.modules():                   # sibling groups launch on side streams: not while capturing
            if isinstance(mod, QuantLinear) and getattr(mod, '_group', None) is not None:
                raise RuntimeError('dissolve the sibling groups (quant.SiblingGroup.dissolve) before capturing')
        state = self._capture_state()
        saved = [t.clone() for t in state]
        side = torch.cuda.Stream(device=self.dev)
        side.wait_stream(torch.cuda.current_stream(self.dev))
        with torch.no_grad(), torch.cuda.stream(side):
            self._warm_up(state, saved)
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph, stream=side, capture_error_mode='thread_local'):
                self._step()
        torch.cuda.current_stream(self.dev).wait_stream(side)
        for t, t0 in zip(state, saved):
            t.copy_(t0)
        return self

    def _capture_state(self):
        """The buffers a step changes, which capture() puts back after its warm-up steps."""
        return [self.position, self.k_cache, self.v_cache]

    def _warm_up(self, state, saved):
        """Two eager steps for the lazy set-up (descriptors, workspaces) outside the graph.  Each starts from the saved
        state with the step counters brought into range (a decoder may be captured with its cache full) and is undone
        afterwards, so no index a warm-up step uses can leave its table."""
        for _ in range(2):
            self._counters_in_range()
            self._step()
            for t, t0 in zip(state, saved):
                t.copy_(t0)

    def _counters_in_range(self):
        self.position.clamp_(max=self.max_len - 1)

    def step(self, tokens):
        """tokens (B,) -> logits (B, vocab) for the next position; advances the cache."""
        if self._pos_host >= self.max_len:
            raise ValueError(f'KV cache of {self.max_len} positions is full')
        self._pos_host += 1
        self.tokens.copy_(tokens.reshape(-1))
        if self.graph is None:
            with torch.no_grad():
                self._step()
        else:
            self.graph.replay()
        return self.logits


def graph_decode_benchmark(model, input_ids, max_len=None, check=False):
    """`decode_benchmark` (reference benchmark(), opt.py:431-482) through the graph: median seconds per token and,
    with check, the perplexity of the fed sequence."""
    import time

    import numpy as np
    ids = input_ids.reshape(-1).to(next(iter(model.parameters())).device)
    dec = GraphDecoder(model, max_len=max_len or int(ids.numel()), batch=1).capture()
    times, tot = [], 0.0
    for i in range(ids.numel()):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        logits = dec.step(ids[i:i + 1])
        torch.cuda.synchronize()
        times.append(time.perf_counter() - t0)
        if check and i != ids.numel() - 1:
            tot += float(F.cross_entropy(logits.float(), ids[i + 1:i + 2]))
    ppl = float(np.exp(tot / (ids.numel() - 1))) if check else None
    return float(np.median(times)), ppl


def graph_decode_throughput(model, batch, steps=32, max_len=64, seed=0):
    """Aggregate tokens/s of `steps` graph-replayed decode steps with `batch` independent sequences (random token ids)."""
    dev = next(iter(model.parameters())).device
    dec = GraphDecoder(model, max_len=max_len, batch=batch).capture()
    gen = torch.Generator().manual_seed(seed)
    ids = torch.randint(0, model.config.vocab_size, (steps + 2, batch), generator=gen).to(dev)
    for i in range(2):
        dec.step(ids[i])
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for i in range(steps):
        dec.step(ids[2 + i])
    e1.record()
    torch.cuda.synchronize()
    ms = e0.elapsed_time(e1) / steps
    return batch * 1e3 / ms, ms


class PromptDecoder(GraphDecoder):
    """GraphDecoder with one position per row, so prompts of different lengths share a batch.

      * `positions` (B,) on the device, advanced inside the graph: rotary rows cos[positions], OPT's learned position
        looked up per row;
      * attention on CUDA is quip_decode_attention (csrc/attn_decode.cu): k / v appended at positions[b] inside the
        kernel, slots 0 .. positions[b] read and no others, GQA without copies.  On the CPU the same step in torch:
        per-row scatter into the cache, SDPA under the mask arange(max_len) <= positions[:, None];
      * `prefill` fills the cache from a batch of prompts with the model's own many-token forward;
      * max_new > 0: selection inside the step -- tokens = argmax(logits), stored in generated[:, t] -- so a host loop
        only replays the graph;
      * sampling=True: the selection is quip_sample (csrc/sample.cu) over the device buffers temperature, top_k, top_p
        and seed (B each, filled by set_sampling) at step t = _t, the index of the token in generated; a row's token
        depends on its logits, settings, seed and t only.  On the CPU the same rule in torch (_sample_torch);
      * kv_dtype=torch.float8_e4m3fn: k_cache / v_cache e4m3 with k_scale / v_scale (L, B, nkv, max_len) fp32, one scale
        per cached head vector.  prefill quantizes the model's keys and values into slots 0 .. P-1
        (quip_kv_quantize_fp8); the step quantizes k / v on append (quip_decode_attention_fp8) and attends over the
        quantized values of every slot, its own included.  On the CPU the same step in torch: quantize, per-row scatter,
        dequantize the cache to the compute dtype, SDPA under the mask.
    The whole model, no layer pipeline."""

    def __init__(self, model, max_len=256, batch=1, max_new=0, ops=None, kv_dtype=None, sampling=False):
        super().__init__(model, max_len=max_len, batch=batch, ops=ops, kv_dtype=kv_dtype)
        B = self.batch
        self.positions = torch.zeros(B, dtype=torch.long, device=self.dev)
        self.max_new = int(max_new)
        self.generated = torch.zeros(B, max(self.max_new, 1), dtype=torch.long, device=self.dev)
        self._t = torch.zeros(1, dtype=torch.long, device=self.dev)
        self._rows = torch.arange(B, device=self.dev)
        self._pos_host = [0] * B
        self._t_host = 0
        self._kernel = self.dev.type == 'cuda'
        self.sampling = bool(sampling)
        if self.sampling:
            self.temperature = torch.ones(B, dtype=torch.float32, device=self.dev)
            self.top_k = torch.zeros(B, dtype=torch.int32, device=self.dev)
            self.top_p = torch.ones(B, dtype=torch.float32, device=self.dev)
            self.seed = torch.zeros(B, dtype=torch.int64, device=self.dev)

    def set_sampling(self, temperature=1.0, top_k=0, top_p=1.0, seed=0):
        """Write the sampling settings into the device buffers a captured step reads: each a scalar for every row or one
        value per row.  seed: ints in [0, 2^64), or an int64 tensor holding their two's-complement bits.  Temperature 0 or
        top_k 1 makes a row greedy (argmax)."""
        if not self.sampling:
            raise ValueError('set_sampling needs a PromptDecoder made with sampling=True')
        B = self.batch

        def rows(v):
            v = v.tolist() if torch.is_tensor(v) else v
            v = list(v) if isinstance(v, (list, tuple)) else [v] * B
            if len(v) != B:
                raise ValueError(f'{len(v)} values for a decoder of batch {B}')
            return v
        if torch.is_tensor(seed) and seed.dtype == torch.int64:
            seeds = rows(seed)
        else:
            seeds = [int(x) for x in rows(seed)]
            if any(not 0 <= x < 2 ** 64 for x in seeds):
                raise ValueError('seeds must lie in [0, 2^64)')
            seeds = [x - 2 ** 64 if x >= 2 ** 63 else x for x in seeds]
        self.temperature.copy_(torch.tensor(rows(temperature), dtype=torch.float32))
        self.top_k.copy_(torch.tensor(rows(top_k), dtype=torch.int32))
        self.top_p.copy_(torch.tensor(rows(top_p), dtype=torch.float32))
        self.seed.copy_(torch.tensor(seeds, dtype=torch.int64))

    def _select(self, logits, out=None):
        """out (default: tokens) = the token chosen for each row from logits (B, vocab) at step _t: argmax, or with
        sampling the rule of quip_sample."""
        out = self.tokens if out is None else out
        if not self.sampling:
            out.copy_(logits.argmax(-1))
        elif self._kernel:
            from . import fused
            fused.sample(logits, self.temperature, self.top_k, self.top_p, self.seed, self._t, out)
        else:
            out.copy_(_sample_torch(logits, self.temperature, self.top_k, self.top_p, self.seed, int(self._t)))

    def _alloc_cache(self, shape, dt, kv_dtype):
        """fp8: e4m3 caches and their fp32 scales, allocated as such (never an fp16 cache first: at the sizes fp8 is for,
        that one would not fit)."""
        self.k_scale = self.v_scale = None
        if kv_dtype != torch.float8_e4m3fn:
            return super()._alloc_cache(shape, dt, kv_dtype)
        self.kv_dtype = kv_dtype
        self.k_cache = torch.zeros(shape, dtype=kv_dtype, device=self.dev)
        self.v_cache = torch.zeros_like(self.k_cache)
        self.k_scale = torch.zeros(shape[:-1], dtype=torch.float32, device=self.dev)
        self.v_scale = torch.zeros_like(self.k_scale)

    @property
    def _fp8(self):
        return self.kv_dtype == torch.float8_e4m3fn

    def _step_positions(self):
        return self.positions

    def _attn_mask(self, pos):
        if self._kernel:
            return None
        if self.T > 1:                                                                 # (B, 1, T, max_len), causal
            return (self._arange[None, None] <= (pos[:, None] + self._tarange)[:, :, None])[:, None]
        return (self._arange[None] <= pos[:, None])[:, None, None, :]                  # (B, 1, 1, max_len)

    def _attend(self, li, q, k, v, mask, scale):
        B, nh, nkv, hd = self.batch, self.nh, self.nkv, self.hd
        if self.T > 1:
            return self._attend_multi(li, q, k, v, mask, scale)
        if self._kernel:
            from . import fused
            sc = dict(k_scale=self.k_scale[li], v_scale=self.v_scale[li]) if self._fp8 else {}
            o = fused.decode_attention(q.reshape(B, nh, hd).contiguous(), k.reshape(B, nkv, hd).contiguous(),
                                       v.reshape(B, nkv, hd).contiguous(), self.k_cache[li], self.v_cache[li],
                                       self.positions, scale, **sc)
            return o.view(B, 1, nh * hd)
        if self._fp8:
            for x, cache, scales in ((k, self.k_cache[li], self.k_scale[li]), (v, self.v_cache[li], self.v_scale[li])):
                xq, xs = _e4m3_quantize(x[:, :, 0])
                cache[self._rows, :, self.positions] = xq
                scales[self._rows, :, self.positions] = xs
            kk = _e4m3_dequantize(self.k_cache[li], self.k_scale[li], q.dtype)
            vv = _e4m3_dequantize(self.v_cache[li], self.v_scale[li], q.dtype)
        else:
            self.k_cache[li][self._rows, :, self.positions] = k[:, :, 0]
            self.v_cache[li][self._rows, :, self.positions] = v[:, :, 0]
            kk, vv = self.k_cache[li], self.v_cache[li]
        if nkv != nh:
            kk = kk.repeat_interleave(nh // nkv, dim=1)
            vv = vv.repeat_interleave(nh // nkv, dim=1)
        o = F.scaled_dot_product_attention(q, kk, vv, attn_mask=mask, scale=scale)
        return o.transpose(1, 2).reshape(B, 1, nh * hd)

    def _attend_multi(self, li, q, k, v, mask, scale):
        """_attend for T > 1 tokens per row (q (B, nh, T, hd), k / v (B, nkv, T, hd)): token i appended at slot
        positions[b] + i and attending over slots 0 .. positions[b] + i.  CUDA: quip_extend_attention(_fp8), token-major
        operands; CPU: per-row scatter of the T slots, SDPA under the causal mask.  Returns (B, T, nh * hd)."""
        B, T, nh, nkv, hd = self.batch, self.T, self.nh, self.nkv, self.hd
        if self._kernel:
            from . import fused
            sc = dict(k_scale=self.k_scale[li], v_scale=self.v_scale[li]) if self._fp8 else {}
            o = fused.extend_attention(q.transpose(1, 2).contiguous(), k.transpose(1, 2).contiguous(),
                                       v.transpose(1, 2).contiguous(), self.k_cache[li], self.v_cache[li],
                                       self.positions, scale, **sc)
            return o.view(B, T, nh * hd)
        rows = self._rows[:, None].expand(B, T)
        slots = self.positions[:, None] + self._tarange                                 # (B, T)
        if self._fp8:
            for x, cache, scales in ((k, self.k_cache[li], self.k_scale[li]), (v, self.v_cache[li], self.v_scale[li])):
                xq, xs = _e4m3_quantize(x.transpose(1, 2))                              # (B, T, nkv, hd), (B, T, nkv)
                cache[rows, :, slots] = xq
                scales[rows, :, slots] = xs
            kk = _e4m3_dequantize(self.k_cache[li], self.k_scale[li], q.dtype)
            vv = _e4m3_dequantize(self.v_cache[li], self.v_scale[li], q.dtype)
        else:
            self.k_cache[li][rows, :, slots] = k.transpose(1, 2)
            self.v_cache[li][rows, :, slots] = v.transpose(1, 2)
            kk, vv = self.k_cache[li], self.v_cache[li]
        if nkv != nh:
            kk = kk.repeat_interleave(nh // nkv, dim=1)
            vv = vv.repeat_interleave(nh // nkv, dim=1)
        o = F.scaled_dot_product_attention(q, kk, vv, attn_mask=mask, scale=scale)
        return o.transpose(1, 2).reshape(B, T, nh * hd)

    def _advance(self):
        self.positions.add_(1)
        if self.max_new:
            self._select(self.logits)
            self.generated.index_copy_(1, self._t, self.tokens[:, None])
            self._t.add_(1)

    def _capture_state(self):
        # Not the cache: a warm-up step writes slot positions[b] (clamped to max_len - 1), and a later step writes that
        # slot before it reads it.  A row clamped from max_len takes no further step: its cache is full.
        return [self.positions, self.tokens, self._t, self.generated]

    def _counters_in_range(self):
        self.positions.clamp_(max=self.max_len - 1)
        self._t.clamp_(max=self.generated.shape[1] - 1)

    def reset(self):
        """Back to an empty cache: every row at position 0, nothing generated."""
        super().reset()
        if self._fp8:
            self.k_scale.zero_()
            self.v_scale.zero_()
        self.positions.zero_()
        self._t.zero_()
        self.generated.zero_()
        self._pos_host = [0] * self.batch
        self._t_host = 0

    def prefill(self, prompts):
        """Fill the cache from `prompts` (B 1-D id tensors): right-padded to the longest, run through the model's own
        forward (`model.model(ids, attention_mask=..., use_cache=True)`, the packed linears at M = B * P), its keys and
        values copied to the cache slots 0 .. P-1.  Slots past a row's length hold padding; the step overwrites them in
        turn and never reads past positions[b].  Returns the logits after each prompt's last token (B, vocab); with
        max_new > 0 the token selected from them (argmax, or sampled at t = 0) is the first generated token and the next
        step's input."""
        B = self.batch
        if len(prompts) != B:
            raise ValueError(f'{len(prompts)} prompts for a decoder of batch {B}')
        lens = [int(p.numel()) for p in prompts]
        if min(lens) < 1:
            raise ValueError('empty prompt')
        P = max(lens)
        if P > self.max_len:
            raise ValueError(f'a prompt of {P} tokens does not fit a cache of {self.max_len} positions')
        ids = torch.zeros(B, P, dtype=torch.long, device=self.dev)
        for b, p in enumerate(prompts):
            ids[b, :lens[b]] = p.reshape(-1).to(self.dev)
        lens_t = torch.tensor(lens, dtype=torch.long, device=self.dev)
        attn = (torch.arange(P, device=self.dev)[None] < lens_t[:, None]).long()
        with torch.no_grad():
            out = self.model.model(input_ids=ids, attention_mask=attn, use_cache=True)
            cache = out.past_key_values
            for li in range(len(self.layers)):
                if self._fp8:
                    self._store_fp8(li, cache.layers[li].keys, cache.layers[li].values)
                else:
                    self.k_cache[li, :, :, :P].copy_(cache.layers[li].keys)
                    self.v_cache[li, :, :, :P].copy_(cache.layers[li].values)
            logits = self.model.lm_head(out.last_hidden_state[self._rows, lens_t - 1])     # last real token per row
            self.positions.copy_(lens_t)
            self._pos_host = list(lens)
            if self.max_new:
                self._first_token(logits)
        return logits

    def _first_token(self, logits):
        """Select the first generated token from the prefill's logits (B, vocab), at t = 0."""
        self._t.zero_()
        self._select(logits)
        self.generated[:, 0].copy_(self.tokens)
        self._t.fill_(1)
        self._t_host = 1

    def _store_fp8(self, li, keys, values):
        """Quantize the prefill's keys / values (B, nkv, P, hd) into slots 0 .. P-1 of layer li's e4m3 cache."""
        P = keys.shape[2]
        for x, cache, scales in ((keys, self.k_cache[li], self.k_scale[li]), (values, self.v_cache[li], self.v_scale[li])):
            if self._kernel:
                from . import fused
                fused.kv_quantize(x.to(torch.float16).contiguous(), cache, scales)
            else:
                xq, xs = _e4m3_quantize(x)
                cache[:, :, :P] = xq
                scales[:, :, :P] = xs

    def step(self, tokens=None):
        """One step at every row's own position: tokens (B,) -- or, when generating, the tokens the previous step
        selected -- to logits (B, vocab); advances every row."""
        if max(self._pos_host) >= self.max_len:
            raise ValueError(f'KV cache of {self.max_len} positions is full')
        if self.max_new and self._t_host >= self.max_new:
            raise ValueError(f'{self.max_new} tokens generated already')
        self._pos_host = [p + 1 for p in self._pos_host]
        self._t_host += 1 if self.max_new else 0
        if tokens is not None:
            self.tokens.copy_(tokens.reshape(-1))
        if self.graph is None:
            with torch.no_grad():
                self._step()
        else:
            self.graph.replay()
        return self.logits



class SpecDecoder(PromptDecoder):
    """PromptDecoder whose step verifies prompt-lookup drafts: T = 1 + draft_tokens tokens per row in one step.

    One captured step runs
      * draft: tokens (B, T) = the current token hist[b, positions[b]] and k drafts by n-gram lookup in the row's own
        prompt and output (quip_ngram_draft; the rule is in include/quip_b200.h);
      * the model on the B * T tokens: token i of row b at position positions[b] + i, attention by
        quip_extend_attention(_fp8) (causal inside the new tokens);
      * select: targets (B, T) from the step's logits (B, T, vocab): argmax, or with sampling the rule of quip_sample at
        t = n_gen[b] + i (quip_sample_at), the index the token would take in generated -- so a token is the one the
        non-speculative decoder chooses from the same logits;
      * accept: the longest prefix of drafts that equals the targets before them, plus one target (quip_spec_accept),
        appended to generated and hist; positions and n_gen advance by that count, accepted by the drafts taken.
    Rejected drafts leave keys and values in slots past positions[b]; no step reads there before overwriting them.
    A row with max_new tokens does not advance.  On the CPU the same step in torch (_ngram_draft_torch,
    _spec_accept_torch, per-row scatter of the T slots and SDPA under the causal mask).  Needs max_len >= the longest
    prompt + max_new + draft_tokens (a finished row's step still writes its T slots)."""

    def __init__(self, model, max_len=256, batch=1, max_new=1, draft_tokens=4, max_ngram=3, ops=None, kv_dtype=None,
                 sampling=False):
        k, n_max = int(draft_tokens), int(max_ngram)
        if not 1 <= k <= 7:
            raise ValueError(f'draft_tokens must lie in [1, 7], got {draft_tokens}')
        if n_max < 1:
            raise ValueError(f'max_ngram must be at least 1, got {max_ngram}')
        if int(max_new) < 1:
            raise ValueError(f'a SpecDecoder selects inside its step: max_new must be at least 1, got {max_new}')
        if int(max_len) < k + 2:
            raise ValueError(f'max_len {max_len} leaves no room for a step of {k + 1} tokens')
        super().__init__(model, max_len=max_len, batch=batch, max_new=max_new, ops=ops, kv_dtype=kv_dtype,
                         sampling=sampling)
        B, dev = self.batch, self.dev
        self.k, self.n_min, self.n_max = k, 1, n_max
        self.T = k + 1
        self._tarange = torch.arange(self.T, device=dev)
        self.tokens = torch.zeros(B, self.T, dtype=torch.long, device=dev)
        self.targets = torch.zeros(B, self.T, dtype=torch.long, device=dev)
        self.hist = torch.zeros(B, self.max_len, dtype=torch.long, device=dev)
        self.n_gen = torch.zeros(B, dtype=torch.long, device=dev)
        self.accepted = torch.zeros(B, dtype=torch.long, device=dev)
        self._first = torch.zeros(B, dtype=torch.long, device=dev)
        self._steps_host = 0

    def _step(self):
        self._draft()
        super()._step()

    def _draft(self):
        if self._kernel:
            from . import fused
            fused.ngram_draft(self.hist, self.positions, self.tokens, self.n_min, self.n_max)
        else:
            self.tokens.copy_(_ngram_draft_torch(self.hist, self.positions, self.k, self.n_min, self.n_max))

    def _advance(self):
        logits = self.logits                                                            # (B, T, vocab)
        if not self.sampling:
            self.targets.copy_(logits.argmax(-1))
        elif self._kernel:
            from . import fused
            fused.sample_at(logits, self.temperature, self.top_k, self.top_p, self.seed, self.n_gen, self.targets)
        else:
            self.targets.copy_(_sample_torch_at(logits, self.temperature, self.top_k, self.top_p, self.seed, self.n_gen))
        if self._kernel:
            from . import fused
            fused.spec_accept(self.tokens, self.targets, self.generated, self.hist, self.positions, self.n_gen,
                              self.accepted, self.max_new)
        else:
            _spec_accept_torch(self.tokens, self.targets, self.generated, self.hist, self.positions, self.n_gen,
                               self.accepted, self.max_new)

    def _capture_state(self):
        return super()._capture_state() + [self.targets, self.hist, self.n_gen, self.accepted]

    def _counters_in_range(self):
        # a warm-up step writes slots positions[b] .. positions[b] + k: keep them inside the cache
        super()._counters_in_range()
        self.positions.clamp_(max=self.max_len - self.T)

    def reset(self):
        super().reset()
        for t in (self.tokens, self.targets, self.hist, self.n_gen, self.accepted):
            t.zero_()
        self._steps_host = 0

    def prefill(self, prompts):
        """PromptDecoder.prefill, plus the history: each prompt and its first generated token in hist, n_gen = 1."""
        lens = [int(torch.as_tensor(p).numel()) for p in prompts]
        if lens and max(lens) + self.max_new + self.k > self.max_len:
            raise ValueError(f'a prompt of {max(lens)} tokens, {self.max_new} new ones and {self.k} drafts exceed the '
                             f'cache of {self.max_len} positions')
        logits = super().prefill(prompts)
        with torch.no_grad():
            for b, p in enumerate(prompts):
                self.hist[b, :lens[b]] = torch.as_tensor(p).reshape(-1).to(self.dev)
        self.accepted.zero_()
        self._steps_host = 0
        return logits

    def _first_token(self, logits):
        self._t.zero_()
        self._select(logits, out=self._first)
        self.generated[:, 0].copy_(self._first)
        self.hist[self._rows, self.positions] = self._first
        self.n_gen.fill_(1)
        self._t.fill_(1)
        self._t_host = 1

    def step(self, tokens=None):
        """One speculative step for every row that has fewer than max_new tokens; returns the logits (B, T, vocab).
        Every row is done after max_new - 1 steps (each gives an unfinished row at least one token)."""
        if tokens is not None:
            raise ValueError('a SpecDecoder step feeds its own tokens (the current one and its drafts)')
        if self._steps_host >= self.max_new - 1:
            raise ValueError(f'{self.max_new} tokens generated already')
        self._steps_host += 1
        if self.graph is None:
            with torch.no_grad():
                self._step()
        else:
            self.graph.replay()
        return self.logits


def _ngram_draft_torch(hist, positions, k, n_min, n_max):
    """The rule of quip_ngram_draft (include/quip_b200.h) in torch, one row at a time: (B, 1 + k)."""
    B, max_len = hist.shape
    out = torch.zeros(B, k + 1, dtype=torch.long)
    for b in range(B):
        c = int(positions[b])
        if not 0 <= c < max_len:
            continue
        h = hist[b, :c + 1].cpu()
        e = torch.arange(c)
        length = torch.zeros(c, dtype=torch.long)
        alive = torch.ones(c, dtype=torch.bool)
        for t in range(min(n_max, c)):                               # suffix element t: h[e - t] == h[c - t]
            alive = alive & (e >= t) & (h[(e - t).clamp(min=0)] == h[c - t])
            length += alive.long()
        key = torch.where(length >= n_min, length * (c + 1) + e, torch.full_like(e, -1))   # longest, then latest
        u = h.tolist()
        best = int(key.argmax()) if c and int(key.max()) >= 0 else -1
        for i in range(1, k + 1):
            u.append(u[c] if best < 0 else u[best + i])
        out[b] = torch.tensor(u[c:])
    return out.to(hist.device)


def _spec_accept_torch(tokens, targets, generated, hist, positions, n_gen, accepted, max_new):
    """The rule of quip_spec_accept (include/quip_b200.h) in torch, in place."""
    B, T = tokens.shape
    a = (tokens[:, 1:] == targets[:, :-1]).long().cumprod(1).sum(1)
    live = n_gen < max_new
    e = torch.where(live, torch.minimum(a + 1, max_new - n_gen), torch.zeros_like(a))
    j = torch.arange(T, device=tokens.device)
    w = j[None] < e[:, None]
    rows = torch.arange(B, device=tokens.device)[:, None].expand(B, T)
    gcol, hcol = n_gen[:, None] + j, positions[:, None] + 1 + j
    generated[rows[w], gcol[w]] = targets[w]
    hw = w & (hcol >= 0) & (hcol < hist.shape[1])
    hist[rows[hw], hcol[hw]] = targets[hw]
    positions += e
    n_gen += e
    accepted += torch.where(live, e - 1, torch.zeros_like(e))


def _sample_torch_at(logits, temperature, top_k, top_p, seed, steps):
    """_sample_torch over logits (B, T, vocab): token i of row b with row b's settings at step steps[b] + i."""
    B, T, _ = logits.shape
    out = torch.empty(B, T, dtype=torch.long)
    for b in range(B):
        for i in range(T):
            out[b, i] = _sample_torch(logits[b, i][None], temperature[b:b + 1], top_k[b:b + 1], top_p[b:b + 1],
                                      seed[b:b + 1], int(steps[b]) + i)[0]
    return out.to(logits.device)

def _e4m3_quantize(x):
    """The e4m3 format of the fp8 cache (include/quip_b200.h) in torch, for the CPU step: x (..., hd) -> (e4m3 (..., hd),
    fp32 scales (...))."""
    x = x.float()
    amax = x.abs().amax(-1)
    s = torch.where(amax == 0, torch.ones_like(amax), amax / torch.full_like(amax, 448.0))       # IEEE division
    return (x / s[..., None]).to(torch.float8_e4m3fn), s


def _e4m3_dequantize(q, s, dtype):
    return (q.float() * s[..., None]).to(dtype)


def _philox_uniform(seed, t):
    """u = (w >> 8) * 2^-24, w the first word of Philox4x32-10 of counter (t lo, t hi, 0, 0) under key (seed lo, seed hi);
    seed and t are Python ints taken mod 2^64."""
    M = 0xFFFFFFFF
    seed, t = seed % 2 ** 64, t % 2 ** 64
    c0, c1, c2, c3 = t & M, t >> 32, 0, 0
    k0, k1 = seed & M, seed >> 32
    for r in range(10):
        if r:
            k0, k1 = (k0 + 0x9E3779B9) & M, (k1 + 0xBB67AE85) & M
        p0, p1 = 0xD2511F53 * c0, 0xCD9E8D57 * c2
        c0, c1, c2, c3 = (p1 >> 32) ^ c1 ^ k0, p1 & M, (p0 >> 32) ^ c3 ^ k1, p0 & M
    return (c0 >> 8) * 2.0 ** -24


def _sample_torch(logits, temperature, top_k, top_p, seed, t):
    """The rule of quip_sample (include/quip_b200.h) in torch, one row at a time: the CPU step of a sampling
    PromptDecoder.  z is fp32 as the kernel has it (same ranking, same top-k set); e and its sums are float64."""
    B, V = logits.shape
    out = torch.empty(B, dtype=torch.long)
    for b in range(B):
        x = logits[b].detach().float().cpu()
        T, k, p = float(temperature[b]), int(top_k[b]), float(top_p[b])
        if not T > 0 or k == 1:
            out[b] = x.argmax()
            continue
        z = x / torch.tensor(T, dtype=torch.float32)
        order = torch.sort(z, descending=True, stable=True).indices
        cand = order[:min(k, V) if k > 0 else V]
        e = torch.exp(z[cand].double() - float(z[order[0]]))
        n = cand.numel()
        if p < 1:
            cs = torch.cumsum(e, 0)
            n = min(n, max(1, int(torch.searchsorted(cs, torch.tensor([p * float(cs[-1])], dtype=torch.float64))) + 1))
        kept, ek = cand[:n], e[:n]
        idx = torch.argsort(kept, stable=True)                     # index order
        run = torch.cumsum(ek[idx], 0)
        thr = _philox_uniform(int(seed[b]), t) * float(run[-1])
        j = min(int(torch.searchsorted(run, torch.tensor([thr], dtype=torch.float64), right=True)), n - 1)
        out[b] = kept[idx[j]]
    return out.to(logits.device)


EOS_CHECK_EVERY = 16


def _per_prompt(name, v, n):
    """A generate() setting as one value per prompt: a scalar for all, or a list / 1-D tensor of n."""
    if torch.is_tensor(v):
        v = v.tolist()
    if isinstance(v, (list, tuple)):
        if len(v) != n:
            raise ValueError(f'{name}: {len(v)} values for {n} prompts')
        return list(v)
    return [v] * n


def _sampling_settings(n, temperature, top_k, top_p, seed):
    """Validated per-prompt (temperature, top_k, top_p, seeds) for n prompts; an int seed gives prompt b the seed
    seed + b (mod 2^64)."""
    temps = [float(t) for t in _per_prompt('temperature', temperature, n)]
    if any(not (math.isfinite(t) and t >= 0) for t in temps):
        raise ValueError(f'temperature must be finite and >= 0, got {temperature}')
    ks = _per_prompt('top_k', top_k, n)
    if any(int(k) != k or k < 0 for k in ks):
        raise ValueError(f'top_k must be an integer >= 0, got {top_k}')
    ps = [float(p) for p in _per_prompt('top_p', top_p, n)]
    if any(not 0 < p <= 1 for p in ps):
        raise ValueError(f'top_p must lie in (0, 1], got {top_p}')
    explicit = torch.is_tensor(seed) or isinstance(seed, (list, tuple))
    seeds = _per_prompt('seed', seed, n) if explicit else [seed]
    if any(int(x) != x or not 0 <= x < 2 ** 64 for x in seeds):
        raise ValueError(f'seeds must be integers in [0, 2^64), got {seed}')
    if not explicit:
        seeds = [(int(seed) + b) % 2 ** 64 for b in range(n)]
    return temps, [int(k) for k in ks], ps, [int(x) for x in seeds]


def generate(model, prompts, max_new_tokens, max_len=None, eos_token_id=None, kv_dtype=None, do_sample=False,
             temperature=1.0, top_k=0, top_p=1.0, seed=0, prompt_lookup_num_tokens=None, max_matching_ngram_size=3,
             spec_stats=None):
    """Continuations of a batch of prompts (1-D id tensors, any lengths) of a Llama or OPT model: one tensor of new token
    ids per prompt, cut after its first `eos_token_id` (an id or a list of ids).  The prompts are prefilled in one
    many-token forward; each new token is one replay of a captured PromptDecoder step on CUDA (eager on the CPU).
    max_len (default: longest prompt + max_new_tokens) is the KV cache length.  Stops early once every row has produced
    an EOS, checked every EOS_CHECK_EVERY steps.  kv_dtype=torch.float8_e4m3fn keeps the KV cache in e4m3 with per-vector
    scales (PromptDecoder); None (the default) keeps it in the model's dtype.

    Greedy (argmax) unless do_sample=True, which samples by the rule of include/quip_b200.h (quip_sample): temperature
    (>= 0, finite; 0 is greedy), top_k (0: off; exactly k candidates, ties by lower id), top_p (in (0, 1]) and seed, each
    a scalar or one value per prompt.  An int seed gives prompt b the seed seed + b (mod 2^64); a list gives each prompt
    its own, and then a prompt's continuation is the same alone or in any batch.  A sampling setting other than the
    default without do_sample=True raises ValueError.

    prompt_lookup_num_tokens=k (1 .. 7; default None: off) generates speculatively (SpecDecoder): each step verifies the
    current token and k drafts copied from the latest longest match (up to max_matching_ngram_size tokens) of the row's
    own prompt and output, and keeps the drafts the model itself would have chosen plus one more token.  The tokens are
    the ones plain generation selects from the same logits (greedy or sampled, with the same seeds); only the step's
    arithmetic differs (other token counts take other kernel routes).  The default max_len grows by k.  spec_stats: a
    dict that receives 'accepted' (drafts taken per row) and 'steps'."""
    prompts = [torch.as_tensor(p).reshape(-1) for p in prompts]
    max_new_tokens = int(max_new_tokens)
    if not prompts:
        raise ValueError('no prompts')
    if max_new_tokens < 1:
        raise ValueError(f'max_new_tokens must be at least 1, got {max_new_tokens}')
    lens = [p.numel() for p in prompts]
    if min(lens) == 0:
        raise ValueError('empty prompt')
    spec = prompt_lookup_num_tokens is not None
    k = 0
    if spec:
        k, n_max = int(prompt_lookup_num_tokens), int(max_matching_ngram_size)
        if k != prompt_lookup_num_tokens or not 1 <= k <= 7:
            raise ValueError(f'prompt_lookup_num_tokens must be an integer in [1, 7], got {prompt_lookup_num_tokens}')
        if n_max != max_matching_ngram_size or n_max < 1:
            raise ValueError(f'max_matching_ngram_size must be an integer >= 1, got {max_matching_ngram_size}')
    max_len = max(lens) + max_new_tokens + k if max_len is None else int(max_len)
    if max(lens) + max_new_tokens + k > max_len:
        raise ValueError(f'a prompt of {max(lens)} tokens plus {max_new_tokens} new ones' +
                         (f' and {k} drafts' if k else '') + f' exceeds max_len {max_len}')
    cfg = model.config
    if cfg.model_type == 'opt' and max_len > cfg.max_position_embeddings:
        raise ValueError(f'max_len {max_len} exceeds the {cfg.max_position_embeddings} learned positions of the model')
    eos = [] if eos_token_id is None else ([int(eos_token_id)] if isinstance(eos_token_id, int) else
                                           [int(e) for e in eos_token_id])
    if not do_sample:
        for name, v, d in (('temperature', temperature, 1.0), ('top_k', top_k, 0), ('top_p', top_p, 1.0), ('seed', seed, 0)):
            if torch.is_tensor(v) or isinstance(v, (list, tuple)) or v != d:
                raise ValueError(f'{name}={v} is a sampling setting: pass do_sample=True (greedy decoding ignores it)')
    else:
        settings = _sampling_settings(len(prompts), temperature, top_k, top_p, seed)
    if spec:
        dec = SpecDecoder(model, max_len=max_len, batch=len(prompts), max_new=max_new_tokens, draft_tokens=k,
                          max_ngram=n_max, kv_dtype=kv_dtype, sampling=bool(do_sample))
    else:
        dec = PromptDecoder(model, max_len=max_len, batch=len(prompts), max_new=max_new_tokens, kv_dtype=kv_dtype,
                            sampling=bool(do_sample))
    if do_sample:
        dec.set_sampling(*settings)
    if dec.dev.type == 'cuda' and max_new_tokens > 1:                # one token comes from the prefill alone
        dec.capture()
    dec.prefill(prompts)
    eos_t = torch.tensor(eos, dtype=torch.long, device=dec.dev)
    if spec:
        return _generate_spec(dec, max_new_tokens, eos_t, spec_stats)
    n = 1
    while n < max_new_tokens:
        if eos and n % EOS_CHECK_EVERY == 0 and bool(torch.isin(dec.generated[:, :n], eos_t).any(1).all()):
            break
        dec.step()
        n += 1
    out = []
    for row in dec.generated[:, :n].cpu():
        hit = torch.isin(row, eos_t.cpu()).nonzero()
        out.append(row[:int(hit[0]) + 1] if hit.numel() else row)
    return out


def _generate_spec(dec, max_new, eos_t, stats):
    """generate()'s host loop over SpecDecoder steps: it syncs only every EOS_CHECK_EVERY steps, to stop once every row
    has max_new tokens or an EOS among its tokens."""
    steps = 0
    cols = torch.arange(dec.generated.shape[1], device=dec.dev)
    while steps < max_new - 1:
        if steps and steps % EOS_CHECK_EVERY == 0:
            done = dec.n_gen >= max_new
            if eos_t.numel():
                done = done | (torch.isin(dec.generated, eos_t) & (cols[None] < dec.n_gen[:, None])).any(1)
            if bool(done.all()):
                break
        dec.step()
        steps += 1
    if stats is not None:
        stats['accepted'] = dec.accepted.tolist()
        stats['steps'] = steps
    out = []
    for row, n in zip(dec.generated.cpu(), dec.n_gen.tolist()):
        row = row[:n]
        hit = torch.isin(row, eos_t.cpu()).nonzero()
        out.append(row[:int(hit[0]) + 1] if hit.numel() else row)
    return out
