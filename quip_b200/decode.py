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
half the cache bytes a step reads, at the cost of one e4m3 rounding of every cached key and value.
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

    def _advance(self):
        self.position.add_(1)

    # ---- the layers of the stage, three kinds of glue.  Each takes the hidden state entering the stage and returns
    # (h, pend): the residual stream and a branch output still to be added to it (None when already added).

    # csrc/glue.cu: 4 launches per layer instead of ~30 (at one token every torch elementwise op is a launch-latency-bound
    # graph node); the residual add of a branch rides on the next RMSNorm
    def _layers_fused(self, h):
        ops = self.ops
        B, nh, nkv, hd = self.batch, self.nh, self.nkv, self.hd
        pos = self._step_positions()
        h = h.contiguous()
        cos = self.cos.index_select(0, pos).expand(B, hd).contiguous()                     # one row per sequence
        sin = self.sin.index_select(0, pos).expand(B, hd).contiguous()
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
            o = self._attend(li, q.view(B, 1, nh, hd).transpose(1, 2), k.view(B, 1, nkv, hd).transpose(1, 2),
                             v.view(B, 1, nkv, hd).transpose(1, 2), mask, 1.0 / math.sqrt(hd))
            h, x = ops.rmsnorm(h, n2.weight, n2.variance_epsilon, residual=a.o_proj(o))
            gate, up = self._parallel(x, [mlp.gate_proj, mlp.up_proj])
            pend = mlp.down_proj(ops.silu_mul(gate, up))
        return h, pend

    def _layers_llama(self, h):
        B, nh, nkv, hd = self.batch, self.nh, self.nkv, self.hd
        pos = self._step_positions()
        cos = self.cos.index_select(0, pos)[:, None, None]                                 # (1 or B, 1, 1, hd)
        sin = self.sin.index_select(0, pos)[:, None, None]
        mask = self._attn_mask(pos)
        for li, layer in enumerate(self.layers):
            a = layer.self_attn
            x = layer.input_layernorm(h)
            q, k, v = self._parallel(x, [a.q_proj, a.k_proj, a.v_proj])
            q = q.view(B, 1, nh, hd).transpose(1, 2)                                       # (B, nh, 1, hd)
            k = k.view(B, 1, nkv, hd).transpose(1, 2)
            v = v.view(B, 1, nkv, hd).transpose(1, 2)
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
        B, nh, hd = self.batch, self.nh, self.hd
        mask = self._attn_mask(self._step_positions())
        for li, layer in enumerate(self.layers):
            a, before = layer.self_attn, layer.do_layer_norm_before
            x = layer.self_attn_layer_norm(h) if before else h
            q, k, v = self._parallel(x, [a.q_proj, a.k_proj, a.v_proj])
            q = (q * a.scaling).view(B, 1, nh, hd).transpose(1, 2)                         # scaled first, as the HF module does
            o = self._attend(li, q, k.view(B, 1, nh, hd).transpose(1, 2), v.view(B, 1, nh, hd).transpose(1, 2), mask, 1.0)
            h = h + a.out_proj(o)
            if not before:
                h = layer.self_attn_layer_norm(h)
            x = layer.final_layer_norm(h) if before else h
            h = h + layer.fc2(layer.activation_fn(layer.fc1(x)))
            if not before:
                h = layer.final_layer_norm(h)
        return h, None

    def _embed(self):
        """Token (and, for OPT, learned position: index position + 2) embeddings of the step: (B, 1, hidden)."""
        if self.family == 'llama':
            return self.model.model.embed_tokens(self.tokens)[:, None, :]
        d = self.model.model.decoder
        h = d.embed_tokens(self.tokens)[:, None, :]
        if d.project_in is not None:
            h = d.project_in(h)
        return h + F.embedding(self._step_positions() + d.embed_positions.offset, d.embed_positions.weight)[:, None]

    def _head(self, h, pend):
        """Final norm (fused with the pending residual add on the glue-kernel path) -> lm_head: logits (B, vocab)."""
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
        return self.model.lm_head(h)[:, 0, :]

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
      * max_new > 0: greedy selection inside the step -- tokens = argmax(logits), stored in generated[:, t] -- so a
        host loop only replays the graph;
      * kv_dtype=torch.float8_e4m3fn: k_cache / v_cache e4m3 with k_scale / v_scale (L, B, nkv, max_len) fp32, one scale
        per cached head vector.  prefill quantizes the model's keys and values into slots 0 .. P-1
        (quip_kv_quantize_fp8); the step quantizes k / v on append (quip_decode_attention_fp8) and attends over the
        quantized values of every slot, its own included.  On the CPU the same step in torch: quantize, per-row scatter,
        dequantize the cache to the compute dtype, SDPA under the mask.
    The whole model, no layer pipeline."""

    def __init__(self, model, max_len=256, batch=1, max_new=0, ops=None, kv_dtype=None):
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
        return None if self._kernel else (self._arange[None] <= pos[:, None])[:, None, None, :]     # (B, 1, 1, max_len)

    def _attend(self, li, q, k, v, mask, scale):
        B, nh, nkv, hd = self.batch, self.nh, self.nkv, self.hd
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

    def _advance(self):
        self.positions.add_(1)
        if self.max_new:
            self.tokens.copy_(self.logits.argmax(-1))
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
        max_new > 0 their argmax is the first generated token and the next step's input."""
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
                self.tokens.copy_(logits.argmax(-1))
                self.generated[:, 0].copy_(self.tokens)
                self._t.fill_(1)
                self._t_host = 1
        return logits

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


def _e4m3_quantize(x):
    """The e4m3 format of the fp8 cache (include/quip_b200.h) in torch, for the CPU step: x (..., hd) -> (e4m3 (..., hd),
    fp32 scales (...))."""
    x = x.float()
    amax = x.abs().amax(-1)
    s = torch.where(amax == 0, torch.ones_like(amax), amax / torch.full_like(amax, 448.0))       # IEEE division
    return (x / s[..., None]).to(torch.float8_e4m3fn), s


def _e4m3_dequantize(q, s, dtype):
    return (q.float() * s[..., None]).to(dtype)


EOS_CHECK_EVERY = 16


def generate(model, prompts, max_new_tokens, max_len=None, eos_token_id=None, kv_dtype=None):
    """Greedy continuations of a batch of prompts (1-D id tensors, any lengths) of a Llama or OPT model: one tensor of
    new token ids per prompt, cut after its first `eos_token_id` (an id or a list of ids).  The prompts are prefilled
    in one many-token forward; each new token is one replay of a captured PromptDecoder step on CUDA (eager on the CPU).
    max_len (default: longest prompt + max_new_tokens) is the KV cache length.  Stops early once every row has produced
    an EOS, checked every EOS_CHECK_EVERY steps.  kv_dtype=torch.float8_e4m3fn keeps the KV cache in e4m3 with per-vector
    scales (PromptDecoder); None (the default) keeps it in the model's dtype."""
    prompts = [torch.as_tensor(p).reshape(-1) for p in prompts]
    max_new_tokens = int(max_new_tokens)
    if not prompts:
        raise ValueError('no prompts')
    if max_new_tokens < 1:
        raise ValueError(f'max_new_tokens must be at least 1, got {max_new_tokens}')
    lens = [p.numel() for p in prompts]
    if min(lens) == 0:
        raise ValueError('empty prompt')
    max_len = max(lens) + max_new_tokens if max_len is None else int(max_len)
    if max(lens) + max_new_tokens > max_len:
        raise ValueError(f'a prompt of {max(lens)} tokens plus {max_new_tokens} new ones exceeds max_len {max_len}')
    cfg = model.config
    if cfg.model_type == 'opt' and max_len > cfg.max_position_embeddings:
        raise ValueError(f'max_len {max_len} exceeds the {cfg.max_position_embeddings} learned positions of the model')
    eos = [] if eos_token_id is None else ([int(eos_token_id)] if isinstance(eos_token_id, int) else
                                           [int(e) for e in eos_token_id])
    dec = PromptDecoder(model, max_len=max_len, batch=len(prompts), max_new=max_new_tokens, kv_dtype=kv_dtype)
    if dec.dev.type == 'cuda' and max_new_tokens > 1:                # one token comes from the prefill alone
        dec.capture()
    dec.prefill(prompts)
    eos_t = torch.tensor(eos, dtype=torch.long, device=dec.dev)
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
