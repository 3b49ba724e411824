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

KV_PAGE = 64                                           # slots per page of a paged KV cache (include/quip_b200.h)


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
        self._tarange = torch.arange(self.T, device=self.dev)
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

    def _attn_mask(self, pos, T=1):
        """Boolean mask over the cache slots for _attend of T tokens per row, broadcast over rows and heads."""
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

    def _tar(self, T):
        """arange(T): the offsets of a row's T tokens from its position (a step's own buffer at the step's T)."""
        return self._tarange if T == self.T else self._arange[:T]

    def _rope_rows(self, pos, T):
        """Rotary cos / sin rows of T tokens per row: (1 or B, hd) at T = 1; (B * T, hd), token i of row b at position
        pos[b] + i, otherwise."""
        if T > 1:
            pos = (pos[:, None] + self._tar(T)).reshape(-1)
            if self._pad_past_end():
                pos = pos.clamp(max=self.cos.shape[0] - 1)
        return self.cos.index_select(0, pos), self.sin.index_select(0, pos)

    def _pad_past_end(self):
        """Whether the padding tokens of a step may sit past the last position (a prefill chunk of a row that starts
        inside it): their rotary rows and learned positions are then clamped to the table.  Padding writes nothing."""
        return False

    def _advance(self):
        self.position.add_(1)

    # ---- the layers of the stage, three kinds of glue.  Each takes the hidden state entering the stage, (B, T, hidden)
    # with T tokens per row (a step's, or a prefill chunk's), and returns (h, pend): the residual stream and a branch
    # output still to be added to it (None when already added).

    def _layers(self, h):
        if self.family == 'opt':
            return self._layers_opt(h)
        if self.ops is not None:
            return self._layers_fused(h)
        return self._layers_llama(h)

    # csrc/glue.cu: 4 launches per layer instead of ~30 (at one token every torch elementwise op is a launch-latency-bound
    # graph node); the residual add of a branch rides on the next RMSNorm
    def _layers_fused(self, h):
        ops = self.ops
        (B, T), nh, nkv, hd = h.shape[:2], self.nh, self.nkv, self.hd
        pos = self._step_positions()
        h = h.contiguous()
        cos, sin = self._rope_rows(pos, T)
        cos = cos.expand(B * T, hd).contiguous()                                          # one row per token
        sin = sin.expand(B * T, hd).contiguous()
        mask = self._attn_mask(pos, T)
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
        (B, T), nh, nkv, hd = h.shape[:2], self.nh, self.nkv, self.hd
        pos = self._step_positions()
        cos, sin = self._rope_rows(pos, T)
        if T == 1:
            cos, sin = cos[:, None, None], sin[:, None, None]                              # (1 or B, 1, 1, hd)
        else:
            cos, sin = cos.view(B, 1, T, hd), sin.view(B, 1, T, hd)
        mask = self._attn_mask(pos, T)
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
        (B, T), nh, hd = h.shape[:2], self.nh, self.hd
        mask = self._attn_mask(self._step_positions(), T)
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

    def _embed(self, tokens=None):
        """Token (and, for OPT, learned position: index position + 2) embeddings of tokens (default: the step's):
        (B, T, hidden); tokens is (B,) for one token per row and (B, T) otherwise."""
        tokens = self.tokens if tokens is None else tokens
        multi = tokens.dim() == 2
        if self.family == 'llama':
            return self.model.model.embed_tokens(tokens) if multi else self.model.model.embed_tokens(tokens)[:, None, :]
        d = self.model.model.decoder
        h = d.embed_tokens(tokens) if multi else d.embed_tokens(tokens)[:, None, :]
        if d.project_in is not None:
            h = d.project_in(h)
        pos = self._step_positions()
        if multi:
            pos = pos[:, None] + self._tar(tokens.shape[1])
            if self._pad_past_end():
                pos = pos.clamp(max=self.max_len - 1)
            return h + F.embedding(pos + d.embed_positions.offset, d.embed_positions.weight)
        return h + F.embedding(pos + d.embed_positions.offset, d.embed_positions.weight)[:, None]

    def _head(self, h, pend):
        """Final norm (fused with the pending residual add on the glue-kernel path) -> lm_head: logits (B, vocab) for
        h (B, 1, hidden), or (B, T, vocab) for T > 1 tokens per row."""
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
        return logits if h.shape[1] > 1 else logits[:, 0, :]

    # one decode step of the stage on the static buffers (what the graph records)
    def _step(self):
        h = self._embed() if self.first else self.h_in
        h, pend = self._layers(h)
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
      * `prefill` fills the cache from a batch of prompts with the model's own many-token forward, or with chunk=C in
        chunks of C tokens through the step's own layer loops, appended and attended by csrc/attn_prefill.cu;
      * max_new > 0: selection inside the step -- tokens = argmax(logits), stored in generated[:, t] -- so a host loop
        only replays the graph;
      * sampling=True: the selection is quip_sample (csrc/sample.cu) over the device buffers temperature, top_k, top_p
        and seed (B each, filled by set_sampling) at step t = _t, the index of the token in generated; a row's token
        depends on its logits, settings, seed and t only.  On the CPU the same rule in torch (_sample_torch);
      * kv_dtype=torch.float8_e4m3fn: k_cache / v_cache e4m3 with k_scale / v_scale (L, B, nkv, max_len) fp32, one scale
        per cached head vector.  prefill quantizes the model's keys and values into slots 0 .. P-1
        (quip_kv_quantize_fp8); the step quantizes k / v on append (quip_decode_attention_fp8) and attends over the
        quantized values of every slot, its own included.  On the CPU the same step in torch: quantize, per-row scatter,
        dequantize the cache to the compute dtype, SDPA under the mask;
      * n_pages=N: a paged cache (include/quip_b200.h).  k_cache / v_cache are pools (L, N, nkv, 64, hd) (scales
        (L, N, nkv, 64)) and `page_table` (B, ceil(max_len / 64)) int32 on the device, shared by all layers, maps slot j
        of row b to slot j % 64 of page page_table[b, j // 64].  The table starts unmapped (-1: nothing is read or
        written there, NaN outputs) and prefill maps it to the page_table given here (default: row b's own pages
        b * max_pages ..), so rows may share pages (plan_prefix_pages).  Every attention launch takes the table; on the
        CPU reads gather pool[page_table] into the contiguous view and writes go through the same translation, so a
        paged decoder computes what a contiguous one does.  A paged cache is filled by chunked prefill only.
    The whole model, no layer pipeline."""

    def __init__(self, model, max_len=256, batch=1, max_new=0, ops=None, kv_dtype=None, sampling=False,
                 page_table=None, n_pages=None):
        if n_pages is None and page_table is not None:
            raise ValueError('a page_table needs n_pages, the size of the page pool')
        self.n_pages = None if n_pages is None else int(n_pages)
        if self.n_pages is not None and self.n_pages < 1:
            raise ValueError(f'n_pages must be at least 1, got {n_pages}')
        self.max_pages = -(-int(max_len) // KV_PAGE)
        super().__init__(model, max_len=max_len, batch=batch, ops=ops, kv_dtype=kv_dtype)
        B = self.batch
        if self.paged:
            if page_table is None:
                page_table = torch.arange(B * self.max_pages, dtype=torch.int32).view(B, self.max_pages)
            self._page_map = self._checked_page_map(page_table)
            self.page_table = torch.full((B, self.max_pages), -1, dtype=torch.int32, device=self.dev)
        self.positions = torch.zeros(B, dtype=torch.long, device=self.dev)
        self.max_new = int(max_new)
        self.generated = torch.zeros(B, max(self.max_new, 1), dtype=torch.long, device=self.dev)
        self._t = torch.zeros(1, dtype=torch.long, device=self.dev)
        self._rows = torch.arange(B, device=self.dev)
        self._pos_host = [0] * B
        self._t_host = 0
        self._kernel = self.dev.type == 'cuda'
        self._chunk = None                       # counts (B,) of the prefill chunk running the layer loops, if any
        self.sampling = bool(sampling)
        if self.sampling:
            self.temperature = torch.ones(B, dtype=torch.float32, device=self.dev)
            self.top_k = torch.zeros(B, dtype=torch.int32, device=self.dev)
            self.top_p = torch.ones(B, dtype=torch.float32, device=self.dev)
            self.seed = torch.zeros(B, dtype=torch.int64, device=self.dev)

    def _checked_page_map(self, page_table):
        """page_table as the host int32 (batch, max_pages) map prefill installs, after checking its shape and ids."""
        B = self.batch
        page_table = torch.as_tensor(page_table).to(torch.int32).cpu()
        if tuple(page_table.shape) != (B, self.max_pages):
            raise ValueError(f'page_table must be (batch {B}, ceil(max_len / {KV_PAGE}) = {self.max_pages}), got '
                             f'{tuple(page_table.shape)}')
        if bool(((page_table < -1) | (page_table >= self.n_pages)).any()):
            raise ValueError(f'page ids must lie in [0, n_pages = {self.n_pages}) or be -1 (unmapped)')
        return page_table

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
        that one would not fit).  Paged: the pools (L, n_pages, nkv, 64, hd) instead of (L, B, nkv, max_len, hd)."""
        if self.paged:
            shape = (shape[0], self.n_pages, shape[2], KV_PAGE, shape[4])
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

    @property
    def paged(self):
        return self.n_pages is not None

    def _kv_kw(self, li):
        """The cache arguments of layer li's attention launches beyond the caches: e4m3 scales, the page table."""
        kw = dict(k_scale=self.k_scale[li], v_scale=self.v_scale[li]) if self._fp8 else {}
        if self.paged:
            kw['page_table'] = self.page_table
        return kw

    def _store(self, li, rows, slots, k, v):
        """CPU: k / v (..., nkv, hd) to slots of rows (index tensors of shape ...) of layer li's cache, e4m3-quantized
        with their scales on an e4m3 cache; paged, through the page table (nothing on an unmapped page)."""
        nkv, hd = k.shape[-2:]
        rows, slots, k, v = rows.reshape(-1), slots.reshape(-1), k.reshape(-1, nkv, hd), v.reshape(-1, nkv, hd)
        if self.paged:
            page = self.page_table[rows, slots // KV_PAGE].long()
            ok = (page >= 0) & (page < self.n_pages)
            rows, slots, k, v = page[ok], (slots % KV_PAGE)[ok], k[ok], v[ok]
        for x, cache, scales in ((k, self.k_cache[li], self.k_scale), (v, self.v_cache[li], self.v_scale)):
            if self._fp8:
                xq, xs = _e4m3_quantize(x)
                cache[rows, :, slots] = xq
                scales[li][rows, :, slots] = xs
            else:
                cache[rows, :, slots] = x

    def _cached(self, li, dtype):
        """CPU: layer li's keys and values as (B, nkv, max_len, hd) in dtype (e4m3: dequantized); paged, gathered through
        the page table (an unmapped page reads page 0: such slots lie past every row's position, under the mask)."""
        out = []
        for cache, scales in ((self.k_cache[li], self.k_scale), (self.v_cache[li], self.v_scale)):
            s = None if scales is None else scales[li]
            if self.paged:
                tbl = self.page_table.long().clamp(min=0)                             # (B, max_pages)
                B, nkv, hd = tbl.shape[0], cache.shape[1], cache.shape[3]
                cache = cache[tbl].transpose(1, 2).reshape(B, nkv, -1, hd)[:, :, :self.max_len]
                if s is not None:
                    s = s[tbl].transpose(1, 2).reshape(B, nkv, -1)[:, :, :self.max_len]
            out.append(cache if s is None else _e4m3_dequantize(cache, s, dtype))
        return out

    def _step_positions(self):
        return self.positions

    def _attn_mask(self, pos, T=1):
        if self._kernel or self._chunk is not None:                                    # a chunk masks in _attend_chunk
            return None
        if T > 1:                                                                      # (B, 1, T, max_len), causal
            return (self._arange[None, None] <= (pos[:, None] + self._tar(T))[:, :, None])[:, None]
        return (self._arange[None] <= pos[:, None])[:, None, None, :]                  # (B, 1, 1, max_len)

    def _attend(self, li, q, k, v, mask, scale):
        B, nh, nkv, hd = self.batch, self.nh, self.nkv, self.hd
        if self._chunk is not None:
            return self._attend_chunk(li, q, k, v, scale)
        if q.shape[2] > 1:
            return self._attend_multi(li, q, k, v, mask, scale)
        if self._kernel:
            from . import fused
            o = fused.decode_attention(q.reshape(B, nh, hd).contiguous(), k.reshape(B, nkv, hd).contiguous(),
                                       v.reshape(B, nkv, hd).contiguous(), self.k_cache[li], self.v_cache[li],
                                       self.positions, scale, **self._kv_kw(li))
            return o.view(B, 1, nh * hd)
        self._store(li, self._rows, self.positions, k[:, :, 0], v[:, :, 0])
        kk, vv = self._cached(li, q.dtype)
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
            o = fused.extend_attention(q.transpose(1, 2).contiguous(), k.transpose(1, 2).contiguous(),
                                       v.transpose(1, 2).contiguous(), self.k_cache[li], self.v_cache[li],
                                       self.positions, scale, **self._kv_kw(li))
            return o.view(B, T, nh * hd)
        rows = self._rows[:, None].expand(B, T)
        slots = self.positions[:, None] + self._tarange                                 # (B, T)
        self._store(li, rows, slots, k.transpose(1, 2), v.transpose(1, 2))
        kk, vv = self._cached(li, q.dtype)
        if nkv != nh:
            kk = kk.repeat_interleave(nh // nkv, dim=1)
            vv = vv.repeat_interleave(nh // nkv, dim=1)
        o = F.scaled_dot_product_attention(q, kk, vv, attn_mask=mask, scale=scale)
        return o.transpose(1, 2).reshape(B, T, nh * hd)

    def _attend_chunk(self, li, q, k, v, scale):
        """_attend for a prefill chunk (q (B, nh, T, hd), k / v (B, nkv, T, hd)) with counts = self._chunk (B,): token
        i < counts[b] appended at slot positions[b] + i and attending over slots 0 .. positions[b] + i; the outputs of
        tokens i >= counts[b] are zero and nothing of theirs is written.  CUDA: quip_kv_append(_fp8), then
        quip_prefill_attention(_fp8).  CPU: per-row scatter of the counted slots, SDPA under the causal mask over the
        slots below positions[b] + counts[b].  Returns (B, T, nh * hd)."""
        (B, nh, T, hd), nkv, counts = q.shape, self.nkv, self._chunk
        if self._kernel:
            from . import fused
            kw = self._kv_kw(li)
            fused.kv_append(k.transpose(1, 2).contiguous(), v.transpose(1, 2).contiguous(), self.k_cache[li],
                            self.v_cache[li], self.positions, counts, **kw)
            o = fused.prefill_attention(q.transpose(1, 2).contiguous(), self.k_cache[li], self.v_cache[li],
                                        self.positions, counts, scale, **kw)
            return o.view(B, T, nh * hd)
        tar = self._tar(T)
        live = tar[None] < counts[:, None]                                             # (B, T)
        rows = self._rows[:, None].expand(B, T)[live]
        slots = (self.positions[:, None] + tar)[live]
        self._store(li, rows, slots, k.transpose(1, 2)[live], v.transpose(1, 2)[live])
        kk, vv = self._cached(li, q.dtype)
        seen = (self._arange[None] < (self.positions + counts)[:, None])[:, None, :, None]   # whatever lies past: not read
        kk, vv = torch.where(seen, kk, 0), torch.where(seen, vv, 0)
        if nkv != nh:
            kk = kk.repeat_interleave(nh // nkv, dim=1)
            vv = vv.repeat_interleave(nh // nkv, dim=1)
        last = self.positions[:, None] + torch.minimum(tar[None], (counts[:, None] - 1).clamp(min=0))   # (B, T)
        mask = (self._arange[None, None] <= last[:, :, None])[:, None]                 # (B, 1, T, max_len)
        o = F.scaled_dot_product_attention(q, kk, vv, attn_mask=mask, scale=scale)
        o = torch.where(live[:, None, :, None], o, 0)
        return o.transpose(1, 2).reshape(B, T, nh * hd)

    def _advance(self):
        self.positions.add_(1)
        if self.max_new:
            self._select(self.logits)
            self.generated.index_copy_(1, self._t, self.tokens[:, None])
            self._t.add_(1)

    def _capture_state(self):
        # Not the cache: a warm-up step writes slot positions[b] (clamped to max_len - 1), and a later step writes that
        # slot before it reads it.  A row clamped from max_len takes no further step: its cache is full.  A paged
        # decoder is captured before prefill maps its table (generate does so): the warm-up steps then run against an
        # unmapped table and write nothing -- with a page shared by several rows, a warm-up write to slot 0 would
        # corrupt another row's prefix.
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
        if self.paged:
            self.page_table.fill_(-1)

    def _pad_past_end(self):
        return self.paged and self._chunk is not None

    def _prefill_args(self, prompts, chunk, starts, page_table):
        """The checked arguments of a prefill: (chunk, lens, starts, host page map or None); raises before any work."""
        B = self.batch
        if len(prompts) != B:
            raise ValueError(f'{len(prompts)} prompts for a decoder of batch {B}')
        chunk = _chunk_size(chunk)
        if self.paged and chunk is None:
            raise ValueError('a paged KV cache is filled by chunked prefill: pass chunk=C')
        lens = [int(p.numel()) for p in prompts]
        if min(lens) < 1:
            raise ValueError('empty prompt')
        P = max(lens)
        if P > self.max_len:
            raise ValueError(f'a prompt of {P} tokens does not fit a cache of {self.max_len} positions')
        starts = [0] * B if starts is None else [int(x) for x in starts]
        if len(starts) != B or any(x % KV_PAGE or not 0 <= x < n for x, n in zip(starts, lens)):
            raise ValueError(f'starts must hold one multiple of {KV_PAGE} per row, below its prompt length; got {starts}')
        if any(starts) and not self.paged:
            raise ValueError('per-row prefill starts need a paged decoder (n_pages=...)')
        if page_table is not None and not self.paged:
            raise ValueError('a page_table needs a paged decoder (n_pages=...)')
        page_map = None if page_table is None else self._checked_page_map(page_table)
        return chunk, lens, starts, page_map

    def prefill(self, prompts, chunk=None, starts=None, page_table=None):
        """Fill the cache from `prompts` (B 1-D id tensors).  Returns the logits after each prompt's last token
        (B, vocab); with max_new > 0 the token selected from them (argmax, or sampled at t = 0) is the first generated
        token and the next step's input.

        chunk=None: right-padded to the longest (P), run through the model's own forward (`model.model(ids,
        attention_mask=..., use_cache=True)`, the packed linears at M = B * P), its keys and values copied (e4m3:
        quantized) to the cache slots 0 .. P-1.  Slots past a row's length hold padding; the step overwrites them in
        turn and never reads past positions[b].

        chunk=C (an int >= 1): the prompts in chunks of C tokens through the decoder's own layers, straight into the
        cache (_prefill_chunks): peak memory follows C, not P, and no fp16 copy of the cache is made.  Only slots
        0 .. len_b - 1 of row b are written.  With an e4m3 cache every token attends over the quantized keys and values
        the cache holds, its own included -- what teacher-forced decode steps compute, not the fp16 attention of
        chunk=None.

        A paged decoder maps its page table first, and takes chunk=C only (the many-token forward cannot start mid-
        prompt).  starts (one multiple of 64 per row, below its length; default 0): row b prefills from slot starts[b]
        on, its slots below read from pages other rows write (plan_prefix_pages: starts[b] = 64 * S_b over a leading run
        of S_b shared pages).  Chunks stay aligned to c0 = 0, C, 2C, ...; in a chunk row b feeds its tokens
        [max(c0, starts[b]), min(c0 + C, len_b)), the first at positions[b].  This is correct because (1) the owner of a
        page row b shares starts at or below that page, so it writes slot j of the page in the chunk holding j, the
        chunk of b's first token (starts[b] > j) or an earlier one; and (2) within a chunk, each layer's kv_append of
        every row runs before that layer's prefill_attention, so b reads the slot after it is written.

        page_table: a new page map for this prefill (checked as the constructor checks it), so one paged decoder serves
        batch after batch; default: the one given before."""
        chunk, lens, starts, page_map = self._prefill_args(prompts, chunk, starts, page_table)
        B, P = self.batch, max(lens)
        if page_map is not None:
            self._page_map = page_map
        if self.paged:
            self.page_table.copy_(self._page_map)
        ids = torch.zeros(B, P, dtype=torch.long, device=self.dev)
        for b, p in enumerate(prompts):
            ids[b, :lens[b]] = p.reshape(-1).to(self.dev)
        lens_t = torch.tensor(lens, dtype=torch.long, device=self.dev)
        with torch.no_grad():
            if chunk is None:
                attn = (torch.arange(P, device=self.dev)[None] < lens_t[:, None]).long()
                out =self.model.model(input_ids=ids, attention_mask=attn, use_cache=True)
                cache = out.past_key_values
                for li in range(len(self.layers)):
                    if self._fp8:
                        self._store_fp8(li, cache.layers[li].keys, cache.layers[li].values)
                    else:
                        self.k_cache[li, :, :, :P].copy_(cache.layers[li].keys)
                        self.v_cache[li, :, :, :P].copy_(cache.layers[li].values)
                logits = self.model.lm_head(out.last_hidden_state[self._rows, lens_t - 1])     # last real token per row
            else:
                logits = self._prefill_chunks(ids, lens, chunk, starts)
            self.positions.copy_(lens_t)
            self._pos_host = list(lens)
            if self.max_new:
                self._first_token(logits)
        return logits

    def _prefill_chunks(self, ids, lens, C, starts):
        """Chunked prefill of ids (B, P): chunk c0 feeds T = min(C, P - c0) tokens per row, row b from position
        lo_b = max(c0, starts[b]) with counts[b] = clamp(min(len_b, c0 + T) - lo_b, 0, T) tokens of its own (with every
        start 0: ids[:, c0:c0 + T] at position c0), through the embedding and layer loops of a step (packed linears at
        M = B * T; attention by _attend_chunk).  Rows with nothing to feed ride along as padding and write nothing.
        The final norm and lm_head run once, on each row's last prompt token, gathered from the chunk it falls in.
        Leaves positions at lo of the last chunk (prefill sets them)."""
        B = ids.shape[0]
        h_last = p_last = None
        for c0, T, lo, h, pend in self._chunks(ids, lens, C, starts):
            ends = [b for b in range(B) if c0 < lens[b] <= c0 + T]                     # rows whose last token is here
            if not ends:
                continue
            if h_last is None:
                h_last = h.new_empty(B, 1, h.shape[-1])
                p_last = None if pend is None else pend.new_empty(B, 1, pend.shape[-1])
            r = torch.tensor(ends, dtype=torch.long, device=self.dev)
            i = torch.tensor([lens[b] - 1 - lo[b] for b in ends], dtype=torch.long, device=self.dev)
            h_last[r, 0] = h[r, i]
            if pend is not None:
                p_last[r, 0] = pend[r, i]
        return self._head(h_last, p_last)

    def _chunks(self, ids, lens, C, starts):
        """The chunk loop of _prefill_chunks: for each chunk that feeds a token, runs the embedding and layer loops and
        yields (c0, T, lo, h, pend) -- the chunk's first position, width, each row's first fed position and the layer
        loops' output (B, T, hidden): token i of row b is position lo[b] + i (real for i < counts[b])."""
        B, P = ids.shape
        counts = torch.empty(B, dtype=torch.long, device=self.dev)
        for c0 in range(0, P, C):
            T = min(C, P - c0)
            lo = [max(c0, s) for s in starts]
            cnt = [min(max(min(n, c0 + T) - l, 0), T) for n, l in zip(lens, lo)]
            if not any(cnt):
                continue
            counts.copy_(torch.tensor(cnt, dtype=torch.long))
            if any(starts):
                lo_t = torch.tensor(lo, dtype=torch.long, device=self.dev)
                self.positions.copy_(lo_t)
                chunk_ids = ids.gather(1, (lo_t[:, None] + torch.arange(T, device=self.dev)).clamp(max=P - 1))
            else:
                self.positions.fill_(c0)
                chunk_ids = ids[:, c0:c0 + T]
            self._chunk = counts
            try:
                h, pend = self._layers(self._embed(chunk_ids))
            finally:
                self._chunk = None
            yield c0, T, lo, h, pend

    def prefill_scores(self, prompts, targets, chunk, starts=None, page_table=None):
        """Chunked prefill that scores the last n_b = len(targets[b]) positions of each prompt: position len_b - n_b + i
        of row b against targets[b][i].  Returns (logprob (N,) fp32, is_greedy (N,) bool) over the N = sum n_b scored
        tokens, row by row in order: log_softmax(logits)[target] and whether the target is the lowest index of the
        largest logit (quip_token_logprobs, csrc/logprob.cu; on the CPU its torch restatement _token_logprobs_torch).

        Arguments as prefill(chunk=C, starts, page_table); n_b may be 0 (a row that only rides along), and no scored
        position may lie below starts[b] (a row has hidden states only for the positions it feeds).  In each chunk the
        hidden states (and the pending residual) of the scored positions it holds are gathered, and the final norm and
        lm_head run on those rows only: M = the chunk's scored tokens, not B * C; no (B, P, vocab) tensor and no
        full-vocab fp32 tensor is made.  Positions are left at each row's length, as after prefill."""
        chunk, lens, starts, page_map = self._prefill_args(prompts, chunk, starts, page_table)
        if chunk is None:
            raise ValueError('prefill_scores runs chunked prefill: pass chunk=C')
        B = self.batch
        if len(targets) != B:
            raise ValueError(f'{len(targets)} target lists for a decoder of batch {B}')
        targets = [torch.as_tensor(t, dtype=torch.long).reshape(-1).cpu() for t in targets]
        n = [int(t.numel()) for t in targets]
        if any(not starts[b] <= lens[b] - n[b] for b in range(B)) or any(k < 0 for k in n):
            raise ValueError('each row scores at most its prompt length and nothing below its prefill start')
        V = self.model.lm_head.out_features
        if any(t.numel() and not (0 <= int(t.min()) and int(t.max()) < V) for t in targets):
            raise ValueError(f'targets must lie in [0, {V})')
        if page_map is not None:
            self._page_map = page_map
        if self.paged:
            self.page_table.copy_(self._page_map)
        P, N = max(lens), sum(n)
        ids = torch.zeros(B, P, dtype=torch.long, device=self.dev)
        for b, p in enumerate(prompts):
            ids[b, :lens[b]] = p.reshape(-1).to(self.dev)
        flat_t = torch.cat(targets).to(self.dev) if N else torch.zeros(0, dtype=torch.long, device=self.dev)
        logprob = torch.empty(N, dtype=torch.float32, device=self.dev)
        greedy = torch.empty(N, dtype=torch.uint8, device=self.dev)
        first = [lens[b] - n[b] for b in range(B)]
        off = [sum(n[:b]) for b in range(B)]
        with torch.no_grad():
            for c0, T, lo, h, pend in self._chunks(ids, lens, chunk, starts):
                rows, cols, dst = [], [], []
                for b in range(B):
                    j0, j1 = max(first[b], lo[b]), min(lens[b], c0 + T)          # scored positions fed in this chunk
                    for j in range(j0, j1):
                        rows.append(b)
                        cols.append(j - lo[b])
                        dst.append(off[b] + j - first[b])
                if not rows:
                    continue
                r = torch.tensor(rows, dtype=torch.long, device=self.dev)
                i = torch.tensor(cols, dtype=torch.long, device=self.dev)
                d = torch.tensor(dst, dtype=torch.long, device=self.dev)
                logits = self._head(h[r, i][:, None], None if pend is None else pend[r, i][:, None])   # (M, vocab)
                tg = flat_t[d]
                if self._kernel:
                    from . import fused
                    lp, gr = fused.token_logprobs(logits, tg, torch.empty_like(tg, dtype=torch.float32),
                                                  torch.empty_like(tg, dtype=torch.uint8))
                else:
                    lp, gr = _token_logprobs_torch(logits, tg)
                logprob[d] = lp
                greedy[d] = gr
            self.positions.copy_(torch.tensor(lens, dtype=torch.long))
            self._pos_host = list(lens)
        return logprob, greedy.bool()

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
                 sampling=False, page_table=None, n_pages=None):
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
                         sampling=sampling, page_table=page_table, n_pages=n_pages)
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

    def prefill(self, prompts, chunk=None, starts=None):
        """PromptDecoder.prefill (chunk and starts as there), plus the history: each whole prompt and its first
        generated token in hist, n_gen = 1."""
        lens = [int(torch.as_tensor(p).numel()) for p in prompts]
        if lens and max(lens) + self.max_new + self.k > self.max_len:
            raise ValueError(f'a prompt of {max(lens)} tokens, {self.max_new} new ones and {self.k} drafts exceed the '
                             f'cache of {self.max_len} positions')
        logits = super().prefill(prompts, chunk=chunk, starts=starts)
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

def _token_logprobs_torch(logits, targets):
    """The rule of quip_token_logprobs (include/quip_b200.h) in torch, for the CPU path: (fp32 log_softmax gathered at
    the targets, uint8 argmax == target), NaN and 0 for rows holding a NaN and for targets outside [0, V)."""
    x = logits.float()
    V = x.shape[-1]
    ok = (targets >= 0) & (targets < V) & ~torch.isnan(x).any(-1)
    t = targets.clamp(0, V - 1)
    lp = torch.log_softmax(x, -1).gather(-1, t[:, None])[:, 0]
    lp = torch.where(ok, lp, torch.full_like(lp, float('nan')))
    return lp, ((x.argmax(-1) == t) & ok).to(torch.uint8)


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


def plan_prefix_pages(prompts, budgets, max_pages=None):
    """Page table of a paged KV cache whose rows share their common prompt prefixes.

    prompts: 1-D id sequences; budgets: the slots row r may fill (its prompt, new tokens and drafts), >= its length.
    Page p of row r (slots 64p .. 64p + 63) is shareable when 64 (p + 1) <= len_r - 1: it is full, and the row's last
    prompt token -- whose logits start generation -- is never on it, nor is any slot decode writes.  Row r maps a
    shareable page p to the page of the first earlier row with the same tokens 0 .. 64 (p + 1) - 1 that also finds page
    p shareable; those pages form a leading run of S_r pages.  Its other pages, up to ceil(budget_r / 64), are its own.

    Returns (page_table (B, max_pages) int32 with -1 past each row's pages; max_pages defaults to the largest row's
    count), n_pages (the distinct pages), starts (64 * S_r: where row r's prefill begins)."""
    B = len(prompts)
    if len(budgets) != B:
        raise ValueError(f'{len(budgets)} budgets for {B} prompts')
    toks = [torch.as_tensor(p).reshape(-1).tolist() for p in prompts]
    if any(int(b) < len(t) or not t for b, t in zip(budgets, toks)):
        raise ValueError('every prompt must be non-empty and fit its budget')
    need = [-(-int(b) // KV_PAGE) for b in budgets]
    max_pages = max(need) if max_pages is None else int(max_pages)
    if max_pages < max(need):
        raise ValueError(f'max_pages {max_pages} is below the {max(need)} pages a row needs')
    table = torch.full((B, max_pages), -1, dtype=torch.int32)
    owner = {}                                    # (prefix node, page tokens) -> (node of the longer prefix, page id)
    n_pages, starts = 0, []
    for r, t in enumerate(toks):
        node, shared = 0, 0
        for p in range(need[r]):
            if KV_PAGE * (p + 1) <= len(t) - 1:      # shareable; once a page is the row's own, no later one is shared
                key = (node, tuple(t[KV_PAGE * p:KV_PAGE * (p + 1)]))
                if key in owner:
                    node, page = owner[key]
                    table[r, p] = page
                    shared += 1
                    continue
                owner[key] = (len(owner) + 1, n_pages)
                node = len(owner)
            table[r, p] = n_pages
            n_pages += 1
        starts.append(KV_PAGE * shared)
    return table, n_pages, starts


def _chunk_size(chunk):
    """A prefill chunk size: None (one many-token forward of the whole prompts) or an int >= 1."""
    if chunk is None:
        return None
    if isinstance(chunk, bool) or not isinstance(chunk, int) or chunk < 1:
        raise ValueError(f'the prefill chunk size must be None or an integer >= 1, got {chunk!r}')
    return chunk


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
             spec_stats=None, prefill_chunk_size=None, share_prompt_prefixes=False, num_return_sequences=1):
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
    dict that receives 'accepted' (drafts taken per row) and 'steps'.

    prefill_chunk_size=C (an int >= 1; default None: one many-token forward of the padded prompts) prefills in chunks
    of C tokens straight into the KV cache (PromptDecoder.prefill(chunk=C)): the prefill's peak memory is bounded by C
    instead of the prompt length, with no fp16 copy of the cache.  With an e4m3 cache the prompt then attends over its
    own quantized keys and values, as the decode steps do.

    share_prompt_prefixes=True keeps the KV cache in 64-slot pages (PromptDecoder(n_pages=...)) and lets prompts share
    the full pages of their common prefixes (plan_prefix_pages): a shared page is prefilled and stored once.  The pool
    holds the plan's pages, not batch * max_len slots; prefill_chunk_size defaults to 512.  The tokens are the ones of
    the unshared call up to the arithmetic of other GEMM token counts (fewer prefilled tokens per chunk).

    num_return_sequences=n > 1 (with do_sample=True: n greedy copies would be one answer) returns n samples of each
    prompt, len(prompts) * n tensors in (prompt, sample) order: by definition, what
    generate([p for p in prompts for _ in range(n)], share_prompt_prefixes=True, ...) returns -- an int seed s gives
    output row r the seed s + r, and a list setting takes one value per output row.  A prompt is prefilled once, but
    for its last partial page and last token."""
    prefill_chunk_size = _chunk_size(prefill_chunk_size)
    n_ret = num_return_sequences
    if isinstance(n_ret, bool) or int(n_ret) != n_ret or n_ret < 1:
        raise ValueError(f'num_return_sequences must be an integer >= 1, got {num_return_sequences!r}')
    n_ret = int(n_ret)
    if n_ret > 1 and not do_sample:
        raise ValueError(f'num_return_sequences={n_ret} needs do_sample=True (greedy samples would all be the same)')
    share = bool(share_prompt_prefixes) or n_ret > 1
    if share and prefill_chunk_size is None:
        prefill_chunk_size = 512
    prompts = [torch.as_tensor(p).reshape(-1) for p in prompts for _ in range(n_ret)]
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
    pages, starts = {}, None
    if share:
        table, n_pages, starts = plan_prefix_pages(prompts, [n + max_new_tokens + k for n in lens],
                                                   max_pages=-(-max_len // KV_PAGE))
        pages = dict(page_table=table, n_pages=n_pages)
    if spec:
        dec = SpecDecoder(model, max_len=max_len, batch=len(prompts), max_new=max_new_tokens, draft_tokens=k,
                          max_ngram=n_max, kv_dtype=kv_dtype, sampling=bool(do_sample), **pages)
    else:
        dec = PromptDecoder(model, max_len=max_len, batch=len(prompts), max_new=max_new_tokens, kv_dtype=kv_dtype,
                            sampling=bool(do_sample), **pages)
    if do_sample:
        dec.set_sampling(*settings)
    if dec.dev.type == 'cuda' and max_new_tokens > 1:                # one token comes from the prefill alone
        dec.capture()                                                # before prefill maps a paged table
    dec.prefill(prompts, chunk=prefill_chunk_size, starts=starts)
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


def _token_ids(name, seqs, vocab):
    """seqs as lists of Python ints, checked on the host: each non-empty, every id in [0, vocab)."""
    out = []
    for s in seqs:
        s = torch.as_tensor(s).reshape(-1).tolist() if torch.is_tensor(s) else [int(x) for x in s]
        if not s:
            raise ValueError(f'empty {name} sequence (the harness maps an empty context to [eot])')
        if min(s) < 0 or max(s) >= vocab:
            raise ValueError(f'{name}: token ids must lie in [0, vocab_size = {vocab})')
        out.append(s)
    return out


def score_windows(contexts, continuations, max_length):
    """The reference harness's request arithmetic (zeroShot/models/models_utils.py, BaseLM._loglikelihood_tokens):
    identical token sequences ctx + cont are one request (its first occurrence's split is used), ordered by descending
    length and then by the tokens; each is scored on inp = (ctx + cont)[-(max_length + 1):][:-1], whose last len(cont)
    positions predict cont.  Returns [(inp, cont, caller indices)] in that order."""
    groups = {}
    for i, (c, x) in enumerate(zip(contexts, continuations)):
        toks = tuple(c + x)
        if toks in groups:
            groups[toks][2].append(i)
        else:
            groups[toks] = (c, x, [i])
    out = []
    for toks in sorted(groups, key=lambda t: (-len(t), t)):
        c, x, idx = groups[toks]
        out.append(((c + x)[-(max_length + 1):][:-1], x, idx))
    return out


def score(model, contexts, continuations, batch_size=32, max_length=None, kv_dtype=None, prefill_chunk_size=512,
          share_prompt_prefixes=True):
    """Log-likelihoods of continuations: for each request (contexts[i], continuations[i]) (token-id sequences), the sum
    over the continuation's tokens of log p(token | the tokens before it) and whether every continuation token is the
    argmax of its logits -- the (logprob, is_greedy) of the reference harness's LM.loglikelihood, with its exact request
    arithmetic (score_windows; max_length defaults to the model's max_position_embeddings).  One (float, bool) per
    request, in the caller's order.  len(cont) >= 1 and len(ctx) >= 1 (the harness maps an empty context to [eot]).

    The requests run batch_size at a time (the last batch padded with one-token rows whose results are dropped) through
    one PromptDecoder by chunked prefill (prefill_chunk_size tokens per chunk) and PromptDecoder.prefill_scores: lm_head
    runs only at the scored positions and csrc/logprob.cu turns their fp16 logits into log-probabilities and greedy
    flags, so no (batch, length, vocab) tensor is made.  kv_dtype=torch.float8_e4m3fn keeps the cache in e4m3 as for
    generation (the context then attends over its own quantized keys and values).

    share_prompt_prefixes=True keeps the cache in 64-slot pages and plans each batch with plan_prefix_pages over
    inp[:first scored position + 1] (budget len(inp)): a full page of a common prefix that ends at or before the first
    scored position is prefilled and stored once -- a multiple-choice document's context is prefilled once for all its
    choices.  One decoder serves every batch: its page pool holds the largest batch's plan and each batch installs its
    own page table.  Results equal the unshared call's up to the rounding of other GEMM token counts.

    Every argument (token ids against the vocabulary included) is checked on the host before any work."""
    cfg = model.config
    vocab = int(cfg.vocab_size)
    if len(contexts) != len(continuations):
        raise ValueError(f'{len(contexts)} contexts for {len(continuations)} continuations')
    if not contexts:
        raise ValueError('no requests')
    ctxs = _token_ids('context', contexts, vocab)
    conts = _token_ids('continuation', continuations, vocab)
    if isinstance(batch_size, bool) or int(batch_size) != batch_size or batch_size < 1:
        raise ValueError(f'batch_size must be an integer >= 1, got {batch_size!r}')
    batch_size = int(batch_size)
    chunk = _chunk_size(prefill_chunk_size)
    if chunk is None:
        raise ValueError('score prefills in chunks: prefill_chunk_size must be an integer >= 1')
    max_length = int(cfg.max_position_embeddings) if max_length is None else max_length
    if isinstance(max_length, bool) or int(max_length) != max_length or max_length < 1:
        raise ValueError(f'max_length must be an integer >= 1, got {max_length!r}')
    max_length = int(max_length)
    if cfg.model_type == 'opt' and max_length > cfg.max_position_embeddings:
        raise ValueError(f'max_length {max_length} exceeds the {cfg.max_position_embeddings} learned positions of the model')
    if max(len(x) for x in conts) > max_length:
        raise ValueError(f'a continuation is longer than max_length {max_length}')
    if kv_dtype not in (None, torch.float16, torch.float8_e4m3fn, model.get_input_embeddings().weight.dtype):
        raise ValueError(f'kv_dtype {kv_dtype} is not supported (None, the model dtype, float16 or float8_e4m3fn)')

    reqs = score_windows(ctxs, conts, max_length)
    B = min(batch_size, len(reqs))
    max_len = len(reqs[0][0])                                     # the longest input comes first
    batches = []
    for s in range(0, len(reqs), B):
        part = reqs[s:s + B]
        inps = [torch.tensor(r[0], dtype=torch.long) for r in part] + [torch.zeros(1, dtype=torch.long)] * (B - len(part))
        tgts = [torch.tensor(r[1], dtype=torch.long) for r in part] + [torch.zeros(0, dtype=torch.long)] * (B - len(part))
        batches.append((part, inps, tgts))
    plans, n_pages = [], None
    if share_prompt_prefixes:
        for _, inps, tgts in batches:
            heads = [p[:p.numel() - t.numel() + 1] for p, t in zip(inps, tgts)]
            plans.append(plan_prefix_pages(heads, [p.numel() for p in inps], max_pages=-(-max_len // KV_PAGE)))
        n_pages = max(n for _, n, _ in plans)
    dec = PromptDecoder(model, max_len=max_len, batch=B, kv_dtype=kv_dtype, n_pages=n_pages,
                        page_table=plans[0][0] if plans else None)
    res = [None] * len(ctxs)
    for k, (part, inps, tgts) in enumerate(batches):
        kw = dict(starts=plans[k][2], page_table=plans[k][0]) if plans else {}
        lp, gr = dec.prefill_scores(inps, tgts, chunk, **kw)
        lp, gr = lp.double().cpu(), gr.cpu()
        o = 0
        for inp, cont, idx in part:
            n = len(cont)
            ans = (float(lp[o:o + n].sum()), bool(gr[o:o + n].all()))
            o += n
            for i in idx:
                res[i] = ans
    return res
