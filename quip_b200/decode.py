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
acceptance by csrc/spec.cu; `AssistedDecoder` (generate(..., assistant_model=small)) drafts them with a smaller model's
own steps inside the same graph.  `ContinuousDecoder` (generate(..., max_batch_size=n)) serves requests continuously: each
holds a decode row and its own pages only while it runs, and queued prompts join through ragged mixed steps
(csrc/attn_prefill.cu's ragged kernels), scheduled by `ContinuousSchedule`.
"""
import bisect
import collections
import heapq
import math

import torch
import torch.nn.functional as F

from .constrain import pack_automata
from .fused import PROC_BAD_LEN, PROC_MAX_BAD, PROC_MAX_EOS, TOPK_MAX_N

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
        for model in self._models():                       # sibling groups launch on side streams: not while capturing
            for mod in model.modules():
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

    def _models(self):
        """The models whose layers a step runs."""
        return [self.model]

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
      * processing=True: between the head and the selection, quip_logits_process (csrc/logits_process.cu; the rule is
        in include/quip_b200.h) applies the repetition penalty, no-repeat n-gram, bad-word and min_new_tokens
        processors in place, from device buffers filled by set_processing, over the row's history `hist` (B, max_len):
        the prompt by position (written by prefill) and each selected token (written inside the step).  On the CPU the
        same rule in torch (_process_torch).  Needs max_new >= 1;
      * constraint=True: after the processors, quip_constrain_mask (csrc/constrain.cu; the rule is in
        include/quip_b200.h) masks each row to the tokens its token-automaton state `cstate` (B,) int32 allows (-1:
        unconstrained), and after the selection quip_constrain_advance moves the state over the committed token.  The
        table and each row's start state come from set_constraint; a row restarts at its start state at its first
        generated token.  On the CPU the same rule in torch (_constrain_torch, _constrain_advance_torch).  Needs
        max_new >= 1;
      * logprobs=n (0 .. 20; default None: off, nothing allocated or launched): after the selection,
        quip_token_topk_logprobs (csrc/topk_logprobs.cu; the rule is in include/quip_b200.h) writes the raw logprob of
        each selected token, and with n >= 1 the n most likely ids and their logprobs, into lp (B, max_new), top_ids and
        top_lp (B, max_new, n) at the token's column of generated.  Raw: log_softmax of the head's fp16 logits before
        any processor or temperature; with processing=True the step first copies the rows the processors change in
        place (with constraint=True, that the mask changes).  On the CPU the same rule in torch
        (_token_topk_logprobs_torch).  Needs max_new >= 1;
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
                 page_table=None, n_pages=None, processing=False, logprobs=None, constraint=False):
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
        self.processing = bool(processing)
        if self.processing:
            if self.max_new < 1:
                raise ValueError('processing=True acts between the head and the selection: max_new must be at least 1')
            z = lambda *shape, dt=torch.long: torch.zeros(shape, dtype=dt, device=self.dev)
            self.hist, self.prompt_len = z(B, self.max_len), z(B)
            self.penalty = torch.ones(B, dtype=torch.float32, device=self.dev)
            self.ngram, self.min_new = z(B, dt=torch.int32), z(B, dt=torch.int32)
            self.proc_eos, self.bad, self.bad_len = z(0), z(0, PROC_BAD_LEN), z(0, dt=torch.int32)
        self.constrained = bool(constraint)
        if self.constrained:
            if self.max_new < 1:
                raise ValueError('constraint=True acts between the head and the selection: max_new must be at least 1')
            i32 = lambda *shape, v=0: torch.full(shape, v, dtype=torch.int32, device=self.dev)
            self.cstate, self.cstart = i32(B, v=-1), i32(B, v=-1)
            self.c_offsets, self.c_ids, self.c_next = i32(1), i32(0), i32(0)
        self.lp = self.top_ids = self.top_lp = None
        if logprobs is not None:
            if isinstance(logprobs, bool) or int(logprobs) != logprobs or not 0 <= logprobs <= TOPK_MAX_N:
                raise ValueError(f'logprobs must be None or an integer in [0, {TOPK_MAX_N}], got {logprobs!r}')
            if self.max_new < 1:
                raise ValueError('logprobs=n records the selected tokens: max_new must be at least 1')
            G, n = self.generated.shape[1], int(logprobs)
            self.lp = torch.full((B, G), float('nan'), dtype=torch.float32, device=self.dev)
            if n:
                self.top_ids = torch.full((B, G, n), -1, dtype=torch.long, device=self.dev)
                self.top_lp = torch.full((B, G, n), float('nan'), dtype=torch.float32, device=self.dev)

    def set_processing(self, repetition_penalty=1.0, no_repeat_ngram_size=0, min_new_tokens=0, bad_words_ids=None,
                       eos=()):
        """Write the logits-processor settings into the device buffers a captured step reads: repetition_penalty,
        no_repeat_ngram_size and min_new_tokens each a scalar for every row or one value per row; bad_words_ids (a list
        of non-empty id lists) and eos (ids) for the whole batch.  Once a step is captured, the number of bad words and
        of eos ids is fixed."""
        if not self.processing:
            raise ValueError('set_processing needs a PromptDecoder made with processing=True')
        B, V = self.batch, self.model.lm_head.out_features
        pen, ngram, min_new, bad, eos = _processing_settings(B, V, repetition_penalty, no_repeat_ngram_size,
                                                             min_new_tokens, bad_words_ids, eos)
        if self.graph is not None and (len(bad) != self.bad.shape[0] or len(eos) != self.proc_eos.numel()):
            raise ValueError(f'the captured step processes {self.bad.shape[0]} bad words and {self.proc_eos.numel()} '
                             f'eos ids; got {len(bad)} and {len(eos)}')
        self.penalty.copy_(torch.tensor(pen, dtype=torch.float32))
        self.ngram.copy_(torch.tensor(ngram, dtype=torch.int32))
        self.min_new.copy_(torch.tensor(min_new, dtype=torch.int32))
        if self.graph is None:
            self.proc_eos = torch.tensor(eos, dtype=torch.long, device=self.dev)
            self.bad = torch.zeros(len(bad), PROC_BAD_LEN, dtype=torch.long, device=self.dev)
            self.bad_len = torch.zeros(len(bad), dtype=torch.int32, device=self.dev)
        self.proc_eos.copy_(torch.tensor(eos, dtype=torch.long))
        pad = torch.zeros(len(bad), PROC_BAD_LEN, dtype=torch.long)
        for j, w in enumerate(bad):
            pad[j, :len(w)] = torch.tensor(w, dtype=torch.long)
        self.bad.copy_(pad)
        self.bad_len.copy_(torch.tensor([len(w) for w in bad], dtype=torch.int32))

    def _process(self, logits, last, rows=None, tokens=None):
        """The processors in place on logits (R, vocab) or (B, T, vocab), each logits row's history ending at
        hist[b, last[b]] (then, with T > 1, the drafts tokens[b, 1 ..]); rows: the decoder row of each logits row."""
        x = logits.reshape(-1, logits.shape[-1])
        T = 1 if tokens is None else tokens.shape[1]
        args = (x, T, self.hist, last, self.prompt_len, self.penalty, self.ngram, self.min_new, self.proc_eos, self.bad,
                self.bad_len)
        if self._kernel:
            from . import fused
            fused.logits_process(*args, tokens=tokens, rows=rows)
        else:
            _process_torch(*args, tokens=tokens, rows=rows)

    def set_constraint(self, offsets, ids, next, starts=None):
        """Write a packed token-automaton table (constrain.pack_automata: offsets (S + 1,), ids and next (nnz,) int32)
        into the device buffers a captured step reads and, given starts (one table state per row, -1: unconstrained),
        each row's start state.  Once a step is captured, S and nnz are fixed."""
        if not self.constrained:
            raise ValueError('set_constraint needs a PromptDecoder made with constraint=True')
        table = (offsets, ids, next)
        if self.graph is None:
            self.c_offsets, self.c_ids, self.c_next = (t.to(torch.int32).to(self.dev) for t in table)
        elif offsets.numel() != self.c_offsets.numel() or ids.numel() != self.c_ids.numel():
            raise ValueError(f'the captured step reads a table of {self.c_offsets.numel() - 1} states and '
                             f'{self.c_ids.numel()} transitions; got {offsets.numel() - 1} and {ids.numel()}')
        else:
            for dst, t in zip((self.c_offsets, self.c_ids, self.c_next), table):
                dst.copy_(t)
        if starts is not None:
            if len(starts) != self.batch:
                raise ValueError(f'{len(starts)} start states for a decoder of batch {self.batch}')
            self.cstart.copy_(torch.tensor(starts, dtype=torch.int32))
            self.cstate.copy_(self.cstart)

    def _constrain(self, logits, rows=None, tokens=None):
        """With constraint=True, the token-automaton mask in place on logits (R, vocab) or (B, T, vocab): each logits
        row at its decoder row's state cstate[b] (rows: the decoder row of each logits row), walked over the drafts
        tokens[b, 1 ..] when T > 1."""
        if not self.constrained:
            return
        x = logits.reshape(-1, logits.shape[-1])
        T = 1 if tokens is None else tokens.shape[1]
        args = (x, T, self.cstate, self.c_offsets, self.c_ids, self.c_next)
        if self._kernel:
            from . import fused
            fused.constrain_mask(*args, tokens=tokens, rows=rows)
        else:
            _constrain_torch(*args, tokens=tokens, rows=rows)

    def _constrain_advance(self, tokens, counts=None, rows=None):
        """With constraint=True, each row's state moved over the first counts[n] (default all) of the committed tokens
        (N, T) of entry n, the decoder row rows[n] (default n)."""
        if not self.constrained:
            return
        args = (self.cstate, tokens, self.c_offsets, self.c_ids, self.c_next)
        if self._kernel:
            from . import fused
            fused.constrain_advance(*args, counts=counts, rows=rows)
        else:
            _constrain_advance_torch(*args, counts=counts, rows=rows)

    def _hist_append(self, rows, tok, live=None):
        """hist[rows, positions[rows]] = tok (where live), at positions below max_len."""
        pos = self.positions[rows]
        ok = pos < self.max_len if live is None else live & (pos < self.max_len)
        col = pos.clamp(max=self.max_len - 1)
        self.hist[rows, col] = torch.where(ok, tok, self.hist[rows, col])

    def _raw(self, logits):
        """The logits the logprobs read: a copy when the processors or the mask are about to change them in place."""
        return logits.clone() if self.lp is not None and (self.processing or self.constrained) else logits

    def _logprobs(self, logits, tokens, cols, rows=None):
        """With logprobs on: the raw logprob of tokens (R,) or (B, T) and the top n of logits (R, vocab) or
        (B, T, vocab) into lp / top_ids / top_lp at column cols[b] + i ((B,), or (1,) for every row) of decoder row
        b = rows[r // T] (default r // T); nothing past the buffers' columns."""
        if self.lp is None:
            return
        T = tokens.shape[1] if tokens.dim() == 2 else 1
        args = (logits.reshape(-1, logits.shape[-1]), tokens.reshape(-1), cols, self.lp, self.top_ids, self.top_lp)
        if self._kernel:
            from . import fused
            fused.token_topk_logprobs(*args, T=T, rows=rows)
        else:
            _token_topk_logprobs_torch(*args, T=T, rows=rows)

    def _logprob_buffers(self):
        return [t for t in (self.lp, self.top_ids, self.top_lp) if t is not None]

    def _prompt_history(self, ids, lens_t):
        """A decoder that keeps a history (processing, SpecDecoder): the prompts ids (B, P) into hist[b, :len_b]; with
        processing, their lengths into prompt_len."""
        if getattr(self, 'hist', None) is not None:
            P = ids.shape[1]
            keep = torch.arange(P, device=self.dev)[None] < lens_t[:, None]
            self.hist[:, :P] = torch.where(keep, ids, self.hist[:, :P])
        if self.processing:
            self.prompt_len.copy_(lens_t)

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
        operands; CPU: per-row scatter of the T slots, SDPA under the causal mask.  Returns (B, T, nh * hd).  T is the
        step's own (q's), so one decoder may run steps of several widths (AssistedDecoder's assistant)."""
        (B, nh, T, hd), nkv = q.shape, self.nkv
        if self._kernel:
            from . import fused
            o = fused.extend_attention(q.transpose(1, 2).contiguous(), k.transpose(1, 2).contiguous(),
                                       v.transpose(1, 2).contiguous(), self.k_cache[li], self.v_cache[li],
                                       self.positions, scale, **self._kv_kw(li))
            return o.view(B, T, nh * hd)
        rows = self._rows[:, None].expand(B, T)
        slots = self.positions[:, None] + self._tar(T)                                  # (B, T)
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
        raw = self._raw(self.logits)
        if self.processing:
            self._process(self.logits, self.positions)                 # the token just fed is hist[b, positions[b]]
        self._constrain(self.logits)
        self.positions.add_(1)
        if self.max_new:
            self._select(self.logits)
            self._logprobs(raw, self.tokens, self._t)
            self.generated.index_copy_(1, self._t, self.tokens[:, None])
            if self.processing:
                self._hist_append(self._rows, self.tokens)
            self._constrain_advance(self.tokens[:, None])
            self._t.add_(1)

    def _capture_state(self):
        # Not the cache: a warm-up step writes slot positions[b] (clamped to max_len - 1), and a later step writes that
        # slot before it reads it.  A row clamped from max_len takes no further step: its cache is full.  A paged
        # decoder is captured before prefill maps its table (generate does so): the warm-up steps then run against an
        # unmapped table and write nothing -- with a page shared by several rows, a warm-up write to slot 0 would
        # corrupt another row's prefix.
        return ([self.positions, self.tokens, self._t, self.generated] + ([self.hist] if self.processing else []) +
                ([self.cstate] if self.constrained else []) + self._logprob_buffers())

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
        if self.processing:
            self.hist.zero_()
            self.prompt_len.zero_()
        if self.constrained:
            self.cstate.copy_(self.cstart)
        for t in self._logprob_buffers():
            t.fill_(-1 if t.dtype == torch.long else float('nan'))

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
            self._prompt_history(ids, lens_t)
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
        """Select the first generated token from the prefill's logits (B, vocab), at t = 0 (processed with the prompt
        as the history, masked at each row's start state)."""
        self._t.zero_()
        raw = self._raw(logits)
        if self.processing:
            self._process(logits, self.positions - 1)
        if self.constrained:
            self.cstate.copy_(self.cstart)
        self._constrain(logits)
        self._select(logits)
        self._logprobs(raw, self.tokens, self._t)
        self.generated[:, 0].copy_(self.tokens)
        if self.processing:
            self._hist_append(self._rows, self.tokens)
        self._constrain_advance(self.tokens[:, None])
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
                 sampling=False, page_table=None, n_pages=None, processing=False, logprobs=None, constraint=False):
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
                         sampling=sampling, page_table=page_table, n_pages=n_pages, processing=processing,
                         logprobs=logprobs, constraint=constraint)
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
        raw = self._raw(logits)
        if self.processing:                  # row i's history: hist[b, :positions[b] + 1], then drafts 1 .. i
            self._process(logits, self.positions, tokens=self.tokens)
        self._constrain(logits, tokens=self.tokens)                  # row i's state: walked over drafts 1 .. i
        if not self.sampling:
            self.targets.copy_(logits.argmax(-1))
        elif self._kernel:
            from . import fused
            fused.sample_at(logits, self.temperature, self.top_k, self.top_p, self.seed, self.n_gen, self.targets)
        else:
            self.targets.copy_(_sample_torch_at(logits, self.temperature, self.top_k, self.top_p, self.seed, self.n_gen))
        self._logprobs(raw, self.targets, self.n_gen)              # accepted targets: columns n_gen .. n_gen + e - 1
        n0 = self.n_gen.clone() if self.constrained else None
        if self._kernel:
            from . import fused
            fused.spec_accept(self.tokens, self.targets, self.generated, self.hist, self.positions, self.n_gen,
                              self.accepted, self.max_new)
        else:
            _spec_accept_torch(self.tokens, self.targets, self.generated, self.hist, self.positions, self.n_gen,
                               self.accepted, self.max_new)
        if self.constrained:                                       # the targets the accept appended
            self._constrain_advance(self.targets, counts=self.n_gen - n0)

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
        self.accepted.zero_()
        self._steps_host = 0
        return logits

    def _first_token(self, logits):
        self._t.zero_()
        raw = self._raw(logits)
        if self.processing:
            self._process(logits, self.positions - 1)
        if self.constrained:
            self.cstate.copy_(self.cstart)
        self._constrain(logits)
        self._select(logits, out=self._first)
        self._constrain_advance(self._first[:, None])
        self._logprobs(raw, self._first, self._t)
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


class AssistedDecoder(SpecDecoder):
    """SpecDecoder whose drafts come from a smaller model of the same vocabulary (generate(..., assistant_model=...)).

    The assistant is a PromptDecoder over `assistant` (`self.assistant`): its own KV cache (the same kv_dtype, and with
    n_pages its own pool under the same page table), its own positions.  One captured step (a round) runs, for each row
    b with c = positions[b] (the slot of its current token hist[b, c]) and g = n_gen[b]:
      1. tokens[b, 0] = hist[b, c];
      2. the assistant at T = 2 on hist[b, c - 1], hist[b, c] at its slots c - 1, c (causal extend attention); the
         logits of the second token give d_1 = select(z, t = g);
      3. for i = 1 .. k - 1, the assistant at T = 1 on d_i at slot c + i; its logits give d_(i+1) = select(z, t = g + i);
      4. tokens[b, 1 .. k] = d_1 .. d_k;
      5. SpecDecoder's verify and accept, unchanged.
    select is argmax, or with sampling the rule of quip_sample with the row's own temperature, top-k, top-p and seed at
    step t (quip_sample_at): the uniform the target draws its token g + i with.  So a draft is the target's token
    whenever the assistant's distribution puts that uniform on the same token (coupled drafts), and the tokens are the
    ones plain generation selects.  The logits processors and the token constraint act on the target's logits only;
    drafts are not pruned.

    The cache rule: at the start of every round the assistant's slots 0 .. c - 2 hold the keys and values of
    hist[b, 0 .. c - 2].  Prefill leaves c at the prompt length, so it holds from the first round.  The T = 2 step
    rewrites slot c - 1, which covers a round that accepted all k drafts (the assistant never fed the last one); slots
    past the accepted prefix hold rejected drafts and are each rewritten before anything reads them, the rule the target
    follows.  A finished row still runs the round and writes at most slot c + k - 1, inside max_len.  On the CPU the same
    round in torch (_sample_torch_at, per-row scatter and SDPA)."""

    def __init__(self, model, assistant, max_len=256, batch=1, max_new=1, draft_tokens=4, ops=None, kv_dtype=None,
                 sampling=False, page_table=None, n_pages=None, processing=False, logprobs=None, constraint=False):
        _check_assistant(model, assistant, max_len)
        super().__init__(model, max_len=max_len, batch=batch, max_new=max_new, draft_tokens=draft_tokens, ops=ops,
                         kv_dtype=kv_dtype, sampling=sampling, page_table=page_table, n_pages=n_pages,
                         processing=processing, logprobs=logprobs, constraint=constraint)
        self.assistant = PromptDecoder(assistant, max_len=self.max_len, batch=self.batch, kv_dtype=kv_dtype,
                                       page_table=page_table, n_pages=n_pages)
        self._draft_tok = torch.zeros(self.batch, 1, dtype=torch.long, device=self.dev)
        self._draft_t = torch.zeros(self.batch, dtype=torch.long, device=self.dev)

    def _models(self):
        return [self.model, self.assistant.model]

    def _assist(self, tokens):
        """The assistant on tokens (B,) or (B, T) at its slots positions[b] + i: the logits (B, vocab) of the last."""
        a = self.assistant
        h, pend = a._layers(a._embed(tokens))
        if h.shape[1] > 1:
            h, pend = h[:, -1:].contiguous(), None if pend is None else pend[:, -1:].contiguous()
        return a._head(h, pend)

    def _assist_select(self, z, i):
        """tokens[:, i + 1] = select(z, t = n_gen + i) for the assistant's logits z (B, vocab)."""
        out = self._draft_tok
        if not self.sampling:
            out.copy_(z.argmax(-1, keepdim=True))
        elif self._kernel:
            from . import fused
            torch.add(self.n_gen, i, out=self._draft_t)
            fused.sample_at(z[:, None], self.temperature, self.top_k, self.top_p, self.seed, self._draft_t, out)
        else:
            out.copy_(_sample_torch_at(z[:, None], self.temperature, self.top_k, self.top_p, self.seed, self.n_gen + i))
        self.tokens[:, i + 1:i + 2].copy_(out)

    def _draft(self):
        a, c = self.assistant, self.positions
        prev = (c - 1).clamp(min=0)           # c >= 1 after prefill; 0 only in a warm-up step before it
        pair = self.hist.gather(1, torch.stack((prev, c), 1))                           # (B, 2)
        self.tokens[:, :1].copy_(pair[:, 1:])
        a.positions.copy_(prev)
        self._assist_select(self._assist(pair), 0)
        a.positions.add_(2)
        for i in range(1, self.k):
            self._assist_select(self._assist(self.tokens[:, i]), i)
            a.positions.add_(1)

    def _capture_state(self):
        # the assistant's positions are set from the target's in every round, so the target's clamp keeps its slots
        # (c - 1 .. c + k - 1) inside the cache as well
        a = self.assistant
        return (super()._capture_state() + [a.positions, a.k_cache, a.v_cache] +
                ([a.k_scale, a.v_scale] if a._fp8 else []))

    def reset(self):
        super().reset()
        self.assistant.reset()

    def prefill(self, prompts, chunk=None, starts=None):
        """SpecDecoder.prefill, then the assistant's prefill of the same prompts (chunk and starts as given)."""
        logits = super().prefill(prompts, chunk=chunk, starts=starts)
        self.assistant.prefill(prompts, chunk=chunk, starts=starts)
        return logits


def _check_assistant(model, assistant, max_len):
    """Raise ValueError unless `assistant` can draft for `model` with a cache of max_len slots: a Llama or OPT model on
    the same device, with the same number of logits, and (OPT) learned positions for every slot."""
    cfg = getattr(assistant, 'config', None)
    if getattr(cfg, 'model_type', None) not in ('llama', 'opt'):
        raise ValueError('assistant_model must be a Llama or OPT model')
    dev, a_dev = next(iter(model.parameters())).device, next(iter(assistant.parameters())).device
    if a_dev != dev:
        raise ValueError(f'the assistant is on {a_dev}, the model on {dev}')
    if assistant.lm_head.out_features != model.lm_head.out_features:
        raise ValueError(f'the assistant has {assistant.lm_head.out_features} logits per token, the model '
                         f'{model.lm_head.out_features}: they must share the vocabulary')
    if cfg.model_type == 'opt' and int(max_len) > cfg.max_position_embeddings:
        raise ValueError(f'max_len {max_len} exceeds the {cfg.max_position_embeddings} learned positions of the '
                         'assistant')


class _Ragged:
    """The packed layout of a mixed step: S sequences over N tokens (fused.RaggedChunk `seqs`), the decoder rows they
    belong to (`rows`, host list, and `rows_t`), each sequence's first position `seq_pos` (S,), its table rows `table`
    (S, max_pages), and per token its sequence `tok_seq` and position `tok_pos` (N,)."""

    def __init__(self, seqs, rows, rows_t, seq_pos, table, tok_seq, tok_pos):
        self.seqs, self.rows, self.rows_t, self.seq_pos, self.table = seqs, rows, rows_t, seq_pos, table
        self.tok_seq, self.tok_pos = tok_seq, tok_pos


class ContinuousDecoder(PromptDecoder):
    """Paged PromptDecoder whose rows serve requests that come and go (generate(..., max_batch_size=batch)).

    Every row has its own device counters: `active` (it holds a request), `n_gen` (tokens generated), `budget` (its
    max_new_tokens) and `done` (an EOS from `eos`, or n_gen reached budget).  A row is live when active and not done.
    Two kinds of step run over the same buffers:

      * decode_step: every row feeds tokens[b] at positions[b] (quip_decode_attention_paged(_fp8)); captured once as a
        CUDA graph and used whenever no row is prefilling.  An idle row's table row is unmapped (-1), so it reads and
        writes nothing and its NaN logits still select an in-range id;
      * mixed_step (eager): the layer loops run on one packed sequence of N tokens -- one token of each decoding row and
        pieces of the prompts being prefilled -- with a per-token position (rotary rows, OPT's learned positions) and
        attention by quip_kv_append_ragged / quip_prefill_attention_ragged(_fp8).  The final norm and lm_head run only
        on the tokens that produce one: each decoding row's, and the last prompt token of each prompt that ends here.

    Selection (both kinds): argmax, or with sampling the rule of quip_sample_at at step n_gen[b] (0 for the first
    token), so a request's tokens depend on its own logits, settings and seed only.  A live row then stores its token
    in generated[b, n_gen[b]] (the column clamped into the buffer), advances positions and n_gen, and sets done.  A row
    that is not live advances nothing; a done row still rewrites its own slot positions[b] (inside its reserved pages)
    until the host retires it.  On the CPU both steps run eagerly, the ragged attention in torch (per-sequence scatter
    through the table, SDPA under each sequence's causal mask)."""

    def __init__(self, model, max_len, batch, n_pages, max_new, ops=None, kv_dtype=None, sampling=False, eos=(),
                 processing=False, logprobs=None, constraint=False):
        max_pages = -(-int(max_len) // KV_PAGE)
        super().__init__(model, max_len=max_len, batch=batch, max_new=max_new, ops=ops, kv_dtype=kv_dtype,
                         sampling=sampling, n_pages=n_pages, processing=processing, logprobs=logprobs,
                         constraint=constraint,
                         page_table=torch.full((int(batch), max_pages), -1, dtype=torch.int32))
        B, dev = self.batch, self.dev
        self.n_gen = torch.zeros(B, dtype=torch.long, device=dev)
        self.budget = torch.zeros(B, dtype=torch.long, device=dev)
        self.active = torch.zeros(B, dtype=torch.bool, device=dev)
        self.done = torch.zeros(B, dtype=torch.bool, device=dev)
        self.eos = torch.tensor([int(e) for e in eos], dtype=torch.long, device=dev)
        self._ragged = None

    # ---- per-row requests

    def admit(self, row, pages, budget, settings=None, prompt=None, proc=None, cstart=-1, start=0):
        """Give row `row` a new request: its pages (host ids, mapped from slot 0 on), its budget of new tokens, when
        sampling its (temperature, top_k, top_p, seed), with processing its prompt (the start of its history) and
        (repetition_penalty, no_repeat_ngram_size, min_new_tokens), and with constraint=True its start state in the
        table of set_constraint (-1: unconstrained).  Its prompt is then fed by mixed steps from position `start` on:
        64 S when its first S pages are shared pages that another request writes (prefix cache), so that its position
        never points into one of them."""
        tbl = torch.full((self.max_pages,), -1, dtype=torch.int32)
        tbl[:len(pages)] = torch.tensor(pages, dtype=torch.int32)
        self.page_table[row].copy_(tbl)
        self.active[row] = True
        self.done[row] = False
        self.n_gen[row] = 0
        self.budget[row] = int(budget)
        self.positions[row] = int(start)
        if self.sampling:
            t, k, p, s = settings
            self.temperature[row] = float(t)
            self.top_k[row] = int(k)
            self.top_p[row] = float(p)
            self.seed[row] = s - 2 ** 64 if s >= 2 ** 63 else s
        if self.processing:
            prompt = torch.as_tensor(prompt).reshape(-1)
            self.hist[row, :prompt.numel()] = prompt.to(self.dev)
            self.prompt_len[row] = prompt.numel()
            self.penalty[row], self.ngram[row], self.min_new[row] = float(proc[0]), int(proc[1]), int(proc[2])
        if self.constrained:
            self.cstate[row] = int(cstart)

    def retire(self, row):
        """Unmap row `row`'s pages and make it idle."""
        self.page_table[row].fill_(-1)
        self.active[row] = False

    # ---- selection and the per-row update shared by both steps

    def _choose(self, logits, rows):
        """Tokens for rows (M,) from their logits (M, vocab), each at its own step n_gen."""
        if not self.sampling:
            return logits.argmax(-1)
        args = (self.temperature[rows], self.top_k[rows], self.top_p[rows], self.seed[rows], self.n_gen[rows])
        if self._kernel:
            from . import fused
            out = torch.empty(rows.shape[0], 1, dtype=torch.long, device=self.dev)
            return fused.sample_at(logits[:, None], *args, out)[:, 0]
        return _sample_torch_at(logits[:, None], *args)[:, 0]

    def _commit(self, rows, tok):
        n = self.n_gen[rows]
        live = self.active[rows] & ~self.done[rows]
        col = n.clamp(max=self.generated.shape[1] - 1)
        self.generated[rows, col] = torch.where(live, tok, self.generated[rows, col])
        self.tokens[rows] = torch.where(live, tok, self.tokens[rows])
        n = n + live.long()
        self.n_gen[rows] = n
        self.positions[rows] = self.positions[rows] + live.long()
        if self.processing:
            self._hist_append(rows, tok, live)
        self._constrain_advance(tok[:, None], counts=live.long(), rows=rows)
        stop = (tok[:, None] == self.eos[None]).any(1) | (n >= self.budget[rows])
        self.done[rows] = self.done[rows] | (live & stop)

    def _advance(self):
        raw = self._raw(self.logits)
        if self.processing:
            self._process(self.logits, self.positions)
        self._constrain(self.logits)
        tok = self._choose(self.logits, self._rows)
        self._logprobs(raw, tok, self.n_gen)                   # a done row's column n_gen lies past its own tokens
        self._commit(self._rows, tok)

    def _capture_state(self):
        return super()._capture_state() + [self.n_gen, self.active, self.done]

    def decode_step(self):
        """One decode step of every row (a graph replay once captured); returns the logits (batch, vocab)."""
        if self.graph is None:
            with torch.no_grad():
                self._step()
        else:
            self.graph.replay()
        return self.logits

    # ---- the mixed step

    def mixed_step(self, decoding, pieces):
        """One eager step over a packed sequence: one token of each row in `decoding` (its tokens[b] at positions[b]),
        then each piece (row, ids, first, ends) -- prompt tokens ids (1-D) of that row at positions first, first + 1, ..,
        ends True when they finish the prompt, whose last token then selects the row's first generated token.  Returns
        the logits (M, vocab) of the tokens that selected one -- the decoding rows', then the ending pieces' -- or None."""
        dev = self.dev
        rows = list(decoding) + [p[0] for p in pieces]
        counts = [1] * len(decoding) + [int(p[1].numel()) for p in pieces]
        offs = [0]
        for c in counts:
            offs.append(offs[-1] + c)
        S, nd = len(rows), len(decoding)
        from . import fused
        seqs = fused.RaggedChunk(offs, dev)
        with torch.no_grad():
            rows_t = torch.tensor(rows, dtype=torch.long).to(dev)
            if pieces:
                self.positions[rows_t[nd:]] = torch.tensor([int(p[2]) for p in pieces], dtype=torch.long).to(dev)
            ids = torch.cat([torch.zeros(nd, dtype=torch.long)] +
                            [torch.as_tensor(p[1]).reshape(-1).long().cpu() for p in pieces]).to(dev)
            if nd:
                ids[:nd] = self.tokens[rows_t[:nd]]
            seq_pos = self.positions[rows_t]
            tok_seq = torch.repeat_interleave(torch.arange(S), torch.tensor(counts)).to(dev)
            tok_off = torch.cat([torch.arange(c) for c in counts]).to(dev)
            self._ragged = _Ragged(seqs, rows, rows_t, seq_pos, self.page_table[rows_t], tok_seq,
                                   seq_pos[tok_seq] + tok_off)
            try:
                h, pend = self._layers(self._embed(ids[None]))
            finally:
                self._ragged = None
            ends = [j for j, p in enumerate(pieces) if p[3]]
            out_rows = list(decoding) + [pieces[j][0] for j in ends]
            if not out_rows:
                return None
            idx = torch.tensor(list(range(nd)) + [offs[nd + j + 1] - 1 for j in ends], dtype=torch.long).to(dev)
            out_t = torch.tensor(out_rows, dtype=torch.long).to(dev)
            if ends:                              # at a prompt's last token: positions[b] is that token's, as for a step
                last = [int(pieces[j][2]) + int(pieces[j][1].numel()) - 1 for j in ends]
                self.positions[out_t[nd:]] = torch.tensor(last, dtype=torch.long).to(dev)
            logits = self._head(h[0, idx][:, None], None if pend is None else pend[0, idx][:, None])
            raw = self._raw(logits)
            if self.processing:
                self._process(logits, self.positions, rows=out_t)
            self._constrain(logits, rows=out_t)
            tok = self._choose(logits, out_t)
            self._logprobs(raw, tok, self.n_gen, rows=out_t)
            self._commit(out_t, tok)
        return logits

    def _rope_rows(self, pos, T):
        if self._ragged is None:
            return super()._rope_rows(pos, T)
        p = self._ragged.tok_pos
        return self.cos.index_select(0, p), self.sin.index_select(0, p)

    def _embed(self, tokens=None):
        if self._ragged is None or self.family == 'llama':
            return super()._embed(tokens)
        d = self.model.model.decoder                  # OPT: the learned position of every packed token
        h = d.embed_tokens(tokens)
        if d.project_in is not None:
            h = d.project_in(h)
        return h + F.embedding(self._ragged.tok_pos + d.embed_positions.offset, d.embed_positions.weight)[None]

    def _attn_mask(self, pos, T=1):
        return None if self._ragged is not None else super()._attn_mask(pos, T)

    def _attend(self, li, q, k, v, mask, scale):
        if self._ragged is None:
            return super()._attend(li, q, k, v, mask, scale)
        return self._attend_ragged(li, q, k, v, scale)

    def _attend_ragged(self, li, q, k, v, scale):
        """_attend of a mixed step: q (1, nh, N, hd), k / v (1, nkv, N, hd), token i of sequence s appended at slot
        seq_pos[s] + i of its row and attending over slots 0 .. seq_pos[s] + i.  Returns (1, N, nh * hd)."""
        rg, (nh, N, hd), nkv = self._ragged, q.shape[1:], self.nkv
        qt, kt, vt = (x[0].transpose(0, 1) for x in (q, k, v))                            # (N, heads, hd)
        if self._kernel:
            from . import fused
            kw = dict(k_scale=self.k_scale[li], v_scale=self.v_scale[li]) if self._fp8 else {}
            fused.kv_append_ragged(kt.contiguous(), vt.contiguous(), self.k_cache[li], self.v_cache[li], rg.seqs,
                                   rg.seq_pos, rg.table, **kw)
            o = fused.prefill_attention_ragged(qt.contiguous(), self.k_cache[li], self.v_cache[li], rg.seqs,
                                               rg.seq_pos, rg.table, scale, **kw)
            return o.view(1, N, nh * hd)
        self._store(li, rg.rows_t[rg.tok_seq], rg.tok_pos, kt, vt)
        kk, vv = self._cached(li, q.dtype)
        out, offs = [], rg.seqs.offsets
        for s, b in enumerate(rg.rows):
            a, e = offs[s], offs[s + 1]
            p = rg.tok_pos[a:e]
            seen = (self._arange <= p[-1])[None, :, None]                               # whatever lies past: not read
            ks, vs = torch.where(seen, kk[b], 0), torch.where(seen, vv[b], 0)
            if nkv != nh:
                ks = ks.repeat_interleave(nh // nkv, dim=0)
                vs = vs.repeat_interleave(nh // nkv, dim=0)
            mask = (self._arange[None] <= p[:, None])[None]                             # (1, count, max_len)
            o = F.scaled_dot_product_attention(q[0, :, a:e], ks, vs, attn_mask=mask, scale=scale)
            out.append(o.transpose(0, 1).reshape(e - a, nh * hd))
        return torch.cat(out)[None]


class BeamDecoder(PromptDecoder):
    """Paged PromptDecoder whose B * K rows are the K beams of B prompts (generate(..., num_beams=K)): row b * K + j is
    beam j of prompt b.  One captured step runs the layers and head, then
      * quip_beam_candidates: the top C = max(2, 1 + n_eos) * K of s = log_softmax(logits) + score per row;
      * quip_beam_select: per prompt, the top C of its K lists, the next K running beams (parents, tokens, scores and
        histories), the K finished slots and the early-stop and done flags, by the rule of include/quip_b200.h (HF's
        _beam_search);
      * positions advance for the prompts that were live, then quip_kv_beam_fork(_fp8): a beam takes its parent's table
        entries for every completed 64-slot span (those pages are never written again, so no refcount) and a copy of its
        parent's slots of the current span into its own current page.
    The first select runs on the prefill's logits (all K rows of a prompt hold the same ones; beams 1 .. K-1 start at
    -1e9).  A done prompt's rows keep stepping at a frozen position inside their own pages.  Pages are never reused and
    nothing is allocated mid-run: the pool is the plan's pages (page_table, n_plan) plus B * K scratch pages for the
    fork.  On the CPU the same step in torch (_beam_candidates_torch, _beam_select_torch, _beam_fork_torch)."""

    def __init__(self, model, max_len, n_prompts, num_beams, max_new, page_table, n_plan, budgets, eos=(),
                 length_penalty=1.0, early_stopping=False, kv_dtype=None, ops=None):
        B, K = int(n_prompts), int(num_beams)
        super().__init__(model, max_len=max_len, batch=B * K, max_new=max_new, ops=ops, kv_dtype=kv_dtype,
                         page_table=page_table, n_pages=int(n_plan) + B * K)
        dev = self.dev
        self.B, self.K, self.scratch0 = B, K, int(n_plan)
        self.C = max(2, 1 + len(eos)) * K
        self.V = model.lm_head.out_features
        self.early_stopping = early_stopping
        self.never_long = early_stopping == 'never' and length_penalty > 0
        self.eos = torch.tensor([int(e) for e in eos], dtype=torch.long, device=dev)
        self.budget = torch.tensor([int(n) for n in budgets], dtype=torch.long, device=dev)
        self.pen = torch.tensor([float(n) ** float(length_penalty) if n else 1.0 for n in range(self.max_new + 1)],
                                dtype=torch.float32, device=dev)
        z = lambda *shape, dt=torch.long: torch.zeros(shape, dtype=dt, device=dev)
        self.beam = dict(score=z(B * K, dt=torch.float32), hist=z(B, K, self.max_new), hist_tmp=z(B, K, self.max_new),
                         fin_score=z(B, K, dt=torch.float32), fin_len=z(B, K), fin_tok=z(B, K, self.max_new),
                         fin_tmp=z(B, K, self.max_new), fin_filled=z(B, K, dt=torch.uint8), heur=z(B, dt=torch.uint8),
                         done=z(B, dt=torch.uint8), tokens=self.tokens, parents=z(B * K), adv=z(B * K))
        self.cand_s = z(B * K, self.C, dt=torch.float32)
        self.cand_i = z(B * K, self.C, dt=torch.int32)
        self.table_tmp = torch.full((B * K, self.max_pages), -1, dtype=torch.int32, device=dev)
        self._init_beams()

    def _init_beams(self):
        st = self.beam
        for name in ('hist', 'fin_len', 'fin_tok', 'fin_filled', 'done', 'parents', 'adv'):
            st[name].zero_()
        st['score'].fill_(-1e9)
        st['score'][::self.K] = 0.0
        st['fin_score'].fill_(-1e9)
        st['heur'].fill_(1)

    @property
    def done(self):
        return self.beam['done']

    def _beam_step(self, logits, advance):
        st, K = self.beam, self.K
        if self._kernel:
            from . import fused
            fused.beam_candidates(logits, st['score'], K, self.C, self.cand_s, self.cand_i)
            fused.beam_select(self.cand_s, self.cand_i, self.eos, self.budget, self._t, self.pen, st, K, self.V,
                              self.early_stopping, self.never_long)
        else:
            cs, ci = _beam_candidates_torch(logits, st['score'], K, self.C)
            self.cand_s.copy_(cs)
            self.cand_i.copy_(ci)
            _beam_select_torch(self.cand_s, self.cand_i, self.eos, self.budget, self._t, self.pen, st, K, self.V,
                               self.early_stopping, self.never_long)
        if advance:
            self.positions.add_(st['adv'])
        kw = dict(k_scale=self.k_scale, v_scale=self.v_scale) if self._fp8 else {}
        if self._kernel:
            from . import fused
            fused.kv_beam_fork(self.k_cache, self.v_cache, self.page_table, self.table_tmp, st['parents'],
                               self.positions, self.scratch0, **kw)
        else:
            _beam_fork_torch(self.k_cache, self.v_cache, self.page_table, st['parents'], self.positions, **kw)
        self._t.add_(1)

    def _advance(self):
        self._beam_step(self.logits, advance=True)

    def _first_token(self, logits):
        self._t.zero_()
        self._beam_step(logits, advance=False)
        self._t_host = 1

    def _capture_state(self):
        return super()._capture_state() + [t for n, t in self.beam.items() if n != 'tokens'] + [self.page_table]

    def reset(self):
        super().reset()
        self._init_beams()

    def results(self, n_ret):
        """The n_ret best finished slots of each prompt, best first: ([new-token tensors in (prompt, rank) order],
        [their scores]), each cut after its first EOS."""
        st = self.beam
        fs, fl, ft = st['fin_score'].cpu(), st['fin_len'].cpu(), st['fin_tok'].cpu()
        eos = self.eos.cpu()
        out, scores = [], []
        for b in range(self.B):
            for k in range(n_ret):
                row = ft[b, k, :int(fl[b, k])]
                hit = torch.isin(row, eos).nonzero()
                out.append(row[:int(hit[0]) + 1] if hit.numel() else row)
                scores.append(float(fs[b, k]))
        return out, scores


def _beam_generate(model, prompts, budgets, K, eos, kv_dtype, chunk, max_len, length_penalty, early_stopping, n_ret,
                   stats):
    """generate()'s beam search: a BeamDecoder over the K copies of each prompt, planned by plan_prefix_pages (a
    prompt's full pages are prefilled and stored once), replayed until every prompt is done (read every
    EOS_CHECK_EVERY steps)."""
    B = len(prompts)
    V = model.lm_head.out_features
    if len(eos) > 3:
        raise ValueError(f'beam search takes at most 3 EOS ids, got {len(eos)}')
    C = max(2, 1 + len(eos)) * K
    if K * V < C:
        raise ValueError(f'{K} beams over a vocabulary of {V} cannot fill {C} candidates')
    rows = [p for p in prompts for _ in range(K)]
    table, n_plan, starts = plan_prefix_pages(rows, [rows[r].numel() + budgets[r // K] for r in range(B * K)],
                                              max_pages=-(-max_len // KV_PAGE))
    max_new = max(budgets)
    dec = BeamDecoder(model, max_len, B, K, max_new, table, n_plan, budgets, eos=eos, length_penalty=length_penalty,
                      early_stopping=early_stopping, kv_dtype=kv_dtype)
    if dec.dev.type == 'cuda' and max_new > 1:
        dec.capture()                                                # before prefill maps the table
    dec.prefill(rows, chunk=chunk, starts=starts)                    # and the first select, on the prefill's logits
    steps = 1
    while steps < max_new:
        if steps % EOS_CHECK_EVERY == 0 and bool(dec.done.all()):
            break
        dec.step()
        steps += 1
    out, scores = dec.results(n_ret)
    if stats is not None:
        stats['scores'] = scores
        stats['steps'] = steps
    return out


def _beam_order_key(x):
    """The order-preserving key of the beam rules (include/quip_b200.h) of fp32 x: int64, larger for larger x, -0 == +0,
    NaN lowest (0)."""
    x = torch.where(x == 0, torch.zeros_like(x), x)
    u = x.contiguous().view(torch.int32).long() & 0xFFFFFFFF
    k = torch.where(u >= 2 ** 31, ~u & 0xFFFFFFFF, u | 2 ** 31)
    return torch.where(torch.isnan(x), torch.zeros_like(k), k)


def _rank(*keys):
    """Indices sorted by keys, most significant first, each ascending; ties by position."""
    order = torch.arange(keys[0].numel())
    for k in reversed(keys):
        order = order[torch.argsort(k[order], stable=True)]
    return order


def _beam_candidates_torch(logits, scores, K, C):
    """The rule of quip_beam_candidates (include/quip_b200.h) in torch: per row, the top min(C, V) of
    s = log_softmax(fp32 logits) + score by (s descending, NaN last, lower index), as (R, C) fp32 values and int32 flat
    indices (r % K) * V + v, padded with (NaN, -1) when V < C."""
    x = logits.detach().float().cpu()
    R, V = x.shape
    s = torch.log_softmax(x, -1) + scores.detach().float().cpu()[:, None]
    s = torch.where((x.amax(-1, keepdim=True) == float('-inf')) & ~torch.isnan(x).any(-1, keepdim=True),
                    torch.full_like(s, float('-inf')), s)
    out_s = torch.full((R, C), float('nan'))
    out_i = torch.full((R, C), -1, dtype=torch.int32)
    n = min(C, V)
    for r in range(R):
        top = _rank(-_beam_order_key(s[r]))[:n]
        out_s[r, :n] = s[r, top]
        out_i[r, :n] = (top + (r % K) * V).int()
    return out_s.to(logits.device), out_i.to(logits.device)


def _beam_select_torch(cand_s, cand_i, eos, budget, step, pen, st, K, V, early_stopping, never_long):
    """The rule of quip_beam_select (include/quip_b200.h) in torch, in place on the state tensors st (fused.beam_select
    has their names and shapes)."""
    R, C = cand_s.shape
    B, t = R // K, int(step.reshape(-1)[0])
    max_new = st['hist'].shape[-1]
    NEG = torch.tensor(-1e9, dtype=torch.float32)
    zero = torch.tensor(0.0, dtype=torch.float32)
    eos_l = [int(e) for e in eos.tolist()]
    for b in range(B):
        rows = slice(b * K, (b + 1) * K)
        if bool(st['done'][b]) or not 0 <= t < max_new:
            st['parents'][rows] = torch.arange(b * K, (b + 1) * K)
            st['adv'][rows] = 0
            continue
        n, bud = t + 1, int(budget[b])
        es_, ei = cand_s[rows].reshape(-1).cpu(), cand_i[rows].reshape(-1).cpu().long()
        order = _rank(-_beam_order_key(es_), torch.where(ei < 0, 2 ** 40, ei), torch.arange(K * C))[:C]
        cs, ci = es_[order], ei[order]
        tok, par = ci % V, ci // V
        hit = torch.tensor([n >= bud or int(v) in eos_l for v in tok.tolist()])
        r = cs + torch.where(hit, NEG, zero)
        run = _rank(-_beam_order_key(r))[:K]
        old = {k: st[k][b].cpu().clone() for k in ('fin_score', 'fin_len', 'fin_tok', 'fin_filled')}
        hist_old = st['hist'][b].cpu().clone()
        full = bool(old['fin_filled'].bool().all()) and early_stopping is True
        h_ok = bool(st['heur'][b])
        did = hit & (torch.arange(C) < K)
        v = cs / pen[n].cpu()
        v = v + (NEG if full else zero)
        v = v + (zero if h_ok else NEG)
        v = v + torch.where(did, zero, NEG)
        fv = torch.cat([old['fin_score'], v])
        fsrc = _rank(-_beam_order_key(fv))[:K]
        new_hist = hist_old.clone()
        for k, i in enumerate(run.tolist()):
            new_hist[k, :t] = hist_old[int(par[i]), :t]
            new_hist[k, t] = tok[i]
        st['hist'][b] = new_hist.to(st['hist'].device)
        st['tokens'][rows] = tok[run].to(st['tokens'].device)
        st['parents'][rows] = (b * K + par[run]).to(st['parents'].device)
        st['score'][rows] = r[run].to(st['score'].device)
        st['adv'][rows] = 1
        fin_tok = torch.zeros_like(old['fin_tok'])
        fs, fl, ff = torch.empty(K), torch.empty(K, dtype=torch.long), torch.empty(K, dtype=torch.bool)
        for k, src in enumerate(fsrc.tolist()):
            fs[k] = fv[src]
            if src < K:
                fin_tok[k] = old['fin_tok'][src]
                fl[k], ff[k] = old['fin_len'][src], bool(old['fin_filled'][src])
            else:
                i = src - K
                fin_tok[k, :t] = hist_old[int(par[i]), :t]
                fin_tok[k, t] = tok[i]
                fl[k], ff[k] = n, bool(did[i])
        for name, val in (('fin_score', fs), ('fin_len', fl), ('fin_tok', fin_tok), ('fin_filled', ff)):
            st[name][b] = val.to(st[name].dtype).to(st[name].device)
        mn = fs.min()
        best = r[run[0]] / pen[min(bud, max_new) if never_long else n].cpu()
        heur = h_ok and bool((best > torch.where(ff, mn, NEG)).any())
        st['heur'][b] = int(heur)
        st['done'][b] = int(not heur or (early_stopping is True and bool(ff.all())) or bool(hit.all()))


def _beam_fork_torch(k_pool, v_pool, table, parents, lens, k_scale=None, v_scale=None):
    """The rule of quip_kv_beam_fork(_fp8) (include/quip_b200.h) in torch, in place: pools (L, n_pages, nkv, 64, hd),
    scales (L, n_pages, nkv, 64), table (R, max_pages) int32."""
    R, max_pages = table.shape
    n_pages = k_pool.shape[1]
    old = table.clone()
    moves = []
    for r in range(R):
        p, ln = int(parents[r]), int(lens[r])
        if not 0 <= p < R or p == r or not 1 <= ln <= max_pages * KV_PAGE:
            continue
        cur, ns = (ln - 1) // KV_PAGE, (ln - 1) % KV_PAGE + 1
        src = int(old[p, cur])
        data = None
        if 0 <= src < n_pages:
            data = [None if x is None else x[:, src, :, :ns].clone() for x in (k_pool, v_pool, k_scale, v_scale)]
        moves.append((r, p, cur, ns, data))
    for r, p, cur, ns, data in moves:
        table[r, :cur] = old[p, :cur]
        dst = int(old[r, cur])
        if data is None or not 0 <= dst < n_pages:
            continue
        for x, d in zip((k_pool, v_pool, k_scale, v_scale), data):
            if x is not None:
                x[:, dst, :, :ns] = d


class ContinuousSchedule:
    """The host side of continuous batching (generate(..., max_batch_size=rows)): which request holds which decoder row
    and pages, and what each step feeds.  Deterministic, and free of device work so it can be checked on its own.

      * admission: FIFO in the caller's order.  The head request is admitted when a row is free and the pool has its
        whole budget free, need = ceil((len + max_new) / 64) pages; it takes the lowest free row and the lowest free page
        ids.  Pages are reserved at admission, so nothing is allocated mid-flight and nothing is preempted;
      * steps (plan): one token of each decoding row (admitted, prompt fed, not retired), plus up to `chunk` prompt
        tokens of the rows still prefilling, taken in admission order -- a long prompt spans several steps and several
        short ones can share a step;
      * retirement (retire): the row and its pages go back to the free lists.
    A request whose budget exceeds the pool raises ValueError here, before any work.

    With `prompts` (the requests' token ids) the pool is a prefix cache of refcounted pages (generate(...,
    prefix_cache=True)).  Shareable pages (shareable_pages) are keyed as plan_prefix_pages keys them (prefix_page_key)
    in an index that lives as long as the schedule:
      * admission: the head request matches the leading run of S indexed pages of its prompt and maps them as the first
        S entries of its table row; it takes need - S pages of its own, registers its own shareable ones in the index at
        once (in flight: a request admitted later can match them), and its prefill starts at position 64 S.  It is
        admitted when a row is free and free + evictable pages cover need - S;
      * counts: a page's count is the number of held rows that map it.  retire() decrements them; a page that reaches
        0 stays in the index as cached if it is indexed, and goes back to the free list otherwise;
      * readiness: an indexed page is ready once plan() has handed out its owner's prompt through the page's last slot,
        in this step or an earlier one.  A filling row whose shared pages are not all ready gets no piece and spends none
        of the step's chunk.  Pieces run in admission order, and each layer appends a step's keys and values before any
        of its attention reads, so a sharer's piece may follow its owner's in the same step; the first filling row never
        waits, so a step with filling rows always has a piece;
      * eviction: a cached page (count 0) the head request does not match is evictable; when the free list is empty,
        the least recently released evictable page with no indexed child (lower id on ties) leaves the index and is
        reused.
    `prefilled` counts the prompt tokens plan() handed out, `shared[i]` the S of request i."""

    def __init__(self, lens, max_new, rows, n_pages, chunk, prompts=None):
        self.lens, self.max_new = [int(n) for n in lens], [int(m) for m in max_new]
        self.need = [-(-(n + m) // KV_PAGE) for n, m in zip(self.lens, self.max_new)]
        self.chunk = int(chunk)
        if max(self.need) > n_pages:
            raise ValueError(f'a request needs {max(self.need)} pages of {KV_PAGE} slots (prompt and new tokens), the '
                             f'pool holds {n_pages}')
        self.queue = collections.deque(range(len(self.lens)))
        self.free_rows = list(range(int(rows)))
        self.free_pages = list(range(int(n_pages)))
        self.req = [None] * int(rows)                # the request each row holds
        self.pages = [[] for _ in range(int(rows))]  # its table row: shared pages first
        self.fed = [0] * int(rows)                   # prompt tokens fed
        self.filling = []                            # rows still prefilling, in admission order
        self.prefilled = 0
        self.shared = [0] * len(self.lens)
        self.tokens = None
        if prompts is None:
            return
        self.tokens = [torch.as_tensor(p).reshape(-1).tolist() for p in prompts]
        if [len(t) for t in self.tokens] != self.lens:
            raise ValueError('prompts must have the lengths in lens')
        n_pages = int(n_pages)
        self.ref = [0] * n_pages                     # rows mapping each page
        self.index = {}                              # prefix_page_key -> page
        self.entry = {}                              # indexed page -> (its key, its node, parent page or -1)
        self.kids = [0] * n_pages                    # indexed pages keyed under each page's node
        self.cached = set()                          # indexed pages of count 0
        self.released = [0] * n_pages                # retire() call that cached each page
        self.ready = set()                           # indexed pages whose owner's prompt has been handed out over them
        self.wait = [[] for _ in range(int(rows))]   # each row's shared pages not yet seen ready
        self.pending = [[] for _ in range(int(rows))]  # each row's own indexed pages: (end slot, page), not yet ready
        self._nodes = self._retired = 0

    def _match(self, i):
        """The indexed pages that lead request i's prompt."""
        t, node, out = self.tokens[i], 0, []
        for p in range(shareable_pages(len(t))):
            page = self.index.get(prefix_page_key(node, t, p))
            if page is None:
                break
            out.append(page)
            node = self.entry[page][1]
        return out

    def _take(self):
        """A page for an admitted row: the lowest free one, else the evicted one."""
        if self.free_pages:
            return heapq.heappop(self.free_pages)
        p = min((self.released[q], q) for q in self.cached if not self.kids[q])[1]
        self.cached.discard(p)
        self.ready.discard(p)
        key, _, parent = self.entry.pop(p)
        del self.index[key]
        if parent >= 0:
            self.kids[parent] -= 1
        return p

    def admit(self):
        """Admit what the policy allows now: [(row, request, pages)], pages the row's table from slot 0 on."""
        out = []
        while self.queue and self.free_rows:
            i = self.queue[0]
            if self.tokens is None:
                if len(self.free_pages) < self.need[i]:
                    break
                pages = [heapq.heappop(self.free_pages) for _ in range(self.need[i])]
                r = heapq.heappop(self.free_rows)
            else:
                shared = self._match(i)
                evictable = len(self.cached) - sum(p in self.cached for p in shared)
                if len(self.free_pages) + evictable < self.need[i] - len(shared):
                    break
                r = heapq.heappop(self.free_rows)
                pages = self._map(r, i, shared)
            self.queue.popleft()
            self.req[r], self.pages[r], self.fed[r] = i, pages, KV_PAGE * self.shared[i]
            self.filling.append(r)
            out.append((r, i, pages))
        return out

    def _map(self, r, i, shared):
        """Row r's table for request i: the matched pages, then its own, whose shareable ones it registers."""
        for p in shared:
            self.ref[p] += 1
            self.cached.discard(p)
        S = len(shared)
        pages = shared + [self._take() for _ in range(self.need[i] - S)]
        for p in pages[S:]:
            self.ref[p] = 1
        parent = shared[-1] if shared else -1
        node = self.entry[parent][1] if shared else 0
        pend = []
        for p in range(S, shareable_pages(self.lens[i])):
            key = prefix_page_key(node, self.tokens[i], p)
            self._nodes += 1
            node = self._nodes
            self.index[key] = pages[p]
            self.entry[pages[p]] = (key, node, parent)
            if parent >= 0:
                self.kids[parent] += 1
            parent = pages[p]
            pend.append((KV_PAGE * (p + 1), pages[p]))
        self.shared[i] = S
        self.wait[r] = [p for p in shared if p not in self.ready]
        self.pending[r] = pend
        return pages

    def plan(self):
        """The next step: (decoding rows, pieces), a piece (row, first prompt position, count); the pieces count as fed.
        No pieces: a decode step."""
        decoding = [r for r, i in enumerate(self.req) if i is not None and r not in self.filling]
        pieces, left = [], self.chunk
        for r in self.filling:
            if not left:
                break
            if self.tokens is not None:
                self.wait[r] = [p for p in self.wait[r] if p not in self.ready]
                if self.wait[r]:
                    continue
            n = min(self.lens[self.req[r]] - self.fed[r], left)
            pieces.append((r, self.fed[r], n))
            self.fed[r] += n
            self.prefilled += n
            left -= n
            if self.tokens is not None:
                pend = self.pending[r]
                while pend and pend[0][0] <= self.fed[r]:
                    self.ready.add(pend.pop(0)[1])
        self.filling = [r for r in self.filling if self.fed[r] < self.lens[self.req[r]]]
        return decoding, pieces

    def retire(self, r):
        """Free row r and its pages; returns the request it held."""
        i = self.req[r]
        if self.tokens is None:
            for p in self.pages[r]:
                heapq.heappush(self.free_pages, p)
        else:
            self._retired += 1
            for p in self.pages[r]:
                self.ref[p] -= 1
                if self.ref[p]:
                    continue
                if p in self.entry:
                    self.cached.add(p)
                    self.released[p] = self._retired
                else:
                    heapq.heappush(self.free_pages, p)
            self.wait[r], self.pending[r] = [], []
        heapq.heappush(self.free_rows, r)
        self.req[r], self.pages[r] = None, []
        return i

    @property
    def finished(self):
        return not self.queue and all(i is None for i in self.req)


def _generate_continuous(model, prompts, max_new, eos, kv_dtype, settings, rows, kv_pages, chunk, max_len,
                         proc=None, logprobs=None, top_logprobs=0, constraint=None, prefix_cache=False):
    """generate()'s continuous path: ContinuousSchedule over a ContinuousDecoder of `rows` rows and `kv_pages` pages;
    proc: the per-prompt (penalties, ngram sizes, min_new_tokens) and the bad words of the logits processors, or None;
    constraint: the packed token automata and each prompt's start state (constrain.pack_automata), or None;
    logprobs: generate()'s dict, or None; prefix_cache: the schedule shares prompt pages (ContinuousSchedule(prompts=)).
    A request's logprob entries are read with its tokens, before its row takes the next prompt (admission resets n_gen,
    and the next request writes the same columns)."""
    lens = [p.numel() for p in prompts]
    sched = ContinuousSchedule(lens, max_new, rows, kv_pages, chunk, prompts=prompts if prefix_cache else None)
    dec = ContinuousDecoder(model, max_len, rows, kv_pages, max(max_new), kv_dtype=kv_dtype,
                            sampling=settings is not None, eos=eos, processing=proc is not None,
                            logprobs=None if logprobs is None else top_logprobs, constraint=constraint is not None)
    if proc is not None:
        dec.set_processing(bad_words_ids=proc[3] or None, eos=eos)
    if constraint is not None:
        dec.set_constraint(*constraint[:3])
    if dec.dev.type == 'cuda':
        dec.capture()                                # before any row is mapped: the warm-up steps write nothing
    out = [None] * len(prompts)
    lps = [None] * len(prompts)
    eos_c = torch.tensor(eos, dtype=torch.long)
    steps = 0
    while True:
        if sched.queue or steps % EOS_CHECK_EVERY == 0:
            held = [r for r, i in enumerate(sched.req) if i is not None]
            done = dec.done.cpu()
            fin = [r for r in held if done[r]]
            if fin:
                fin_t = torch.tensor(fin, dtype=torch.long).to(dec.dev)
                gen, n_gen = dec.generated[fin_t].cpu(), dec.n_gen[fin_t].cpu()
                cut = []
                for j, r in enumerate(fin):
                    row = gen[j, :int(n_gen[j])]
                    hit = torch.isin(row, eos_c).nonzero()
                    cut.append(row[:int(hit[0]) + 1] if hit.numel() else row)
                if logprobs is not None:
                    for r, e in zip(fin, _read_logprobs(dec, fin, cut)):
                        lps[sched.req[r]] = e
                for r, row in zip(fin, cut):
                    out[sched.retire(r)] = row
                    dec.retire(r)
            for r, i, pages in sched.admit():
                dec.admit(r, pages, max_new[i], None if settings is None else [s[i] for s in settings],
                          prompts[i], None if proc is None else [s[i] for s in proc[:3]],
                          -1 if constraint is None else constraint[3][i], start=KV_PAGE * sched.shared[i])
        if sched.finished:
            break
        decoding, pieces = sched.plan()
        if pieces:
            dec.mixed_step(decoding, [(r, prompts[sched.req[r]][lo:lo + n], lo, lo + n == lens[sched.req[r]])
                                      for r, lo, n in pieces])
        else:
            dec.decode_step()
        steps += 1
    if logprobs is not None:
        _put_logprobs(logprobs, lps)
    return out


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

def _process_torch(logits, T, hist, last, prompt_len, penalty, ngram, min_new, eos, bad, bad_len, tokens=None,
                   rows=None):
    """The rule of quip_logits_process (include/quip_b200.h) in torch, in place on logits (R, V) (fp32 on the CPU,
    fp16 on the GPU: the penalty in fp32, rounded once), one row at a time; arguments as fused.logits_process."""
    R, V = logits.shape
    B, max_len = hist.shape
    eos_l = [int(e) for e in eos.tolist()]
    bad_l = [w[:n] for w, n in zip(bad.tolist(), bad_len.tolist()) if 1 <= n <= PROC_BAD_LEN]
    bad_l = [w for w in bad_l if not (len(w) == 1 and w[0] in eos_l)]
    rows_l = None if rows is None else rows.tolist()
    hist_c, last_l, plen = hist.cpu(), last.tolist(), prompt_len.tolist()
    drafts = None if tokens is None else tokens.cpu()
    pen, ngs, mns = penalty.to(logits.device), ngram.tolist(), min_new.tolist()
    neg = torch.tensor(float('-inf'), dtype=torch.float32, device=logits.device)
    for r in range(R):
        b = r // T if rows_l is None else rows_l[r // T]
        if not 0 <= b < B or not 0 <= last_l[b] < max_len:
            continue
        i = r % T
        h = hist_c[b, :last_l[b] + 1].tolist() + ([] if i == 0 else drafts[b, 1:i + 1].tolist())
        L, n, x = len(h), ngs[b], logits[r]
        if float(penalty[b]) != 1.0:
            ids = torch.tensor(sorted({v for v in h if 0 <= v < V}), dtype=torch.long, device=logits.device)
            xs = x[ids].float()
            x[ids] = torch.where(xs < 0, xs * pen[b], xs / pen[b]).to(x.dtype)
        hard = set()
        if 1 <= n <= L:
            hard.update(h[e + n - 1] for e in range(L - n + 1) if h[e:e + n - 1] == h[L - n + 1:])
        biased = {w[-1] for w in bad_l if len(w) == 1 or (len(w) <= L and h[L - len(w) + 1:] == w[:-1])}
        if eos_l and L - plen[b] < mns[b]:
            hard.update(eos_l)
        if bad.shape[0]:                              # x + bias row: -inf at the banned tokens, +0 elsewhere
            x[x == 0] = 0
            ids = torch.tensor(sorted(v for v in biased if 0 <= v < V), dtype=torch.long, device=logits.device)
            x[ids] = (x[ids].float() + neg).to(x.dtype)
        ids = torch.tensor(sorted(v for v in hard if 0 <= v < V), dtype=torch.long, device=logits.device)
        x[ids] = float('-inf')
    return logits


def _table_walk(offsets, ids, next, s, tokens):
    """delta of include/quip_b200.h (quip_constrain_mask) over tokens from state s, on the host lists of a table."""
    for v in tokens:
        if not 0 <= s < len(offsets) - 1:
            return s
        lo = min(max(offsets[s], 0), len(ids))
        hi = min(max(offsets[s + 1], lo), len(ids))
        k = bisect.bisect_left(ids, v, lo, hi)
        s = next[k] if k < hi and ids[k] == v else s
    return s


def _constrain_torch(logits, T, state, offsets, ids, next, tokens=None, rows=None):
    """The rule of quip_constrain_mask (include/quip_b200.h) in torch, in place on logits (R, V) (fp32 on the CPU,
    fp16 on the GPU): x + (allowed ? +0 : -inf), HF's scores + mask; arguments as fused.constrain_mask."""
    R, V = logits.shape
    st, off, idl, nxl = state.tolist(), offsets.tolist(), ids.tolist(), next.tolist()
    rows_l = None if rows is None else rows.tolist()
    drafts = None if tokens is None else tokens.tolist()
    for r in range(R):
        b, i = (r // T if rows_l is None else rows_l[r // T]), r % T
        if not 0 <= b < len(st):
            continue
        s = _table_walk(off, idl, nxl, st[b], drafts[b][1:i + 1] if i else [])
        if not 0 <= s < len(off) - 1:
            continue
        lo = min(max(off[s], 0), len(idl))
        hi = min(max(off[s + 1], lo), len(idl))
        mask = torch.full((V,), float('-inf'), dtype=logits.dtype, device=logits.device)
        mask[torch.tensor([v for v in idl[lo:hi] if 0 <= v < V], dtype=torch.long, device=logits.device)] = 0
        logits[r] += mask
    return logits


def _constrain_advance_torch(state, tokens, offsets, ids, next, counts=None, rows=None):
    """The rule of quip_constrain_advance (include/quip_b200.h) in torch, in place on state; arguments as
    fused.constrain_advance."""
    N, T = tokens.shape
    st, off, idl, nxl, tok = state.tolist(), offsets.tolist(), ids.tolist(), next.tolist(), tokens.tolist()
    rows_l = None if rows is None else rows.tolist()
    cnt = None if counts is None else counts.tolist()
    for n in range(N):
        b = n if rows_l is None else rows_l[n]
        if 0 <= b < len(st):
            c = T if cnt is None else min(max(cnt[n], 0), T)
            st[b] = _table_walk(off, idl, nxl, st[b], tok[n][:c])
    state.copy_(torch.tensor(st, dtype=torch.int32))
    return state


def _processing_settings(n, V, repetition_penalty, no_repeat_ngram_size, min_new_tokens, bad_words_ids, eos):
    """Validated per-row (penalties, ngram sizes, min_new_tokens) for n rows and the call's (bad words, eos ids):
    raises ValueError on any malformed or out-of-bound value."""
    pen = [float(p) for p in _per_prompt('repetition_penalty', repetition_penalty, n)]
    if any(not (math.isfinite(p) and p > 0) for p in pen):
        raise ValueError(f'repetition_penalty must be finite and > 0, got {repetition_penalty}')
    out = [pen]
    for name, v in (('no_repeat_ngram_size', no_repeat_ngram_size), ('min_new_tokens', min_new_tokens)):
        vals = _per_prompt(name, v, n)
        if any(isinstance(x, bool) or int(x) != x or not 0 <= x < 2 ** 31 for x in vals):
            raise ValueError(f'{name} must be an integer >= 0, got {v}')
        out.append([int(x) for x in vals])
    bad = []
    if bad_words_ids is not None:
        if not isinstance(bad_words_ids, (list, tuple)) or not bad_words_ids:
            raise ValueError(f'bad_words_ids must be a non-empty list of id lists, got {bad_words_ids!r}')
        for w in bad_words_ids:
            w = w.tolist() if torch.is_tensor(w) else w
            if not isinstance(w, (list, tuple)) or not 1 <= len(w) <= PROC_BAD_LEN:
                raise ValueError(f'each bad word must be a list of 1 .. {PROC_BAD_LEN} ids, got {w!r}')
            if any(isinstance(x, bool) or int(x) != x or not 0 <= x < V for x in w):
                raise ValueError(f'bad word ids must be integers in [0, {V}), got {w!r}')
            bad.append([int(x) for x in w])
        if len(bad) > PROC_MAX_BAD:
            raise ValueError(f'at most {PROC_MAX_BAD} bad words, got {len(bad)}')
    eos = [int(e) for e in eos]
    if len(eos) > PROC_MAX_EOS:
        raise ValueError(f'the logits processors take at most {PROC_MAX_EOS} eos ids, got {len(eos)}')
    return out[0], out[1], out[2], bad, eos


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


def _token_topk_logprobs_torch(logits, tokens, cols, lp, top_ids=None, top_lp=None, T=1, rows=None):
    """The rule of quip_token_topk_logprobs (include/quip_b200.h) in torch, in place, arguments as
    fused.token_topk_logprobs; logits fp16, or fp32 on the CPU (ranked by their own values).  Each value is gathered
    from the log_softmax _token_logprobs_torch takes, so a greedy row's top value is its token's, bit for bit."""
    R, V = logits.shape
    B, G = lp.shape
    dev = lp.device
    r = torch.arange(R, device=dev)
    b = r // T if rows is None else rows.to(dev)[r // T]
    c = cols.to(dev)[b.clamp(0, B - 1) if cols.numel() == B else torch.zeros_like(b)] + r % T
    ok = (b >= 0) & (b < B) & (c >= 0) & (c < G)
    b, c = b[ok], c[ok]
    x = logits[ok.to(logits.device)]
    tok_lp, _ = _token_logprobs_torch(x, tokens[ok.to(tokens.device)])
    lp[b, c] = tok_lp.to(dev)
    if top_ids is None:
        return lp
    n, k = top_ids.shape[-1], min(top_ids.shape[-1], V)
    xf = x.float()
    ids = torch.full((x.shape[0], n), -1, dtype=torch.long, device=x.device)
    vals = torch.full((x.shape[0], n), float('nan'), dtype=torch.float32, device=x.device)
    ids[:, :k] = torch.sort(xf + 0.0, dim=-1, descending=True, stable=True).indices[:, :k]   # -0 + 0 = +0: ties by id
    vals[:, :k] = torch.log_softmax(xf, -1).gather(-1, ids[:, :k])
    nan = torch.isnan(xf).any(-1)
    ids[nan], vals[nan] = -1, float('nan')
    top_ids[b, c] = ids.to(dev)
    top_lp[b, c] = vals.to(dev)
    return lp


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


def shareable_pages(n):
    """How many leading pages of an n-token prompt other prompts may share: page p (slots 64p .. 64p + 63) when
    64 (p + 1) <= n - 1 -- it is full, and the last prompt token, whose logits start generation, is never on it, nor
    is any slot decode writes."""
    return max(int(n) - 1, 0) // KV_PAGE


def prefix_page_key(node, tokens, p):
    """The key of page p of a prompt (a list of ids) whose pages 0 .. p - 1 lead to prefix node `node` (0: the empty
    prefix): prompts share page p exactly when their tokens 0 .. 64 (p + 1) - 1 agree."""
    return node, tuple(tokens[KV_PAGE * p:KV_PAGE * (p + 1)])


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
            if p < shareable_pages(len(t)):          # once a page is the row's own, no later one is shared
                key = prefix_page_key(node, t, p)
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
             spec_stats=None, prefill_chunk_size=None, share_prompt_prefixes=False, num_return_sequences=1,
             max_batch_size=None, kv_pages=None, num_beams=1, length_penalty=1.0, early_stopping=False,
             beam_stats=None, repetition_penalty=1.0, no_repeat_ngram_size=0, min_new_tokens=0, bad_words_ids=None,
             logprobs=None, top_logprobs=0, token_constraint=None, assistant_model=None, num_assistant_tokens=None,
             prefix_cache=False):
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

    assistant_model=small (default None: off) generates with assisted drafts (AssistedDecoder): a Llama or OPT model on
    the same device with the same lm_head.out_features (packed or not; an OPT one needs learned positions for max_len)
    proposes num_assistant_tokens=k drafts per row (an integer in [1, 7]; default 4) with k cheap steps of its own, and
    the model verifies them in the same captured step, as for prompt lookup.  The assistant selects each draft by the
    row's own rule: argmax, or with do_sample the same seed and step the model draws that token with, so the returned
    tokens are the ones plain generation returns with the same arguments (on the GPU up to the rounding of other token
    counts); the assistant only changes how many tokens a step yields.  Processors and token_constraint act on the
    model's logits only, and logprobs are the model's.  The default max_len grows by k; spec_stats receives 'accepted'
    and 'steps'.  num_assistant_tokens without assistant_model, or assistant_model with prompt_lookup_num_tokens,
    num_beams > 1 or max_batch_size, raises ValueError before any work.

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
    for its last partial page and last token.

    max_new_tokens may also be a list with one value per prompt (per output row with num_return_sequences): each row is
    cut to its own budget.

    max_batch_size=n (default None: one fixed batch of every prompt) serves the prompts continuously on n decode rows
    (ContinuousDecoder, ContinuousSchedule), by this deterministic policy:
      * admission is FIFO in the caller's order: the next prompt is admitted when a row is free and the page pool has
        its whole budget free, ceil((len + max_new) / 64) pages of 64 slots, reserved at admission -- nothing is
        allocated mid-flight and nothing is preempted.  A prompt whose budget exceeds the pool raises ValueError before
        any work.  kv_pages sets the pool (default: n times the largest budget);
      * while any row is prefilling, each step is a mixed step: one token of each decoding row plus up to
        prefill_chunk_size (default 512) prompt tokens of the admitted prompts, taken in FIFO order, packed without
        padding (ragged kernels).  Otherwise a step is one replay of the captured decode step;
      * the host reads the rows' done flags after every step while prompts wait, and every EOS_CHECK_EVERY steps once
        none waits; a done row's pages go back to the pool and its row to the next prompt.
    Each prompt's tokens are those of generate([p], prefill_chunk_size=C) run alone with its own settings (an int seed
    gives prompt i the seed seed + i), up to the arithmetic of other GEMM token counts.  prompt_lookup_num_tokens,
    share_prompt_prefixes and num_return_sequences > 1 do not combine with max_batch_size.

    prefix_cache=True (with max_batch_size; default False: every request prefills its whole prompt into pages of its
    own) makes the page pool a prefix cache of refcounted pages for the length of the call (ContinuousSchedule with
    prompts): a request maps the full prompt pages before its last prompt token that an earlier request -- running or
    finished -- already holds for the same leading tokens (plan_prefix_pages' rule), prefills only the rest, and waits
    to be fed until those pages are written.  A finished request's indexed pages stay cached until the pool needs them
    (least recently released first).  For several samples of one prompt, repeat it in the list: its full prompt pages
    are prefilled once.  It combines with everything max_batch_size takes (sampling, the processors, token_constraint,
    logprobs, kv_dtype, kv_pages), and each request's tokens stay those of the prompt run alone, up to the arithmetic
    of other GEMM token counts.  A value that is not a bool, or True without max_batch_size, raises ValueError.

    num_beams=K (2 .. 16; default 1: the paths above, unchanged) runs beam search (BeamDecoder): for each prompt p the
    result is what HF's model.generate(p[None], num_beams=K, do_sample=False, max_new_tokens=n_p, length_penalty,
    early_stopping, num_return_sequences, eos_token_id) returns with the prompt alone -- transformers'
    GenerationMixin._beam_search, with ties ranked by lower index (include/quip_b200.h has the rule) -- in any batch,
    up to ties and rounding.  length_penalty (a float): a finished hypothesis of n new tokens scores
    sum log p / n ** length_penalty.  early_stopping: False (HF's heuristic), True (stop once K hypotheses are finished)
    or 'never'.  num_return_sequences=r <= K then returns the r best finished hypotheses of each prompt, best first:
    len(prompts) * r tensors in (prompt, rank) order, each cut after its first EOS.  beam_stats: a dict that receives
    'scores' (HF's sequences_scores, in the same order) and 'steps'.  At most 3 EOS ids.  The K beams of a prompt share
    its full prompt pages (prefilled once, prefill_chunk_size default 512) and fork by page-table rows; the page pool is
    fixed before any work.  do_sample, prompt_lookup_num_tokens, max_batch_size and share_prompt_prefixes do not combine
    with num_beams > 1.

    Logits processors (HF's, applied in HF's order between the head and the selection by quip_logits_process inside
    the captured step; the rule is in include/quip_b200.h): repetition_penalty (finite, > 0; 1: off), no_repeat_ngram_size
    (0: off) and min_new_tokens (0: off; needs eos_token_id), each a scalar or one value per prompt (per output row with
    num_return_sequences, as the sampling settings), and bad_words_ids, one non-empty list of at most 256 id lists of 1 ..
    16 ids in [0, vocab).  For each prompt p the result is what HF's model.generate(p[None], ...the same settings...,
    eos_token_id=...) returns with the prompt alone, in any batch; it may differ by ties and by the single fp16 rounding
    of a penalised logit on the GPU (HF processes fp32).  A sampled row is what quip_sample picks from the processed row.
    They combine with greedy and sampled decoding, num_return_sequences, share_prompt_prefixes, prefill_chunk_size,
    kv_dtype, prompt_lookup_num_tokens (the tokens stay those of plain generation) and max_batch_size; with at most 8 EOS
    ids.  Any setting other than the default with num_beams > 1 raises ValueError (HF processes the beams' log-softmax,
    which quip_beam_candidates computes itself).  With every default, nothing of this runs.

    logprobs: a dict that receives the log-probabilities of the returned tokens under the model's raw distribution --
    log_softmax of the fp16 lm_head logits, before any processor, temperature, top-k or top-p (HF's output_logits) --
    computed inside the captured step by quip_token_topk_logprobs (the rule is in include/quip_b200.h).  For output row
    i (the order of the returned list) with len_i tokens, logprobs['token'][i] is an fp32 tensor (len_i,); with
    top_logprobs=n (1 .. 20) logprobs['top_ids'][i] (int64) and logprobs['top'][i] (fp32) are (len_i, n): the n most
    likely ids at each position, by logit descending and then lower id, and their logprobs.  They are the same for
    greedy, sampled and speculative runs and combine with every path but num_beams > 1 (beam_stats has the beams'
    scores).  With logprobs=None nothing is allocated or launched; the returned tokens never change.

    token_constraint: a constrain.TokenAutomaton for every output row, or a list with one TokenAutomaton or None per
    prompt (per output row with num_return_sequences, as the sampling settings); None rows are unconstrained.  Each
    row starts at its automaton's start state at its first generated token (the prompt is not walked); inside the
    captured step, after the logits processors and before temperature, top-k and top-p, quip_constrain_mask adds -inf
    to every token its state does not allow (HF's PrefixConstrainedLogitsProcessor: scores + mask), and
    quip_constrain_advance moves the state over the tokens the step commits (the rule is in include/quip_b200.h).  For
    each prompt p the greedy result is what HF's model.generate(p[None], prefix_allowed_tokens_fn=
    a.hf_prefix_allowed_tokens_fn(len(p)), ...the same settings...) returns with the prompt alone, in any batch, up to
    ties and the fp16 rounding the processors document; a sampled row is what quip_sample picks from the masked row.
    It combines with sampling, the logits processors, prompt_lookup_num_tokens (the tokens stay those of plain
    constrained generation; drafts are not pruned), max_batch_size, share_prompt_prefixes, num_return_sequences,
    prefill_chunk_size, kv_dtype and logprobs (which stay raw).  num_beams > 1, a token id outside the vocabulary, or a
    list of the wrong length raises ValueError before any work.  With None, nothing of this is allocated or launched."""
    if logprobs is not None and not isinstance(logprobs, dict):
        raise ValueError(f'logprobs must be None or a dict that receives the results, got {type(logprobs).__name__}')
    if isinstance(top_logprobs, bool) or not isinstance(top_logprobs, int) or not 0 <= top_logprobs <= TOPK_MAX_N:
        raise ValueError(f'top_logprobs must be an integer in [0, {TOPK_MAX_N}], got {top_logprobs!r}')
    if top_logprobs and logprobs is None:
        raise ValueError('top_logprobs needs a logprobs dict to receive the results')
    n_lp = None if logprobs is None else int(top_logprobs)
    if not isinstance(prefix_cache, bool):
        raise ValueError(f'prefix_cache must be True or False, got {prefix_cache!r}')
    if prefix_cache and max_batch_size is None:
        raise ValueError('prefix_cache shares pages between the requests of continuous batching: it needs '
                         'max_batch_size')
    prefill_chunk_size = _chunk_size(prefill_chunk_size)
    n_ret = num_return_sequences
    if isinstance(n_ret, bool) or int(n_ret) != n_ret or n_ret < 1:
        raise ValueError(f'num_return_sequences must be an integer >= 1, got {num_return_sequences!r}')
    n_ret = int(n_ret)
    if isinstance(num_beams, bool) or int(num_beams) != num_beams or not 1 <= num_beams <= 16:
        raise ValueError(f'num_beams must be an integer in [1, 16], got {num_beams!r}')
    nb = int(num_beams)
    assisted = assistant_model is not None
    if num_assistant_tokens is not None and not assisted:
        raise ValueError('num_assistant_tokens sets the drafts of assisted generation: it needs assistant_model')
    if assisted:
        for name, on in (('prompt_lookup_num_tokens', prompt_lookup_num_tokens is not None), ('num_beams > 1', nb > 1),
                         ('max_batch_size', max_batch_size is not None)):
            if on:
                raise ValueError(f'{name} does not combine with assistant_model (assisted generation)')
        k_a = 4 if num_assistant_tokens is None else num_assistant_tokens
        if isinstance(k_a, bool) or not isinstance(k_a, int) or not 1 <= k_a <= 7:
            raise ValueError(f'num_assistant_tokens must be an integer in [1, 7], got {num_assistant_tokens!r}')
    if nb > 1 and logprobs is not None:
        raise ValueError('logprobs does not combine with num_beams > 1 (beam_stats has the beams\' scores)')
    if nb > 1:
        for name, on in (('do_sample', bool(do_sample)), ('prompt_lookup_num_tokens', prompt_lookup_num_tokens is not None),
                         ('max_batch_size', max_batch_size is not None), ('kv_pages', kv_pages is not None),
                         ('share_prompt_prefixes', bool(share_prompt_prefixes))):
            if on:
                raise ValueError(f'{name} does not combine with num_beams > 1 (beam search)')
        if n_ret > nb:
            raise ValueError(f'num_return_sequences={n_ret} exceeds num_beams={nb}')
        if isinstance(length_penalty, bool) or not isinstance(length_penalty, (int, float)) or \
                not math.isfinite(length_penalty):
            raise ValueError(f'length_penalty must be a finite number, got {length_penalty!r}')
        if not (early_stopping is True or early_stopping is False or early_stopping == 'never'):
            raise ValueError(f"early_stopping must be False, True or 'never', got {early_stopping!r}")
    elif n_ret > 1 and not do_sample:
        raise ValueError(f'num_return_sequences={n_ret} needs do_sample=True (greedy samples would all be the same)')
    share = bool(share_prompt_prefixes) or (n_ret > 1 and nb == 1)
    if (share or nb > 1) and prefill_chunk_size is None:
        prefill_chunk_size = 512
    prompts = [torch.as_tensor(p).reshape(-1) for p in prompts for _ in range(n_ret if nb == 1 else 1)]
    if not prompts:
        raise ValueError('no prompts')
    budgets = _per_prompt('max_new_tokens', max_new_tokens, len(prompts))
    if any(isinstance(m, bool) or int(m) < 1 for m in budgets):
        raise ValueError(f'max_new_tokens must be at least 1, got {max_new_tokens}')
    budgets = [int(m) for m in budgets]
    max_new_tokens = max(budgets)
    lens = [p.numel() for p in prompts]
    if min(lens) == 0:
        raise ValueError('empty prompt')
    if max_batch_size is not None:
        if isinstance(max_batch_size, bool) or int(max_batch_size) != max_batch_size or max_batch_size < 1:
            raise ValueError(f'max_batch_size must be an integer >= 1, got {max_batch_size!r}')
        for name, on in (('prompt_lookup_num_tokens', prompt_lookup_num_tokens is not None),
                         ('share_prompt_prefixes', bool(share_prompt_prefixes)), ('num_return_sequences', n_ret > 1)):
            if on:
                raise ValueError(f'{name} does not combine with max_batch_size (continuous batching)')
    elif kv_pages is not None:
        raise ValueError('kv_pages sizes the page pool of continuous batching: it needs max_batch_size')
    spec = prompt_lookup_num_tokens is not None
    k = 0
    if spec:
        k, n_max = int(prompt_lookup_num_tokens), int(max_matching_ngram_size)
        if k != prompt_lookup_num_tokens or not 1 <= k <= 7:
            raise ValueError(f'prompt_lookup_num_tokens must be an integer in [1, 7], got {prompt_lookup_num_tokens}')
        if n_max != max_matching_ngram_size or n_max < 1:
            raise ValueError(f'max_matching_ngram_size must be an integer >= 1, got {max_matching_ngram_size}')
    if assisted:
        k = k_a
    # a fixed batch steps every row max(budgets) times; continuous batching steps each row to its own budget
    n, m = (max(zip(lens, budgets), key=sum) if max_batch_size is not None else (max(lens), max_new_tokens))
    max_len = n + m + k if max_len is None else int(max_len)
    if n + m + k > max_len:
        raise ValueError(f'a prompt of {n} tokens plus {m} new ones' +
                         (f' and {k} drafts' if k else '') + f' exceeds max_len {max_len}')
    cfg = model.config
    if cfg.model_type == 'opt' and max_len > cfg.max_position_embeddings:
        raise ValueError(f'max_len {max_len} exceeds the {cfg.max_position_embeddings} learned positions of the model')
    if assisted:
        _check_assistant(model, assistant_model, max_len)
    eos =[] if eos_token_id is None else ([int(eos_token_id)] if isinstance(eos_token_id, int) else
                                           [int(e) for e in eos_token_id])
    if not do_sample:
        for name, v, d in (('temperature', temperature, 1.0), ('top_k', top_k, 0), ('top_p', top_p, 1.0), ('seed', seed, 0)):
            if torch.is_tensor(v) or isinstance(v, (list, tuple)) or v != d:
                raise ValueError(f'{name}={v} is a sampling setting: pass do_sample=True (greedy decoding ignores it)')
    else:
        settings = _sampling_settings(len(prompts), temperature, top_k, top_p, seed)
    pen, ngram, min_new, bad, _ = _processing_settings(len(prompts), model.lm_head.out_features, repetition_penalty,
                                                       no_repeat_ngram_size, min_new_tokens, bad_words_ids, ())
    proc = (pen, ngram, min_new, bad) if (any(p != 1.0 for p in pen) or any(ngram) or any(min_new) or
                                          bad_words_ids is not None) else None
    if proc is not None:
        if nb > 1:
            raise ValueError('repetition_penalty, no_repeat_ngram_size, min_new_tokens and bad_words_ids do not combine '
                             'with num_beams > 1 (beam search)')
        if any(min_new) and not eos:
            raise ValueError('min_new_tokens bans the EOS ids: it needs eos_token_id')
        if len(eos) > PROC_MAX_EOS:
            raise ValueError(f'the logits processors take at most {PROC_MAX_EOS} eos ids, got {len(eos)}')
    constraint = None
    if token_constraint is not None:
        automata = _per_prompt('token_constraint', token_constraint, len(prompts))
        constraint = pack_automata(automata, model.lm_head.out_features)
        if all(s < 0 for s in constraint[3]):
            constraint = None
        elif nb > 1:
            raise ValueError('token_constraint does not combine with num_beams > 1 (beam search)')
    if nb > 1:
        return _beam_generate(model, prompts, budgets, nb, eos, kv_dtype, prefill_chunk_size, max_len,
                              float(length_penalty), early_stopping, n_ret, beam_stats)
    if max_batch_size is not None:
        rows = min(int(max_batch_size), len(prompts))
        need = max(-(-(n + m) // KV_PAGE) for n, m in zip(lens, budgets))
        kv_pages = rows * need if kv_pages is None else kv_pages
        if isinstance(kv_pages, bool) or int(kv_pages) != kv_pages or kv_pages < 1:
            raise ValueError(f'kv_pages must be an integer >= 1, got {kv_pages!r}')
        return _generate_continuous(model, prompts, budgets, eos, kv_dtype, settings if do_sample else None, rows,
                                    int(kv_pages), 512 if prefill_chunk_size is None else prefill_chunk_size, max_len,
                                    proc, logprobs, int(top_logprobs), constraint, prefix_cache)
    pages, starts = {}, None
    if share:
        table, n_pages, starts = plan_prefix_pages(prompts, [n + m + k for n, m in zip(lens, budgets)],
                                                   max_pages=-(-max_len // KV_PAGE))
        pages = dict(page_table=table, n_pages=n_pages)
    if proc is not None:
        pages['processing'] = True
    if n_lp is not None:
        pages['logprobs'] = n_lp
    if constraint is not None:
        pages['constraint'] = True
    if assisted:
        dec = AssistedDecoder(model, assistant_model, max_len=max_len, batch=len(prompts), max_new=max_new_tokens,
                              draft_tokens=k, kv_dtype=kv_dtype, sampling=bool(do_sample), **pages)
    elif spec:
        dec = SpecDecoder(model, max_len=max_len, batch=len(prompts), max_new=max_new_tokens, draft_tokens=k,
                          max_ngram=n_max, kv_dtype=kv_dtype, sampling=bool(do_sample), **pages)
    else:
        dec = PromptDecoder(model, max_len=max_len, batch=len(prompts), max_new=max_new_tokens, kv_dtype=kv_dtype,
                            sampling=bool(do_sample), **pages)
    if do_sample:
        dec.set_sampling(*settings)
    if proc is not None:
        dec.set_processing(*proc[:3], proc[3] or None, eos)
    if constraint is not None:
        dec.set_constraint(*constraint)
    if dec.dev.type == 'cuda' and max_new_tokens > 1:                # one token comes from the prefill alone
        dec.capture()                                                # before prefill maps a paged table
    dec.prefill(prompts, chunk=prefill_chunk_size, starts=starts)
    eos_t = torch.tensor(eos, dtype=torch.long, device=dec.dev)
    if spec or assisted:
        return _generate_spec(dec, budgets, eos_t, spec_stats, logprobs)
    n = 1
    while n < max_new_tokens:
        if (eos or min(budgets) < max_new_tokens) and n % EOS_CHECK_EVERY == 0:
            fin = torch.tensor([m <= n for m in budgets], device=dec.dev)     # a row past its own budget is finished
            if eos:
                fin = fin | torch.isin(dec.generated[:, :n], eos_t).any(1)
            if bool(fin.all()):
                break
        dec.step()
        n += 1
    out = []
    for row, m in zip(dec.generated[:, :n].cpu(), budgets):
        row = row[:m]
        hit = torch.isin(row, eos_t.cpu()).nonzero()
        out.append(row[:int(hit[0]) + 1] if hit.numel() else row)
    if logprobs is not None:
        _put_logprobs(logprobs, _read_logprobs(dec, list(range(len(out))), out))
    return out


def _read_logprobs(dec, rows, outs):
    """The logprob entries of decoder rows `rows`, each cut to the length of its returned tokens outs[i]:
    [(token (len,), top_ids (len, n) or None, top (len, n) or None)]."""
    idx = torch.tensor(rows, dtype=torch.long, device=dec.dev)
    bufs = [None if t is None else t[idx].cpu() for t in (dec.lp, dec.top_ids, dec.top_lp)]
    return [tuple(None if t is None else t[j, :o.numel()] for t in bufs) for j, o in enumerate(outs)]


def _put_logprobs(dest, entries):
    """generate()'s logprobs dict from the entries of _read_logprobs, in output order."""
    dest['token'] = [e[0] for e in entries]
    if entries[0][1] is not None:
        dest['top_ids'] = [e[1] for e in entries]
        dest['top'] = [e[2] for e in entries]


def _generate_spec(dec, budgets, eos_t, stats, logprobs=None):
    """generate()'s host loop over SpecDecoder steps: it syncs only every EOS_CHECK_EVERY steps, to stop once every row
    has max_new tokens or an EOS among its tokens.  Each row is cut to its own budget."""
    max_new = max(budgets)
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
    for row, n, m in zip(dec.generated.cpu(), dec.n_gen.tolist(), budgets):
        row = row[:min(n, m)]
        hit = torch.isin(row, eos_t.cpu()).nonzero()
        out.append(row[:int(hit[0]) + 1] if hit.numel() else row)
    if logprobs is not None:
        _put_logprobs(logprobs, _read_logprobs(dec, list(range(len(out))), out))
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
