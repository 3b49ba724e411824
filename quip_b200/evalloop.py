"""Per-layer perplexity evaluation loop shared by opt.py and llama.py.

Keeps the reference's structure (opt.py:193-299, llama.py:174-253): catch the inputs of decoder layer
0 with a `Catcher`, run the decoder layers one by one on one 2048-token sample at a time (batch 1),
then final norm -> lm_head -> CrossEntropy on fp16 logits -> ppl = exp(sum NLL / (nsamples*seqlen)).

Differences from the reference loop:
  * packed layers are small (2-bit Llama-2-7B: 1.6 GB codes + 1.9 GB butterfly factors), so the whole
    model stays resident in HBM instead of being shuttled layer by layer over PCIe (opt.py:260,265);
    `offload=True` restores the reference's layer-by-layer residency for models that do not fit;
  * the loop can run sample-major (`sample_nll`): one sample through all layers, so a benchmark step
    can include the H2D copy of the token ids and the D2H read of the NLL;
  * Llama layers get `position_embeddings` (required by transformers >= 4.48; the reference loop
    crashes there, SURVEY section 8c);
  * `sample_ids` / `layer_range` let the data-parallel and pipeline drivers (pipeline.py) reuse it.
"""
from dataclasses import dataclass
from typing import Callable, List, Optional

import torch
import torch.nn as nn


@dataclass
class Arch:
    name: str
    layers: Callable            # model -> nn.ModuleList of decoder layers
    set_layer: Callable         # (model, i, module)
    pre: Callable               # model -> modules needed to produce layer-0 inputs
    post: Callable              # model -> modules applied after the last layer (norm / project_out)
    head: Callable              # model -> lm_head


def _opt_pre(m):
    d = m.model.decoder
    mods = [d.embed_tokens, d.embed_positions]
    if getattr(d, 'project_in', None) is not None:
        mods.append(d.project_in)
    return mods


def _opt_post(m):
    d = m.model.decoder
    return [x for x in (d.final_layer_norm, getattr(d, 'project_out', None)) if x is not None]


def _set_opt(m, i, mod):
    m.model.decoder.layers[i] = mod


def _set_llama(m, i, mod):
    m.model.layers[i] = mod


OPT = Arch('opt', lambda m: m.model.decoder.layers, _set_opt, _opt_pre, _opt_post, lambda m: m.lm_head)
LLAMA = Arch('llama', lambda m: m.model.layers, _set_llama,
             lambda m: [m.model.embed_tokens] + ([m.model.rotary_emb] if hasattr(m.model, 'rotary_emb') else []),
             lambda m: [m.model.norm] if m.model.norm is not None else [], lambda m: m.lm_head)


class _Stop(Exception):
    pass


def _resident(model, arch, dev):
    """Cheap check that the model already lives on `dev` (first / last decoder layer, embedding, head)."""
    def on(mod):
        t = next(iter(mod.parameters()), None)
        if t is None:
            t = next(iter(mod.buffers()), None)
        return t is None or (t.device.type == dev.type and (dev.index is None or t.device.index == dev.index))
    layers = arch.layers(model)
    mods = [layers[0], layers[len(layers) - 1], arch.head(model)] + list(arch.pre(model))
    qs = [m for m in layers[len(layers) - 1].modules() if hasattr(m, 'qweight')]
    return all(on(m) for m in mods + qs[:1])


class Catcher(nn.Module):
    """Stands in for decoder layer 0, records its inputs and aborts the forward (opt.py:222-241)."""

    def __init__(self, module, sink):
        super().__init__()
        self.module, self.sink = module, sink

    def forward(self, inp, **kwargs):
        self.sink['inp'] = inp
        self.sink['kwargs'] = {k: v for k, v in kwargs.items()
                               if k in ('attention_mask', 'position_ids', 'position_embeddings')}
        raise _Stop


def layer_inputs(model, arch: Arch, batch):
    """Hidden states entering decoder layer 0 for `batch` (1, S) token ids, plus the layer kwargs."""
    sink = {}
    layer0 = arch.layers(model)[0]
    arch.set_layer(model, 0, Catcher(layer0, sink))
    try:
        model(batch)
    except _Stop:
        pass
    finally:
        arch.set_layer(model, 0, layer0)
    return sink['inp'], sink['kwargs']


_NVTX = None


def _nvtx():
    """QUIP_NVTX=1: an NVTX range per decoder layer / stack / head (visible to ncu and nsys; SURVEY section 5)."""
    global _NVTX
    if _NVTX is None:
        import os
        _NVTX = os.environ.get('QUIP_NVTX') == '1' and torch.cuda.is_available()
    return _NVTX


class _Range:
    def __init__(self, name):
        self.name = name

    def __enter__(self):
        if _nvtx():
            torch.cuda.nvtx.range_push(self.name)

    def __exit__(self, *exc):
        if _nvtx():
            torch.cuda.nvtx.range_pop()
        return False


def _call_layer(layer, h, kwargs):
    with _Range('quip.decoder_layer'):
        out = layer(h, **kwargs)
    return out[0] if isinstance(out, (tuple, list)) else out


def run_layers(model, arch: Arch, layers, h, kwargs):
    """h through `layers` in order.  Llama layers on a CUDA device go through the fused stack (quip_b200/fused.py: the
    glue between the linears as four kernels per layer) when QUIP_FUSED_LAYER=1; otherwise the HF layers are called."""
    if arch.name == 'llama' and h.is_cuda:
        from . import fused
        if fused.enabled() and fused.supports(model, h, kwargs):
            with _Range('quip.fused_llama_stack'):
                return fused.llama_stack(layers, h, kwargs)
    for layer in layers:
        h = _call_layer(layer, h, kwargs)
    return h


def sample_logits_nll(model, arch: Arch, h, labels, seqlen):
    """final norm -> lm_head -> shifted CE on fp16 logits, scaled by seqlen (opt.py:280-295)."""
    with _Range('quip.head_and_loss'):
        for mod in arch.post(model):
            h = mod(h)
        logits = arch.head(model)(h)
    shift_logits = logits[:, :-1, :].contiguous()
    shift_labels = labels[:, 1:]
    loss = nn.CrossEntropyLoss()(shift_logits.view(-1, shift_logits.size(-1)), shift_labels.reshape(-1))
    return loss.float() * seqlen


@torch.no_grad()
def sample_nll(model, arch: Arch, batch, layer_range=None):
    """One sample (1, S) through the decoder stack, sample-major.  Returns the NLL (0-dim tensor)."""
    h, kw = layer_inputs(model, arch, batch)
    layers = arch.layers(model)
    lo, hi = layer_range or (0, len(layers))
    h = run_layers(model, arch, [layers[i] for i in range(lo, hi)], h, kw)
    return sample_logits_nll(model, arch, h, batch, model.seqlen)


class GraphedSampleNLL:
    """`sample_nll` for samples of one fixed length with the decoder stack, final norm, lm_head and loss replayed from
    one CUDA graph.  A 7B step is ~1900 kernel launches; issued eagerly they keep a host core busy for most of the step,
    and four ranks on a host with few cores run four times slower each.  The embedding / mask / rotary front end
    (`layer_inputs`, a handful of kernels) stays eager; its layer kwargs are the same for every sample of that length."""

    def __init__(self, model, arch: Arch, example_batch):
        self.model, self.arch = model, arch
        dev = example_batch.device
        with torch.no_grad():
            h, kw = layer_inputs(model, arch, example_batch)
        self.h, self.kw, self.labels = h.clone(), kw, example_batch.clone()
        self.shape = tuple(example_batch.shape)
        side = torch.cuda.Stream(device=dev)
        side.wait_stream(torch.cuda.current_stream(dev))
        with torch.no_grad(), torch.cuda.stream(side):
            for _ in range(2):                              # lazy set-up (descriptors, workspaces) outside the graph
                self._body()
            self.graph = torch.cuda.CUDAGraph()
            with torch.cuda.graph(self.graph, stream=side, capture_error_mode='thread_local'):
                self.out = self._body()
        torch.cuda.current_stream(dev).wait_stream(side)

    def _body(self):
        h = run_layers(self.model, self.arch, list(self.arch.layers(self.model)), self.h, self.kw)
        return sample_logits_nll(self.model, self.arch, h, self.labels, self.model.seqlen)

    @torch.no_grad()
    def __call__(self, batch):
        if tuple(batch.shape) != self.shape:
            raise ValueError(f'graph was captured for samples of shape {self.shape}, got {tuple(batch.shape)}')
        h, _ = layer_inputs(self.model, self.arch, batch)
        self.h.copy_(h)
        self.labels.copy_(batch)
        self.graph.replay()
        return self.out.clone()


def enable_graphed_eval(model, arch: Arch, example_batch):
    """Capture once; `eval_ppl` then replays the graph for every resident, same-length sample.  Returns the stepper
    (also callable directly: nll = stepper(ids))."""
    model._quip_graph_step = GraphedSampleNLL(model, arch, example_batch)
    return model._quip_graph_step


@torch.no_grad()
def eval_ppl(model, arch: Arch, testenc, dev, sample_ids: Optional[List[int]] = None, offload=False,
             verbose=True, reduce_fn=None):
    """Reference-order (layer-major) evaluation.  `testenc` is the tokenizer output (has .input_ids) or a
    (1, nsamples*seqlen) LongTensor.  Returns ppl (the reference only prints it, SURVEY A10)."""
    ids = testenc.input_ids if hasattr(testenc, 'input_ids') else testenc
    seqlen = model.seqlen
    nsamples_total = ids.numel() // seqlen
    mine = list(range(nsamples_total)) if sample_ids is None else list(sample_ids)
    use_cache = model.config.use_cache
    model.config.use_cache = False
    layers = arch.layers(model)
    if not offload:
        if not _resident(model, arch, torch.device(dev)):              # walking a 7B module tree costs milliseconds
            model.to(dev)
    else:
        for mod in arch.pre(model):
            mod.to(dev)
        layers[0].to(dev)
    stepper = getattr(model, '_quip_graph_step', None)
    if stepper is not None and not offload and stepper.shape == (1, seqlen):
        # sample-major through the captured graph: same numbers, no per-kernel host work
        nll = torch.zeros((), dtype=torch.float32, device=dev)
        for i in mine:
            nll += stepper(ids[:, i * seqlen:(i + 1) * seqlen].to(dev, non_blocking=True))
        count = torch.tensor(float(len(mine) * seqlen), device=dev)
        if reduce_fn is not None:
            nll, count = reduce_fn(nll, count)
        ppl = torch.exp(nll / count).item()
        if verbose:
            print(ppl)
        model.config.use_cache = use_cache
        return ppl
    dtype = next(iter(model.parameters())).dtype
    inps = torch.zeros((len(mine), seqlen, model.config.hidden_size), dtype=dtype, device=dev)
    kw = {}
    for slot, i in enumerate(mine):
        batch = ids[:, i * seqlen:(i + 1) * seqlen].to(dev)
        h, kw = layer_inputs(model, arch, batch)
        inps[slot] = h[0]
    if offload:
        layers[0].cpu()
        for mod in arch.pre(model):
            mod.cpu()
        kw = {k: (tuple(t.to(dev) for t in v) if isinstance(v, tuple) else (v.to(dev) if torch.is_tensor(v) else v))
              for k, v in kw.items()}
    outs = torch.zeros_like(inps)
    for li in range(len(layers)):
        layer = layers[li].to(dev) if offload else layers[li]
        for j in range(len(mine)):
            outs[j] = _call_layer(layer, inps[j].unsqueeze(0), kw)[0]
        if offload:
            layers[li] = layer.cpu()
            torch.cuda.empty_cache() if torch.cuda.is_available() else None
        inps, outs = outs, inps
    if offload:
        for mod in arch.post(model):
            mod.to(dev)
        arch.head(model).to(dev)
    nll = torch.zeros((), dtype=torch.float32, device=dev)
    for slot, i in enumerate(mine):
        labels = ids[:, i * seqlen:(i + 1) * seqlen].to(dev)
        nll += sample_logits_nll(model, arch, inps[slot].unsqueeze(0), labels, seqlen)
    count = torch.tensor(float(len(mine) * seqlen), device=dev)
    if reduce_fn is not None:
        nll, count = reduce_fn(nll, count)
    ppl = torch.exp(nll / count).item()
    if verbose:
        print(ppl)
    model.config.use_cache = use_cache
    return ppl


@torch.no_grad()
def decode_benchmark(model, input_ids, check=False, sync=None):
    """Token-by-token decode with a KV cache: the reference's benchmark() (opt.py:431-482).  Returns
    (median seconds per token, ppl or None)."""
    import time
    import numpy as np
    dev = next(iter(model.parameters())).device
    input_ids = input_ids.to(dev)
    sync = sync or (torch.cuda.synchronize if dev.type == 'cuda' else (lambda: None))
    past = None
    times, tot = [], 0.0
    loss_fn = nn.CrossEntropyLoss()
    for i in range(input_ids.numel()):
        sync()
        tick = time.perf_counter()
        out = model(input_ids[:, i:i + 1], past_key_values=past, use_cache=True)
        sync()
        times.append(time.perf_counter() - tick)
        past = out.past_key_values
        if check and i != input_ids.numel() - 1:
            tot += loss_fn(out.logits[0].float(), input_ids[:, i + 1]).item()
    ppl = float(np.exp(tot / (input_ids.numel() - 1))) if check else None
    return float(np.median(times)), ppl
