"""OPT entry points of the reference's opt.py, on the packed H100 path.

Kept names (reference opt.py): get_opt (:14-26), opt_eval (:193-299), opt_pack3 (:303-315) ->
opt_pack, load_quant3 (:317-348) / load_quant (:350-381), opt_multigpu (:384-428), benchmark
(:431-482), opt_sequential (:29-190) -> quip_b200.quantize.sequential (torch LDLQ producer; a reference run under
quip_b200.capture.Capture hands the same LayerParts to opt_pack).
"""
import math

import torch

from . import evalloop
from .modelutils import find_layers
from .quant import QuantLinear, make_quant, spec_from_parts

ARCH = evalloop.OPT
SKIP = ('model.decoder.project_out', 'model.decoder.project_in', 'lm_head')       # opt.py:367-372


def _no_init():
    def noop(*args, **kwargs):
        pass
    torch.nn.init.kaiming_uniform_ = noop
    torch.nn.init.uniform_ = noop
    torch.nn.init.normal_ = noop


def get_opt(model, dtype=torch.float16):
    """`model` is a name/path for from_pretrained, or an OPTConfig for a random-init model (no network here)."""
    from transformers import OPTConfig, OPTForCausalLM
    if isinstance(model, OPTConfig):
        prev = torch.get_default_dtype()
        torch.set_default_dtype(dtype)
        try:
            m = OPTForCausalLM(model)
        finally:
            torch.set_default_dtype(prev)
    else:
        _no_init()
        m = OPTForCausalLM.from_pretrained(model, torch_dtype='auto')
    m.seqlen = m.config.max_position_embeddings           # opt.py:25
    return m.eval()


@torch.no_grad()
def opt_eval(model, testenc, dev, **kw):
    return evalloop.eval_ppl(model, ARCH, testenc, dev, **kw)


@torch.no_grad()
def opt_sequential(model, dataloader, dev, args, **kw):
    """Reference opt_sequential (opt.py:29-190) with `args` passed explicitly; returns {name: LayerParts}."""
    from . import quantize
    return quantize.sequential(model, ARCH, dataloader, dev, args, **kw)


def opt_pack(model, parts_by_name):
    """Swap every named Linear for a QuantLinear and pack it (reference opt_pack3, opt.py:303-315, for any
    bit width; the packing itself runs on the GPU when the model is there -- the TODO at opt.py:302)."""
    make_quant(model, parts_by_name)
    qlayers = find_layers(model, [QuantLinear])
    for name, parts in parts_by_name.items():
        qlayers[name].pack_parts(parts)
    return model


def opt_pack3(model, quantizers):
    """Reference signature (opt.py:303-315): dense grid weights + Quantizer objects (qfn 'a', no incoherence)."""
    layers = find_layers(model)
    layers = {n: layers[n] for n in quantizers}
    make_quant(model, list(quantizers.keys()), bits=3)
    qlayers = find_layers(model, [QuantLinear])
    for name in qlayers:
        qlayers[name].pack(layers[name], quantizers[name].scale.cpu(), quantizers[name].zero.cpu())
    return model


def _specs_from_state_dict(sd):
    """Per-layer QuantLinear constructor kwargs inferred from a packed checkpoint."""
    specs = {}
    for key, t in sd.items():
        if not key.endswith('.qweight'):
            continue
        name = key[:-len('.qweight')]
        N = sd[name + '.scales'].shape[0]
        specs[name] = dict(words=t.numel(), N=N, bias=(name + '.bias') in sd, rescale=(name + '.inv_scale') in sd,
                           incoh=None)
        f0 = sd.get(name + '.v_f0')
        if f0 is not None:
            specs[name]['incoh'] = 'kron' if (f0.shape[0] == 1 and sd[name + '.v_idx'].numel() // f0.shape[-1] > 1) \
                else 'blocked'
    return specs


def swap_for_checkpoint(model, sd, skip=SKIP):
    layers = find_layers(model)
    specs = _specs_from_state_dict(sd)
    names = {}
    for name, s in specs.items():
        if name in skip or name not in layers:
            continue
        K, N = layers[name].in_features, layers[name].out_features
        bits = s['words'] * 32 // (N * K)
        names[name] = dict(bits=bits, bias=s['bias'], incoh=s['incoh'], rescale=s['rescale'])
    make_quant(model, names)
    return model


def load_quant(model, checkpoint):
    """Reference load_quant (opt.py:350-381) with its commented-out swap point (:373) made real: a packed
    checkpoint (state_dict with qweight/... buffers) loads into QuantLinear modules; a dense fp16
    state_dict written by the reference's --save still loads as plain nn.Linear."""
    from transformers import OPTConfig
    config = model if isinstance(model, OPTConfig) else OPTConfig.from_pretrained(model)
    _no_init()
    m = get_opt(config)
    sd = checkpoint if isinstance(checkpoint, dict) else torch.load(checkpoint, map_location='cpu')
    swap_for_checkpoint(m, sd)
    m.load_state_dict(sd)
    m.seqlen = m.config.max_position_embeddings
    return m


load_quant3 = load_quant


def layer_placement(nlayers, ngpus):
    """Contiguous layer ranges per pipeline stage: ceil(L/G) per GPU, as opt.py:424-426."""
    per = math.ceil(nlayers / ngpus)
    return [(min(s * per, nlayers), min((s + 1) * per, nlayers)) for s in range(ngpus)]


def opt_multigpu(model, gpus):
    """Single-process layer placement over `gpus` (reference opt.py:384-428, MoveModule semantics).  The
    multi-process NCCL pipeline lives in quip_b200/pipeline.py."""
    import torch.nn as nn

    class MoveModule(nn.Module):
        def __init__(self, module):
            super().__init__()
            self.module = module
            self.dev = next(iter(self.module.parameters())).device

        def forward(self, *inp, **kwargs):
            inp = [t.to(self.dev) if torch.is_tensor(t) else t for t in inp]
            kwargs = {k: (v.to(self.dev) if torch.is_tensor(v) else
                          (tuple(t.to(self.dev) for t in v) if isinstance(v, tuple) and v and torch.is_tensor(v[0]) else v))
                      for k, v in kwargs.items()}
            return self.module(*inp, **kwargs)

    d = model.model.decoder
    d.embed_tokens.to(gpus[0]); d.embed_positions.to(gpus[0])
    if getattr(d, 'project_in', None) is not None:
        d.project_in.to(gpus[0])
    if getattr(d, 'project_out', None) is not None:
        d.project_out.to(gpus[-1])
    if d.final_layer_norm is not None:
        d.final_layer_norm.to(gpus[-1])
    import copy
    model.lm_head = copy.deepcopy(model.lm_head).to(gpus[-1])
    for (lo, hi), g in zip(layer_placement(len(d.layers), len(gpus)), gpus):
        for i in range(lo, hi):
            d.layers[i] = MoveModule(d.layers[i].to(g))
    model.gpus = gpus


def benchmark(model, input_ids, check=False, graph=False):
    """The reference's benchmark() (opt.py:431-482): token-by-token decode with a KV cache.  graph=True replays the same
    step from one CUDA graph (quip_b200.decode.GraphDecoder) instead of the eager HF forward."""
    if graph:
        from .decode import graph_decode_benchmark
        return graph_decode_benchmark(model, input_ids, check=check)
    return evalloop.decode_benchmark(model, input_ids, check=check)
