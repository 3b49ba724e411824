"""Llama entry points of the reference's llama.py, on the packed H100 path.

Kept names (reference llama.py): get_llama (:19-33), llama_eval (:174-253), llama_pack (:256-275),
load_quant (:322-358), llama_multigpu (:361-415), benchmark (:418-471).  The reference's llama.py is
inconsistent as shipped (no --incoh_processing, Balance.configure arity, OPT key prefix: SURVEY A2-A4);
these implement the intended behaviour = opt.py's flow applied to Llama modules.
"""
import torch

from . import evalloop
from .modelutils import find_layers
from .opt import _no_init, layer_placement, swap_for_checkpoint
from .quant import QuantLinear, make_quant

ARCH = evalloop.LLAMA
SKIP = ('lm_head',)                                       # llama.py:341-343


def get_llama(model, dtype=torch.float16, seqlen=2048):
    from transformers import LlamaConfig, LlamaForCausalLM
    if isinstance(model, LlamaConfig):
        prev = torch.get_default_dtype()
        torch.set_default_dtype(dtype)
        try:
            m = LlamaForCausalLM(model)
        finally:
            torch.set_default_dtype(prev)
    else:
        _no_init()
        m = LlamaForCausalLM.from_pretrained(model, torch_dtype=torch.float16)
    m.seqlen = seqlen                                     # llama.py:31
    return m.eval()


@torch.no_grad()
def llama_eval(model, testenc, dev, **kw):
    return evalloop.eval_ppl(model, ARCH, testenc, dev, **kw)


@torch.no_grad()
def llama_sequential(model, dataloader, dev, args, **kw):
    """Reference llama_sequential (llama.py:26-171) as it was meant to run -- opt.py's flow on the Llama layers (the
    shipped one reads an inconsistent flag set and a module global, SURVEY A2/A3); returns {name: LayerParts} with the
    Llama module names (not the OPT prefix of llama.py:154-155, SURVEY A4)."""
    from . import quantize
    return quantize.sequential(model, ARCH, dataloader, dev, args, **kw)


def llama_pack(model, parts_by_name):
    make_quant(model, parts_by_name)
    qlayers = find_layers(model, [QuantLinear])
    for name, parts in parts_by_name.items():
        qlayers[name].pack_parts(parts)
    return model


def load_quant(model, checkpoint, seqlen=2048):
    from transformers import LlamaConfig
    config = model if isinstance(model, LlamaConfig) else LlamaConfig.from_pretrained(model)
    m = get_llama(config, seqlen=seqlen)
    if isinstance(checkpoint, dict):
        sd = checkpoint
    elif str(checkpoint).endswith('.safetensors'):       # llama.py:348-350
        from safetensors.torch import load_file
        sd = load_file(checkpoint)
    else:
        sd = torch.load(checkpoint, map_location='cpu')
    swap_for_checkpoint(m, sd, skip=SKIP)
    m.load_state_dict(sd, strict=False)                  # rotary buffers, llama.py:352
    return m


def parse_layers_dist(spec, nlayers):
    """`--layers-dist a:b:c` (llama.py:400-413,509-512): explicit layer counts per GPU."""
    counts = [int(x) for x in spec.split(':')]
    assert sum(counts) == nlayers, 'layers-dist must sum to the number of layers'
    out, lo = [], 0
    for c in counts:
        out.append((lo, lo + c))
        lo += c
    return out


def llama_multigpu(model, gpus, layers_dist=None):
    """Single-process placement (reference llama.py:361-415).  NCCL pipeline: quip_b200/pipeline.py."""
    import copy
    import torch.nn as nn

    class MoveModule(nn.Module):
        def __init__(self, module):
            super().__init__()
            self.module = module
            self.dev = next(iter(self.module.parameters())).device

        def forward(self, *inp, **kwargs):
            def mv(v):
                if torch.is_tensor(v):
                    return v.to(self.dev)
                if isinstance(v, tuple) and v and torch.is_tensor(v[0]):
                    return tuple(t.to(self.dev) for t in v)
                return v
            return self.module(*[mv(t) for t in inp], **{k: mv(v) for k, v in kwargs.items()})

    mm = model.model
    mm.embed_tokens.to(gpus[0])
    if hasattr(mm, 'rotary_emb'):
        mm.rotary_emb.to(gpus[0])
    mm.norm.to(gpus[-1])
    model.lm_head = copy.deepcopy(model.lm_head).to(gpus[-1])
    ranges = parse_layers_dist(layers_dist, len(mm.layers)) if layers_dist else layer_placement(len(mm.layers), len(gpus))
    for (lo, hi), g in zip(ranges, gpus):
        for i in range(lo, hi):
            mm.layers[i] = MoveModule(mm.layers[i].to(g))
    model.gpus = gpus


def benchmark(model, input_ids, check=False, graph=False):
    """The reference's benchmark() (llama.py / opt.py:431-482): token-by-token decode with a KV cache.  graph=True
    replays the same step from one CUDA graph (quip_b200.decode.GraphDecoder) instead of the eager HF forward."""
    if graph:
        from .decode import graph_decode_benchmark
        return graph_decode_benchmark(model, input_ids, check=check)
    return evalloop.decode_benchmark(model, input_ids, check=check)
