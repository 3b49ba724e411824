"""Quantise real Llama-2-7B-shaped decoder layers ON THE GPU with this package's producer (quip_b200/quantize.py: tensor-core
Hessian accumulation, incoherence processing, LDLQ-RG with the column loops of csrc/ldlq.cu), pack them, and measure the
perplexity of the packed model against the dense fake-quantised model the reference would evaluate (needs a CUDA device).

    python tools/quantize_bench.py [--layers 2] [--calib 4] [--eval 2] > gpurun_out/quantize_bench.json

This is BASELINE configs[2] end to end on random-init weights (no checkpoints here): `--wbits 2 --quant ldlqRG
--incoh_processing --npasses 2`.  The "ppl delta vs ref" of the metric is measured on an actual quantisation rather than on
synthetic codes: dense path = HF layers with W_ref = fp16(fp16(U^T Q V)/s) (method.py:195-214, what opt_eval / llama_eval
of the reference run), packed path = QuantLinear through the same eval loop.  Only --layers decoder layers are built (the
full 32 need the same code 16 times over); timings are per Linear.
"""
import argparse
import json
import os
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--layers', type=int, default=2)
    ap.add_argument('--calib', type=int, default=4)
    ap.add_argument('--eval', type=int, default=2)
    ap.add_argument('--method', default='ldlq_rg')
    ap.add_argument('--npasses', type=int, default=2)
    ap.add_argument('--dry-cpu', action='store_true', help='tiny model on the CPU, no packed evaluation: checks the script only')
    a = ap.parse_args()
    from quip_b200 import _lib, evalloop, quantize as qz
    from quip_b200.llama import get_llama, llama_eval, llama_pack
    from quip_b200.synth import model_config
    dev = torch.device('cpu' if a.dry_cpu else 'cuda:0')
    lib = _lib.load()
    S = 64 if a.dry_cpu else 2048
    cfg = model_config('llama7b', num_hidden_layers=a.layers, **(dict(hidden_size=128, intermediate_size=256, num_attention_heads=4,
                                                                      num_key_value_heads=4, vocab_size=512) if a.dry_cpu else {}))
    torch.manual_seed(0)
    model = get_llama(cfg, seqlen=S, **(dict(dtype=torch.float32) if a.dry_cpu else {})).to(dev)
    g = torch.Generator().manual_seed(1)
    calib = [torch.randint(0, cfg.vocab_size, (1, S), generator=g) for _ in range(a.calib)]
    test = torch.randint(0, cfg.vocab_size, (1, S * a.eval), generator=g)
    out = dict(config=f'Llama-2-7B layer shapes, {a.layers} decoder layers, 2-bit {a.method} npasses {a.npasses}, --incoh_processing',
               calib_samples=a.calib, eval_samples=a.eval)
    with torch.no_grad():
        ppl_fp16 = llama_eval(model, test, dev, verbose=False)
        sync = (lambda: None) if a.dry_cpu else torch.cuda.synchronize
        sync()
        l0 = lib.quip_launch_count()
        t0 = time.perf_counter()
        parts = qz.quantize_model(model, evalloop.LLAMA, calib, dev=dev, bits=2, method=a.method, greedy_passes=a.npasses,
                                  qfn='b', rescale=True, incoh='blocked', generator=torch.Generator().manual_seed(2), pack=False)
        sync()
        t_quant = time.perf_counter() - t0
        out['quantize_seconds'] = t_quant
        out['quantize_seconds_per_linear'] = t_quant / len(parts)
        out['quantizer_kernel_launches'] = int(lib.quip_launch_count() - l0)
        out['linears'] = len(parts)
        # the model now holds the dense fake-quantised weights W_ref: the reference's effective model
        ppl_ref = llama_eval(model, test, dev, verbose=False)
        if a.dry_cpu:
            print(json.dumps(dict(out, ppl_fp16_unquantized=ppl_fp16, ppl_reference_dense_fake_quant=ppl_ref)))
            return
        t0 = time.perf_counter()
        model.cpu()
        llama_pack(model, parts)
        model.to(dev)
        out['pack_seconds'] = time.perf_counter() - t0
        ppl_packed = llama_eval(model, test, dev, verbose=False)
    out.update(ppl_fp16_unquantized=ppl_fp16, ppl_reference_dense_fake_quant=ppl_ref, ppl_packed=ppl_packed,
               ppl_rel_delta_packed_vs_reference=abs(ppl_packed - ppl_ref) / ppl_ref, tolerance=1e-3)
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
