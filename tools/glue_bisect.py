"""Where does the fused Llama stack (quip_b200/fused.py) part from the HF decoder layers?  (needs a CUDA device)

    python tools/glue_bisect.py [--layers 2] > gpurun_out/glue_bisect.json

Runs the first decoder layers of the benchmark model (Llama-2-7B sizes, synthetic packed linears, one 2048-token sample)
both ways, records every intermediate of both (HF: module hooks + a recording wrapper around F.scaled_dot_product_attention;
fused: llama_stack(trace=...)), and prints per stage
  * `chain`: fused-path tensor vs HF-path tensor (errors accumulate along the layer),
  * `isolated`: the fused op applied to the HF path's OWN inputs vs the HF output of that stage (one op at a time),
  * `repeat`: the same QuantLinear called twice on the same input (determinism of the packed path).
"""
import argparse
import json
import os
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def err(a, b):
    a, b = a.double().reshape(-1), b.double().reshape(-1)
    return dict(rel=float((a - b).norm() / b.norm().clamp_min(1e-300)), frac_equal=float((a == b).double().mean()),
                max_abs=float((a - b).abs().max()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--layers', type=int, default=2)
    ap.add_argument('--no-groups', action='store_true')
    a = ap.parse_args()
    from transformers import LlamaConfig
    from quip_b200 import evalloop, fused
    from quip_b200.quant import group_siblings
    from quip_b200.synth import LLAMA2_7B, build_synthetic_model
    dev = torch.device('cuda:0')
    cfg = LlamaConfig(**{**LLAMA2_7B, 'num_hidden_layers': a.layers})
    model = build_synthetic_model(cfg, dev, bits=2, incoh='blocked', rescale=True, seed=0, seqlen=2048)
    if not a.no_groups:
        group_siblings(model)
    ids = torch.randint(0, cfg.vocab_size, (1, 2048), device=dev)
    out = dict(layers=a.layers, groups=not a.no_groups, stages=[])
    with torch.no_grad():
        h0, kw = evalloop.layer_inputs(model, evalloop.LLAMA, ids)
        out['mask'] = None if kw.get('attention_mask') is None else list(kw['attention_mask'].shape)
        layers = list(model.model.layers)
        # ---- HF path with recording ----
        hf = {}
        hooks = []
        sd_calls = []
        real_sdpa = F.scaled_dot_product_attention

        def rec_sdpa(q, k, v, *args, **kwargs):
            o = real_sdpa(q, k, v, *args, **kwargs)
            sd_calls.append(dict(q=q, k=k, v=v, o=o, kwargs={kk: (None if vv is None else (list(vv.shape) if torch.is_tensor(vv) else vv))
                                                              for kk, vv in kwargs.items()},
                                 q_stride=list(q.stride()), k_stride=list(k.stride()), v_stride=list(v.stride())))
            return o

        def hook(li, name, mod, want_in=None):
            def fn(m, inp, outp):
                if want_in:
                    hf[(li, want_in)] = inp[0].clone()
                hf[(li, name)] = (outp[0] if isinstance(outp, tuple) else outp).clone()
            hooks.append(mod.register_forward_hook(fn))

        for li, L in enumerate(layers):
            hook(li, 'x_attn', L.input_layernorm, 'h_in')
            hook(li, 'q_lin', L.self_attn.q_proj)
            hook(li, 'k_lin', L.self_attn.k_proj)
            hook(li, 'v_lin', L.self_attn.v_proj)
            hook(li, 'o_lin', L.self_attn.o_proj, 'attn_out')
            hook(li, 'x_mlp', L.post_attention_layernorm, 'h_mid')
            hook(li, 'gate', L.mlp.gate_proj)
            hook(li, 'up', L.mlp.up_proj)
            hook(li, 'down', L.mlp.down_proj, 'act')
        F.scaled_dot_product_attention = rec_sdpa
        torch.nn.functional.scaled_dot_product_attention = rec_sdpa
        try:
            r = h0
            for L in layers:
                r = evalloop._call_layer(L, r, kw)
            hf_final = r.clone()
            hf_sd = list(sd_calls)
            sd_calls.clear()
            for hk in hooks:                                # the fused stack calls the same linear modules: stop recording
                hk.remove()
            hooks.clear()
            trace = []
            fu_final = fused.llama_stack(layers, h0.clone(), kw, trace=trace)
            fu_sd = list(sd_calls)
        finally:
            F.scaled_dot_product_attention = real_sdpa
            torch.nn.functional.scaled_dot_product_attention = real_sdpa
            for hk in hooks:
                hk.remove()
        S = 2048
        for li, c in enumerate(hf_sd):
            nq = c['q'].shape[1]
            hf[(li, 'q_rope')] = c['q'].transpose(1, 2).reshape(1, S, -1).clone()
            hf[(li, 'k_rope')] = c['k'].transpose(1, 2).reshape(1, S, -1).clone()
        out['sdpa_hf'] = [dict(kwargs=c['kwargs'], q_stride=c['q_stride'], k_stride=c['k_stride'], v_stride=c['v_stride']) for c in hf_sd]
        out['sdpa_fused'] = [dict(kwargs=c['kwargs'], q_stride=c['q_stride'], k_stride=c['k_stride'], v_stride=c['v_stride']) for c in fu_sd]
        out['final'] = err(fu_final, hf_final)
        for (li, name, t) in trace:
            if (li, name) in hf:
                out['stages'].append(dict(layer=li, stage=name, chain=err(t, hf[(li, name)])))
        # ---- isolated ops on the HF path's own inputs ----
        ops = fused.CudaGlue()
        cos, sin = kw['position_embeddings']
        cos, sin = cos[0].contiguous(), sin[0].contiguous()
        iso = []
        for li, L in enumerate(layers):
            n1, n2 = L.input_layernorm, L.post_attention_layernorm
            hd = L.self_attn.head_dim
            iso.append(dict(layer=li, op='rmsnorm(h_in)', **err(ops.rmsnorm(hf[(li, 'h_in')].contiguous(), n1.weight, n1.variance_epsilon), hf[(li, 'x_attn')])))
            q, k = hf[(li, 'q_lin')].clone(), hf[(li, 'k_lin')].clone()
            ops.rope_(q, k, cos, sin, hd)
            iso.append(dict(layer=li, op='rope q', **err(q, hf[(li, 'q_rope')])))
            iso.append(dict(layer=li, op='rope k', **err(k, hf[(li, 'k_rope')])))
            c = hf_sd[li]
            nq = c['q'].shape[1]
            qh = hf[(li, 'q_rope')].view(1, S, nq, hd).transpose(1, 2)
            kh = hf[(li, 'k_rope')].view(1, S, nq, hd).transpose(1, 2)
            vh = hf[(li, 'v_lin')].view(1, S, nq, hd).transpose(1, 2)
            mask = kw.get('attention_mask')
            o = real_sdpa(qh, kh, vh, attn_mask=mask, dropout_p=0.0, scale=L.self_attn.scaling, is_causal=(mask is None))
            o = o.transpose(1, 2).reshape(1, S, nq * hd)
            iso.append(dict(layer=li, op='sdpa(strided views of HF q,k,v)', **err(o, hf[(li, 'attn_out')])))
            iso.append(dict(layer=li, op='sdpa recorded inputs equal HF module tensors',
                            q_equal=bool(torch.equal(c['q'], qh)), v_equal=bool(torch.equal(c['v'], vh))))
            s, y = ops.rmsnorm(hf[(li, 'h_in')].contiguous(), n2.weight, n2.variance_epsilon, residual=hf[(li, 'o_lin')].contiguous())
            iso.append(dict(layer=li, op='h_in + o_lin', **err(s, hf[(li, 'h_mid')])))
            iso.append(dict(layer=li, op='rmsnorm(h_in + o_lin)', **err(y, hf[(li, 'x_mlp')])))
            iso.append(dict(layer=li, op='silu_mul', **err(ops.silu_mul(hf[(li, 'gate')].contiguous(), hf[(li, 'up')].contiguous()), hf[(li, 'act')])))
            for name, mod, xin in (('q_proj', L.self_attn.q_proj, 'x_attn'), ('o_proj', L.self_attn.o_proj, 'attn_out'),
                                   ('gate_proj', L.mlp.gate_proj, 'x_mlp'), ('down_proj', L.mlp.down_proj, 'act')):
                xi = hf[(li, xin)].contiguous()
                y1 = mod._forward_impl(xi)
                y2 = mod._forward_impl(xi.clone())
                ref_name = {'q_proj': 'q_lin', 'o_proj': 'o_lin', 'gate_proj': 'gate', 'down_proj': 'down'}[name]
                iso.append(dict(layer=li, op=f'repeat {name}', twice_equal=bool(torch.equal(y1, y2)), **err(y1, hf[(li, ref_name)])))
        out['isolated'] = iso
    print(json.dumps(out, indent=1))


if __name__ == '__main__':
    main()
