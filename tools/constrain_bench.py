"""Overhead of constrained generation (quip_constrain_mask + quip_constrain_advance, csrc/constrain.cu) on a synthetic
Llama-2-7B-shaped packed model (quip_b200.synth, 2-bit, vocab 32000).  Needs a CUDA device.

    python tools/constrain_bench.py [--out DIR] [--layers 32] [--steps 127] [--trials 3]

For B in {1, 32}: the captured PromptDecoder step (512-token prompts, greedy, CUDA events over the replays after the
prefill) unconstrained, with every row in a one-state automaton allowing all 32000 tokens, and with one allowing 10
tokens; the three decoders alternate over the trials and the best trial counts.  Also the mask and advance kernels
alone (20 launches captured in one CUDA graph) at each B for both states.  Prints the card's name and power limit
with the numbers, and one JSON line; --out also writes it to DIR/constrain_bench.json.
"""
import argparse
import json
import os
import subprocess
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def card():
    info = dict(name=torch.cuda.get_device_name(0))
    try:
        r = subprocess.run(['nvidia-smi', '--query-gpu=name,power.limit,clocks.max.sm', '--format=csv,noheader'],
                           capture_output=True, text=True, timeout=30)
        info['nvidia_smi'] = r.stdout.strip().splitlines()[0] if r.stdout.strip() else r.stderr.strip()
    except (OSError, subprocess.SubprocessError) as e:
        info['nvidia_smi'] = f'unavailable: {e}'
    return info


def events_ms(fn, reps):
    torch.cuda.synchronize()
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(reps):
        fn()
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1) / reps


def one_state(vocab, n):
    """Every token of the first n ids of a fixed permutation loops on the one state."""
    from quip_b200.constrain import TokenAutomaton
    ids = torch.randperm(vocab, generator=torch.Generator().manual_seed(0))[:n].tolist()
    return TokenAutomaton({0: {v: 0 for v in ids}}, 0)


def kernels_alone(B, V, auto, reps=1000):
    from quip_b200 import fused
    from quip_b200.constrain import pack_automata
    offsets, ids, nxt, starts = (t.cuda() if torch.is_tensor(t) else t for t in pack_automata([auto] * B, V))
    state = torch.tensor(starts, dtype=torch.int32, device='cuda')
    x = torch.randn(B, V, device='cuda').half()
    tok = torch.zeros(B, 1, dtype=torch.long, device='cuda')
    tok[:, 0] = int(ids[0])
    out = {}
    for name, fn in (('mask', lambda: fused.constrain_mask(x, 1, state, offsets, ids, nxt)),
                     ('advance', lambda: fused.constrain_advance(state, tok, offsets, ids, nxt))):
        fn()
        graph, per = torch.cuda.CUDAGraph(), 20
        with torch.cuda.graph(graph):
            for _ in range(per):
                fn()
        graph.replay()
        out[name + '_us'] = 1e3 * events_ms(graph.replay, reps // per) / per
    out['mask_bytes_per_s'] = 2 * B * V * 2 / (out['mask_us'] * 1e-6)     # each row read and written once
    return out


def step_times(model, B, V, steps, trials, P=512):
    from quip_b200.constrain import pack_automata
    from quip_b200.decode import PromptDecoder
    g = torch.Generator().manual_seed(1)
    prompts = [torch.randint(0, V, (P,), generator=g) for _ in range(B)]
    cases = {'unconstrained': None, 'all_tokens': one_state(V, V), 'ten_tokens': one_state(V, 10)}
    decs = {}
    for name, auto in cases.items():
        d = PromptDecoder(model, max_len=P + steps + 1, batch=B, max_new=steps + 1, constraint=auto is not None)
        if auto is not None:
            d.set_constraint(*pack_automata([auto] * B, V))
        decs[name] = d.capture()
    ms = {name: [] for name in decs}
    for _ in range(trials):
        for name, d in decs.items():
            d.prefill(prompts, chunk=512)
            d.graph.replay()                                           # one warm replay
            ms[name].append(events_ms(d.graph.replay, steps - 1))
    ok = {}
    for name, auto in cases.items():
        if auto is not None:
            allowed = torch.tensor(auto.allowed(0), device='cuda')
            ok[name] = bool(torch.isin(decs[name].generated, allowed).all())
    best = {name: min(v) for name, v in ms.items()}
    r = dict(B=B, P=P, steps=steps, step_ms=best, trials_ms=ms, tokens_obey=ok)
    r['overhead'] = {name: best[name] / best['unconstrained'] - 1 for name in ('all_tokens', 'ten_tokens')}
    del decs
    torch.cuda.empty_cache()
    return r


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--out', default=None)
    ap.add_argument('--layers', type=int, default=32, help='decoder layers of the 7B shape to build (of 32)')
    ap.add_argument('--steps', type=int, default=127)
    ap.add_argument('--trials', type=int, default=3)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit('constrain_bench needs a CUDA device')
    from quip_b200.synth import build_synthetic_model, model_config
    info = card()
    print(f"card: {info['name']} ({info['nvidia_smi']})", flush=True)
    cfg = model_config('llama7b', num_hidden_layers=a.layers)
    model = build_synthetic_model(cfg, torch.device('cuda:0'), bits=2, seed=0, seqlen=1024)
    V = cfg.vocab_size
    res = dict(card=info, layers=a.layers, vocab=V, kernels=[], steps=[])
    for B in (1, 32):
        for name, n in (('all_tokens', V), ('ten_tokens', 10)):
            k = kernels_alone(B, V, one_state(V, n))
            k.update(B=B, state=name)
            res['kernels'].append(k)
            print(f"B={B} {name}: mask {k['mask_us']:.2f} us ({k['mask_bytes_per_s'] / 1e12:.2f} TB/s), "
                  f"advance {k['advance_us']:.2f} us", flush=True)
        r = step_times(model, B, V, a.steps, a.trials)
        res['steps'].append(r)
        print(f"B={B} step ms: " + ', '.join(f'{k} {v:.3f}' for k, v in r['step_ms'].items()) +
              ' | overhead ' + ', '.join(f'{k} {100 * v:+.2f}%' for k, v in r['overhead'].items()) +
              f" | tokens obey {r['tokens_obey']}", flush=True)
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, 'constrain_bench.json'), 'w') as f:
            f.write(line + '\n')


if __name__ == '__main__':
    main()
