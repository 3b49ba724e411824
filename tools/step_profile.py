"""Where the time of the headline step goes: per-kernel device time of one timed step of bench.py, from torch.profiler.

    python tools/step_profile.py --out-dir DIR [--replays 3] [--warmup 3]

Builds the bench model (Llama-2-7B, 2-bit, blocked butterflies + rescale, seed 0, 2048 tokens), primes it, picks the
glue and captures the step in a CUDA graph exactly as bench.py does, replays it `warmup` times, then profiles `replays`
replays with CUDA activities.  Kernels whose names differ only in template arguments stay apart (the dense pass and the
packed GEMM are both qgemm_tc_kernel).  Writes DIR/step_profile.json: per-kernel total device ms per step, launches per
step and share of the step (the graph replay's CUDA-event time, measured without the profiler), plus the card name,
power limit and SM clocks.  Environment switches of the library (QUIP_TC_ROWS, QUIP_DENSE_TILE, ...) apply as in bench.
"""
import argparse
import collections
import json
import os
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
import bench                                    # noqa: E402
from bench import SEQ, ClockSampler             # noqa: E402


def card():
    import subprocess
    q = 'name,power.limit,clocks.max.sm'
    try:
        out = subprocess.run(['nvidia-smi', '-i', '0', f'--query-gpu={q}', '--format=csv,noheader,nounits'],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, plim, smax = [c.strip() for c in out.split(',')]
        return dict(name=name, power_limit_w=float(plim), sm_max_mhz=float(smax))
    except Exception as e:                      # reported, never silently replaced by a guess
        return dict(error=f'nvidia-smi: {e}')


def build_step(dev):
    """The model and the timed step of bench.py main() (dp, one rank)."""
    from quip_b200 import evalloop
    from quip_b200.quant import group_siblings
    from quip_b200.synth import build_synthetic_model, model_config
    arch = evalloop.LLAMA
    cfg = model_config('llama7b')
    model = build_synthetic_model(cfg, dev, bits=2, incoh='blocked', rescale=True, seed=0, seqlen=SEQ)
    model.seqlen = SEQ
    if os.environ.get('QUIP_NO_OVERLAP') != '1':
        group_siblings(model)
    with torch.no_grad():
        prime = torch.randint(0, cfg.vocab_size, (1, SEQ), device=dev)
        for _ in range(2):
            evalloop.sample_nll(model, arch, prime)
    torch.cuda.synchronize()
    glue = bench.pick_glue(model, prime)
    if glue['mode'] == 'fused':
        with torch.no_grad():
            evalloop.sample_nll(model, arch, prime)
        torch.cuda.synchronize()
    stepper = evalloop.enable_graphed_eval(model, arch, prime)
    ids = torch.randint(0, cfg.vocab_size, (1, SEQ), generator=torch.Generator().manual_seed(1234)).to(dev)
    return stepper, ids, glue


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--replays', type=int, default=3)
    ap.add_argument('--warmup', type=int, default=3)
    ap.add_argument('--out-dir', required=True, help='directory for step_profile.json')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'step_profile needs a GPU'
    dev = torch.device('cuda', 0)
    torch.cuda.set_device(dev)
    info = card()
    stepper, ids, glue = build_step(dev)
    with torch.no_grad(), ClockSampler(0) as clk:
        for _ in range(a.warmup):
            stepper(ids)
        torch.cuda.synchronize()
        # step time without the profiler: CUDA events around the same number of replays
        clk.mark_start()
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for _ in range(a.replays):
            stepper(ids)
        e1.record()
        torch.cuda.synchronize()
        clk.mark_end()
        step_ms = e0.elapsed_time(e1) / a.replays
        from torch.profiler import ProfilerActivity, profile
        with profile(activities=[ProfilerActivity.CUDA]) as prof:
            for _ in range(a.replays):
                stepper(ids)
            torch.cuda.synchronize()
    tot = collections.defaultdict(float)
    cnt = collections.Counter()
    for ev in prof.events():
        if ev.device_type == torch.autograd.DeviceType.CUDA and ev.device_time > 0:
            tot[ev.name] += ev.device_time / 1e3            # us -> ms
            cnt[ev.name] += 1
    busy = sum(tot.values()) / a.replays
    rows = sorted(({'kernel': k, 'ms_per_step': v / a.replays, 'launches_per_step': cnt[k] / a.replays,
                    'share_of_step': v / a.replays / step_ms} for k, v in tot.items()), key=lambda r: -r['ms_per_step'])
    out = dict(card=info, clocks=clk.summary(), glue=glue.get('mode'), replays=a.replays, step_ms=step_ms,
               kernel_ms_per_step=busy,
               note='step_ms: CUDA events around graph replays without the profiler; kernel times from torch.profiler '
                    '(a separate set of replays).  Sibling linears run on side streams, so kernel time can exceed the step.',
               env={k: v for k, v in os.environ.items() if k.startswith('QUIP_')}, kernels=rows)
    os.makedirs(a.out_dir, exist_ok=True)
    path = os.path.join(a.out_dir, 'step_profile.json')
    with open(path, 'w') as f:
        json.dump(out, f, indent=1)
    print(json.dumps(dict(card=info, step_ms=step_ms, kernel_ms_per_step=busy, out=path)))
    for r in rows[:25]:
        print(f"{r['share_of_step'] * 100:6.2f} %  {r['ms_per_step']:8.3f} ms  {r['launches_per_step']:6.1f}  {r['kernel'][:150]}")


if __name__ == '__main__':
    main()
