"""The wgmma dense pass at 128- and 256-token tiles, at the three uses of the 688-wide pass in a Llama-2-7B layer.

    python tools/dense_pass_bench.py [--rounds 5] [--iters 40] [--M 2048] [--out FILE.json]

The 11008-wide sides run the 688 x 688 block pass three times per decoder layer: gate's and up's N side and down's K
side.  Each use has its own 16 factor blocks (15 MB), so every arm rotates through copies of the three factor sets,
as the step does.  Each round times every use once per tile shape, alternating which shape goes first (CUDA events
around `iters` launches).  Reports the median over rounds of the time, the TFLOP/s of the algorithmic 2 M p^2 nblk
flops, and the L2->SM bytes the tiling implies: every tile reads its token slab (tokens x K_pad fp16) and its factor
slab (columns x K_pad fp16), K_pad = p rounded up to the 64-wide k stage.  The two shapes' outputs are compared bit for
bit first.  The card name, power limit and the SM clocks sampled during the timed rounds are part of the output.
"""
import argparse
import ctypes as C
import json
import os
import statistics
import sys

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)
from bench import ClockSampler                  # noqa: E402
from quip_b200 import _lib                      # noqa: E402
from tools.step_profile import card             # noqa: E402

DEV = 'cuda:0'
P, NBLK, BK = 688, 16, 64
USES = ('gate.U', 'up.U', 'down.V')


def dense_cols(p):
    """Factor columns per 256-token tile (qgemm_tc.cu dense_cols)."""
    t = -(-p // 184)
    return 8 * -(-p // (8 * t))


def tiling(tile, p=P, nblk=NBLK, M=2048):
    """(tokens, columns, tiles, L2->SM bytes) of one launch."""
    cols = 128 if tile == 128 else dense_cols(p)
    kpad = -(-p // BK) * BK
    tiles = -(-p // cols) * -(-M // tile) * nblk
    return tile, cols, tiles, tiles * (tile + cols) * kpad * 2


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--iters', type=int, default=40)
    ap.add_argument('--M', type=int, default=2048)
    ap.add_argument('--out', default=None, help='also write the results to this JSON file')
    a = ap.parse_args()
    assert torch.cuda.is_available(), 'dense_pass_bench needs a GPU'
    info = card()
    print(json.dumps(info), flush=True)
    lib = _lib.load()
    g = torch.Generator(device=DEV).manual_seed(0)
    n = P * NBLK
    copies = 8                                  # 8 x 3 x 15 MB of factors: more than L2, as across a step's layers
    x = torch.randn(a.M, n, device=DEV, generator=g).half()
    out = torch.empty_like(x)
    facs = [[(torch.randn(NBLK, P, P, device=DEV, generator=g) / P ** 0.5).half() for _ in USES] for _ in range(copies)]
    st = C.c_void_p(torch.cuda.current_stream().cuda_stream)

    def launch(f):
        ps = _lib.QuipPass(p=P, nblk=NBLK, strided=0, shared=0, factors=f.data_ptr())
        _lib.check(lib.quip_rot_pass(C.byref(ps), _lib.ptr(x), _lib.ptr(out), a.M, n, 2, st))

    def set_tile(t):
        _lib.check(lib.quip_config(b'dense_tile', t))

    same = {}
    for u, use in enumerate(USES):
        outs = []
        for t in (128, 256):
            set_tile(t)
            launch(facs[0][u])
            torch.cuda.synchronize()
            outs.append(out.clone())
        same[use] = bool(torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16)))

    def time_us(t, u):
        set_tile(t)
        for i in range(4):
            launch(facs[i % copies][u])
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(a.iters):
            launch(facs[i % copies][u])
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / a.iters * 1e3

    times = {(use, t): [] for use in USES for t in (128, 256)}
    with ClockSampler(0) as clk:
        clk.mark_start()
        for r in range(a.rounds):
            order = (128, 256) if r % 2 == 0 else (256, 128)
            for u, use in enumerate(USES):
                for t in order:
                    times[(use, t)].append(time_us(t, u))
        clk.mark_end()
    set_tile(0)
    flops = 2.0 * a.M * P * P * NBLK
    res = []
    for use in USES:
        row = dict(use=use, p=P, nblk=NBLK, M=a.M, bits_identical=same[use])
        for t in (128, 256):
            ts = times[(use, t)]
            us = statistics.median(ts)
            tok, cols, tiles, l2 = tiling(t, M=a.M)
            row[f'tile{t}'] = dict(tokens=tok, cols=cols, tiles=tiles, us=us, us_min=min(ts), us_max=max(ts),
                                   TFLOPs=flops / us / 1e6, l2_MB=l2 / 1e6, l2_TBps=l2 / us / 1e6)
        row['speedup_256'] = row['tile128']['us'] / row['tile256']['us']
        res.append(row)
        print(json.dumps(row), flush=True)
    result = dict(card=info, clocks=clk.summary(), rounds=a.rounds, iters=a.iters, uses=res)
    print(json.dumps(dict(card=info, clocks=result['clocks'])), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(result, f, indent=1)


if __name__ == '__main__':
    main()
