"""The 2-bit wgmma packed GEMM at 128- and 256-row weight tiles, at the three Llama-2-7B shapes x 2048 tokens.

    python tools/gemm_tiles.py [--rounds 5] [--iters 40] [--out FILE.json]

Each round times every (shape, tile height) once, alternating the two heights (CUDA events around `iters` launches,
rotating weight copies so that the packed words come from HBM).  Reports the median over rounds of the time, TFLOP/s
and the L2->SM bytes/s the tiling implies: every tile reads its activation tile (BN x 64 fp16 per 64-k stage) and
its packed words (BM / 16 row blocks x one super-block per 128 k), so the activations are read N / BM times.  The card
name, power limit and the SM clocks sampled during the timed rounds are part of the output.  Results are printed as
JSON lines; --out also writes them to one JSON file.
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
from quip_b200 import _lib, quant as Q          # noqa: E402

DEV = 'cuda:0'
SHAPES = [(4096, 4096), (11008, 4096), (4096, 11008)]   # (N, K): q/k/v/o, gate/up, down
BN, BK, SB_K, SB_ROWS = 128, 64, 128, 16


def l2_bytes(N, K, M, rows, bits=2):
    """Bytes the tiles fetch from L2 into shared memory: activation tiles + packed words."""
    tiles = -(-N // rows) * -(-M // BN)
    words = {2: 128, 3: 192, 4: 256}[bits] * 4 * (rows // SB_ROWS)
    return tiles * ((K // BK) * BN * BK * 2 + (K // SB_K) * words)


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


class Arm:
    def __init__(self, N, K, M, copies):
        self.N, self.K, self.M = N, K, M
        words = Q.packed_words(N, K, 2)
        g = torch.Generator(device=DEV).manual_seed(N + K)
        self.qw = torch.randint(-2 ** 31, 2 ** 31 - 1, (copies, words), dtype=torch.int32, device=DEV, generator=g)
        self.sc = torch.rand(N, device=DEV, generator=g) * 0.01 + 0.005
        self.ze = self.sc * 1.5
        self.x = torch.randn(M, K, device=DEV, generator=g).half()
        self.xsum = self.x.float().sum(1)
        self.z = torch.empty(M, N, dtype=torch.float16, device=DEV)
        self.descs = []
        for c in range(copies):
            d = _lib.QuipLinearDesc()
            d.K, d.N, d.bits, d.flags = K, N, 2, 0          # asymmetric: the epilogue the model runs
            d.qweight, d.scales, d.zeros = self.qw[c].data_ptr(), self.sc.data_ptr(), self.ze.data_ptr()
            self.descs.append(d)

    def launch(self, i):
        lib = _lib.load()
        _lib.check(lib.quip_qgemm(C.byref(self.descs[i % len(self.descs)]), _lib.ptr(self.x), _lib.ptr(self.xsum),
                                  None, _lib.ptr(self.z), self.M, 2, None, 0,
                                  C.c_void_p(torch.cuda.current_stream().cuda_stream)))

    def time_us(self, rows, iters):
        lib = _lib.load()
        _lib.check(lib.quip_config(b'tc_rows', rows))
        for i in range(4):
            self.launch(i)
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        e0.record()
        for i in range(iters):
            self.launch(i)
        e1.record()
        torch.cuda.synchronize()
        return e0.elapsed_time(e1) / iters * 1e3


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument('--rounds', type=int, default=5)
    ap.add_argument('--iters', type=int, default=40)
    ap.add_argument('--M', type=int, default=2048)
    ap.add_argument('--out', default=None, help='also write the results to this JSON file')
    a = ap.parse_args()
    info = card()
    print(info, flush=True)
    lib = _lib.load()
    arms = [Arm(N, K, a.M, copies=max(2, int(300e6 // (N * K // 4)))) for (N, K) in SHAPES]
    same = {}
    for arm in arms:                            # the two tile heights must agree bit for bit
        outs = []
        for rows in (128, 256):
            _lib.check(lib.quip_config(b'tc_rows', rows))
            arm.launch(0)
            torch.cuda.synchronize()
            outs.append(arm.z.clone())
        same[f'{arm.N}x{arm.K}'] = bool(torch.equal(outs[0].view(torch.int16), outs[1].view(torch.int16)))
    times = {(arm.N, arm.K, rows): [] for arm in arms for rows in (128, 256)}
    with ClockSampler(0) as clk:
        clk.mark_start()
        for r in range(a.rounds):
            order = (128, 256) if r % 2 == 0 else (256, 128)
            for arm in arms:
                for rows in order:
                    times[(arm.N, arm.K, rows)].append(arm.time_us(rows, a.iters))
        clk.mark_end()
    lib.quip_config(b'tc_rows', 0)
    res = []
    for arm in arms:
        row = dict(N=arm.N, K=arm.K, M=a.M, bits_identical=same[f'{arm.N}x{arm.K}'])
        for rows in (128, 256):
            ts = times[(arm.N, arm.K, rows)]
            us = statistics.median(ts)
            row[f'rows{rows}'] = dict(us=us, us_min=min(ts), us_max=max(ts), TFLOPs=2.0 * a.M * arm.N * arm.K / us / 1e6,
                                      l2_GB=l2_bytes(arm.N, arm.K, a.M, rows) / 1e9,
                                      l2_TBps=l2_bytes(arm.N, arm.K, a.M, rows) / us / 1e6)
        row['speedup_256'] = row['rows128']['us'] / row['rows256']['us']
        res.append(row)
        print(json.dumps(row), flush=True)
    out = dict(card=info, clocks=clk.summary(), rounds=a.rounds, iters=a.iters, shapes=res)
    print(json.dumps(dict(card=info, clocks=out['clocks'])), flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, 'w') as f:
            json.dump(out, f, indent=1)


if __name__ == '__main__':
    main()
