"""Disparity mappers on the engine: us per call of the fused per-frame min/max + mapper pass (nb200_minmax_mapper, what
stereo_sbs runs) and of the standalone mapper (nb200_mapper_apply), for none, div_6, mul_2, inv_mul_2, shift_20, a blend and
a two-stage chain, on the depth shapes of bench.py's iw3_1080p (4 x 392 x 686) and iw3_4k_zoe (2 x 384 x 704) lines.
GB/s is against the floor of 8 bytes per pixel (one fp32 read and one write); the fused pass also reads the map once more
for its min/max.  Names are timed round-robin, ROUNDS times, and the spread over the rounds is printed with the median.
Prints the card and its power limit.  Results go to stdout and, with --out, to DIR/result.json.
    python profiles/bench_mapper.py [--iters 200] [--rounds 5] [--out DIR]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nunif_b200 import synth, _lib  # noqa: E402
from nunif_b200.iw3.mapper import descriptor  # noqa: E402

NAMES = ["none", "div_6", "mul_2", "inv_mul_2", "shift_20", "div_6+div_4=0.5", "mul_1+mul_2=0.5:div_6"]
SHAPES = {"iw3_1080p": (4, 392, 686), "iw3_4k_zoe": (2, 384, 704)}


def timed(fn, iters):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(iters):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) * 1e3 / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=200)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for result.json")
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    print("card:", q)
    dev = "cuda:0"
    L = _lib.lib()
    rows = []
    for tag, (B, h, w) in SHAPES.items():
        n = h * w
        raw = (synth.synth_depth(1, B, h, w) * 7 + 2).to(dev)
        d01 = synth.synth_depth(2, B, h, w).to(dev)
        out = torch.empty_like(raw)
        st = _lib.stream_ptr()
        calls = {}
        for name in NAMES:
            desc = ctypes.byref(descriptor(name))
            calls[("fused", name)] = (lambda d=desc: _lib.check(L.nb200_minmax_mapper(_lib.ptr(raw), B, n, d, _lib.ptr(out), None, st)))
            calls[("mapper", name)] = (lambda d=desc: _lib.check(L.nb200_mapper_apply(_lib.ptr(d01), B * n, d, _lib.ptr(out), st)))
        for f in calls.values():
            f(); f()
        torch.cuda.synchronize()
        samples = {k: [] for k in calls}
        for _ in range(a.rounds):
            for k, f in calls.items():
                samples[k].append(timed(f, a.iters))
        for (kind, name), us in samples.items():
            med = statistics.median(us)
            row = dict(shape=tag, B=B, h=h, w=w, pass_=kind, mapper=name, us_median=round(med, 2), us_min=round(min(us), 2),
                       us_max=round(max(us), 2), gbps_8B_floor=round(8.0 * B * n / (med * 1e-6) / 1e9, 1))
            rows.append(row)
            print(json.dumps(row))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "result.json"), "w") as fh:
            json.dump(dict(card=q, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
