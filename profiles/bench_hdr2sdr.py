"""HDR -> SDR input stage at 3840 x 2160: ms per frame of the fused kernel (csrc/hdr2sdr.cu, uint16 and float outputs) and of the
reference's torch op sequence (oracle/hdr2sdr.py on the same GPU, frame by frame as the reference calls it, without its
device -> host copy), for PQ and HLG at B = 1 and 4.  GB/s counts the bytes the fused kernel must move - 6 in + 6 out per
pixel for the uint16 output, 6 + 12 for the float output - and is set against the H100 SXM data-sheet 3.35 TB/s; the op
sequence is charged the same bytes, so its GB/s is only a speed ratio.  Calls are timed with CUDA events, round-robin,
ROUNDS times, after a warm-up; median and spread are printed.

Then the end-to-end frame rate of FrameBatchPipeline over 4K uint16 frames (pinned, identity callback, batch 4) with and
without hdr2sdr=(16, "bt709"), alternated.  Prints the card and its power limit.
    python profiles/bench_hdr2sdr.py [--iters 20] [--rounds 5] [--frames 96] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nunif_b200.nunif.video import FrameBatchPipeline, hdr2sdr  # noqa: E402
from oracle import hdr2sdr as ohs  # noqa: E402

H, W = 2160, 3840
PEAK_BPS = 3.35e12


def timed(fn, iters):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(iters):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / iters


def pipeline_fps(frames, option, batch):
    pipe = FrameBatchPipeline(lambda x: x, batch, "cuda:0", use_16bit=True, copy_output=False, hdr2sdr=option)
    n = 0
    t0 = time.perf_counter()
    for f in frames:
        n += len(pipe(f))
    n += len(pipe(None))
    torch.cuda.synchronize()
    assert n == len(frames)
    return n / (time.perf_counter() - t0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=96)
    ap.add_argument("--out", default=None, help="directory for result.json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_hdr2sdr needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    print("card:", q)
    dev = "cuda:0"
    g = torch.Generator().manual_seed(1)
    rows = []
    for B in (1, 4):
        x = torch.randint(0, 65536, (B, H, W, 3), generator=g, dtype=torch.int32).to(torch.uint16).to(dev)
        for trc, cs in ((ohs.PQ, "bt709"), (ohs.HLG, "bt709")):
            calls = {
                "fused_uint16": (lambda: hdr2sdr(x, trc, cs), 12),
                "fused_float": (lambda: hdr2sdr(x, trc, cs, output="float"), 18),
                "torch_ops": (lambda: [ohs.hdr2sdr(f, trc, cs, device=dev) for f in x], 12),
            }
            for f, _ in calls.values():
                f(); f()
            torch.cuda.synchronize()
            samples = {k: [] for k in calls}
            for _ in range(a.rounds):
                for k, (f, _) in calls.items():
                    samples[k].append(timed(f, a.iters) / B)
            for k, ms in samples.items():
                med = statistics.median(ms)
                gbps = calls[k][1] * H * W / (med * 1e-3) / 1e9
                row = dict(B=B, trc=trc, colorspace=cs, step=k, ms_per_frame=round(med, 4), ms_min=round(min(ms), 4),
                           ms_max=round(max(ms), 4), gbps=round(gbps, 1), pct_of_3350=round(100 * gbps * 1e9 / PEAK_BPS, 1))
                rows.append(row)
                print(json.dumps(row))
        del x
    torch.cuda.empty_cache()
    frames = [torch.randint(0, 65536, (H, W, 3), generator=g, dtype=torch.int32).to(torch.uint16).pin_memory() for _ in range(8)]
    seq = [frames[i % len(frames)] for i in range(a.frames)]
    options = {"plain": None, "hdr2sdr_pq_bt709": (16, "bt709")}
    for opt in options.values():
        pipeline_fps(seq[:16], opt, 4)
    fps = {k: [] for k in options}
    for _ in range(a.rounds):
        for k, opt in options.items():
            fps[k].append(pipeline_fps(seq, opt, 4))
    for k, v in fps.items():
        row = dict(step="pipeline_4k_uint16", option=k, batch=4, frames=a.frames, fps_median=round(statistics.median(v), 1),
                   fps_min=round(min(v), 1), fps_max=round(max(v), 1))
        rows.append(row)
        print(json.dumps(row))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "result.json"), "w") as fh:
            json.dump(dict(card=q, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
