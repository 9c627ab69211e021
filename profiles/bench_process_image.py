"""The frame steps of iw3's process_image on the engine: us per frame of the autocrop detector (nb200_autocrop_detect, both
axes, black and flat modes), of rot90 (--rotate-left) and of the --max-output-height pre-resize 2160 -> 1080 (bicubic,
antialias, align_corners=True), at 1080p and 4K.  GB/s is against the floor of one fp32 read of the RGB frame (12 B/px: at
4K 99.5 MB, about 30 us at the H100 SXM data-sheet 3.35 TB/s); the detector reads it once for the rows and once for the
columns, rot90 also writes it once.  Steps are timed round-robin, ROUNDS times; the median and the spread over the rounds
are printed.  Prints the card and its power limit.  Results go to stdout and, with --out, to DIR/result.json.
    python profiles/bench_process_image.py [--iters 100] [--rounds 5] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nunif_b200 import synth, _lib  # noqa: E402

SHAPES = {"1080p": (1080, 1920), "4k": (2160, 3840)}


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
    ap.add_argument("--iters", type=int, default=100)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for result.json")
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    print("card:", q)
    dev = "cuda:0"
    L = _lib.lib()
    st = _lib.stream_ptr()
    rows = []
    for tag, (H, W) in SHAPES.items():
        x = synth.letterbox_frame(1, H, W, H // 8, H // 8, W // 16, W // 16, "tv").to(dev)
        count_tb = torch.zeros(H, dtype=torch.int32, device=dev)
        count_lr = torch.zeros(W, dtype=torch.int32, device=dev)
        rot = torch.empty(3, W, H, device=dev)
        calls = {
            "detect_black": lambda: _lib.check(L.nb200_autocrop_detect(_lib.ptr(x), 1, H, W, 1, 3, None, None, _lib.ptr(count_tb),
                                                                       _lib.ptr(count_lr), None, None, st)),
            "detect_flat": lambda: _lib.check(L.nb200_autocrop_detect(_lib.ptr(x), 1, H, W, 0, 3, None, None, _lib.ptr(count_tb),
                                                                      _lib.ptr(count_lr), None, None, st)),
            "rot90": lambda: _lib.check(L.nb200_rot90(_lib.ptr(x), 3, H, W, 1, _lib.ptr(rot), st)),
        }
        if H == 2160:
            out = torch.empty(3, 1080, 1920, device=dev)
            calls["resize_2160_to_1080"] = lambda: _lib.check(L.nb200_resize_bicubic_aa_ac(_lib.ptr(x), 3, H, W, 1080, 1920, 1, 1,
                                                                                          _lib.ptr(out), st))
        for f in calls.values():
            f(); f()
        torch.cuda.synchronize()
        samples = {k: [] for k in calls}
        for _ in range(a.rounds):
            for k, f in calls.items():
                samples[k].append(timed(f, a.iters))
        floor_bytes = 12.0 * H * W
        for step, us in samples.items():
            med = statistics.median(us)
            row = dict(shape=tag, H=H, W=W, step=step, us_median=round(med, 2), us_min=round(min(us), 2), us_max=round(max(us), 2),
                       gbps_vs_one_read=round(floor_bytes / (med * 1e-6) / 1e9, 1))
            rows.append(row)
            print(json.dumps(row))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "result.json"), "w") as fh:
            json.dump(dict(card=q, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
