"""Frames per second of iw3's batch video callback (nunif_b200/iw3/video.py bind_batch_frame_callback) at 1920 x 1080:
Depth-Anything-V2-S (seeded weights) + dilate_edge 2 + forward_fill + full SBS, B = 4 frames per call, frames resident on
the device as float B,3,H,W.

Three arms, alternated round by round in one process:
  ema1    --ema-normalize with buffer 1: the callback keeps the preprocessed float frames;
  ema30   buffer 30 (iw3's --ema-buffer default): every frame waits in the device ring as uint8 until the look-ahead
          releases its depth, and is converted back on release;
  direct  the same per-frame work without a callback (depth model, normalise, warp, SBS), as bench.py's device-resident
          iw3 arm (with_depth_forward_fill) runs it.
Each callback run feeds the whole clip and flushes at its end, so ema30 releases as many frames as it takes in.  A host
clock around each run, which ends in a device synchronise; median, min and max frames/s over ROUNDS rounds are printed
with the card and its power limit.
    python profiles/bench_iw3_video.py [--frames 96] [--rounds 5]
"""
import argparse
import os
import statistics
import subprocess
import sys
import time
from argparse import Namespace

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nunif_b200 import synth  # noqa: E402
from nunif_b200.iw3 import DepthAnythingModel, bind_batch_frame_callback, stereo_sbs  # noqa: E402

H, W, B = 1080, 1920, 4


def make_args(dev):
    return Namespace(method="forward_fill", divergence=2.0, convergence=0.5, synthetic_view="both", ipd_offset=0, mapper="none",
                     edge_dilation=2, tta=False, low_vram=False, disable_amp=False, depth_aa=False, rotate_left=False,
                     rotate_right=False, max_output_height=None, max_output_width=None, keep_aspect_ratio=False, pad=None,
                     pad_mode=None, vr180=False, half_sbs=False, tb=False, half_tb=False, cross_eyed=False, anaglyph=None,
                     rgbd=False, half_rgbd=False, debug_depth=False, preserve_screen_border=False, pix_fmt="yuv420p",
                     batch_size=B, cuda_stream=False, state={"device": dev, "convergence_model": None})


def main():
    p = argparse.ArgumentParser()
    p.add_argument("--frames", type=int, default=96)
    p.add_argument("--rounds", type=int, default=5)
    opt = p.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    print("card:", q)
    dev = torch.device("cuda:0")
    dm = DepthAnythingModel("Any_V2_S").load_state_dict(synth.depth_anything_v2_state_dict(0), gpu=0)
    src = torch.stack([synth.synth_image(50 + i, 3, H, W, smooth=False) for i in range(8)]).to(dev)
    clip = [src[(i * B) % 8:(i * B) % 8 + B] for i in range(opt.frames // B)]
    args = make_args(dev)

    def run_callback(buffer_size):
        if buffer_size == 1:
            dm.disable_ema()
        else:
            dm.enable_ema(decay=0.9, buffer_size=buffer_size)
        cb = bind_batch_frame_callback(dm, None, set(), args)
        n = 0
        for i, x in enumerate(clip):
            y = cb(x, list(range(i * B, (i + 1) * B)), False)
            n += 0 if y is None else y.shape[0]
        y = cb(None, None, True)
        n += 0 if y is None else y.shape[0]
        assert n == len(clip) * B, n
        return n

    def run_direct():
        dm.disable_ema()
        with torch.inference_mode():
            for x in clip:
                depth = dm.infer(x, edge_dilation=2)
                stereo_sbs(x, depth, 2.0, 0.5, method="forward_fill", edge_dilation=0)
        return len(clip) * B

    arms = {"ema1": lambda: run_callback(1), "ema30": lambda: run_callback(30), "direct": run_direct}
    for fn in arms.values():           # warm every shape
        fn()
    torch.cuda.synchronize()
    fps = {k: [] for k in arms}
    for _ in range(opt.rounds):
        for name, fn in arms.items():
            torch.cuda.synchronize()
            t0 = time.perf_counter()
            n = fn()
            torch.cuda.synchronize()
            fps[name].append(n / (time.perf_counter() - t0))
    print(f"1080p, B = {B}, {len(clip) * B} frames per run, {opt.rounds} rounds (frames/s: median [min, max])")
    for name, v in fps.items():
        print(f"  {name:7s} {statistics.median(v):8.1f}  [{min(v):.1f}, {max(v):.1f}]")
    med = {k: statistics.median(v) for k, v in fps.items()}
    print(f"  ema30 / ema1 = {med['ema30'] / med['ema1']:.3f}, ema1 / direct = {med['ema1'] / med['direct']:.3f}")


if __name__ == "__main__":
    main()
