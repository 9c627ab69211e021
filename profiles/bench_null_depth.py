#!/usr/bin/env python
"""The stereo stage of iw3 measured alone: frames per second of the per-frame path with the NULL depth model
(--depth-model NULL, nunif_b200/iw3/null_depth_model.py) in place of a depth network, and the NULL kernel's own time.

Path: bind_batch_frame_callback (nunif_b200/iw3/video.py) with EMA off, edge_dilation 2 and full SBS output, fed B,3,H,W float
frames already resident in HBM: NULL depth (392 x 392) -> dilate_edge -> per-frame min/max -> warp -> postprocess_image.
Methods forward_fill, backward, row_flow_v3 and mlbw_l2 (the learned warps on seeded weights) at 1080p B = 4 and 4K B = 2.
Each run feeds --batches batches; a host clock around the run, which ends in a device synchronise; the methods are
alternated run by run after one warm-up run each, and the median, min and max over --rounds rounds are reported.

NULL kernel: CUDA events around --iters launches of nb200_null_depth at each shape.  Its byte floor is the least DRAM traffic
the resize needs, computed here from the shapes: every 32-byte sector of the frames that holds a bilinear tap (ATen's
source-index rule), read once, plus the fp32 output written once.  The time floor divides it by the H100 SXM data-sheet
3.35 TB/s (a figure for a card allowed 700 W, not a measured one).

The card's name, power limit and max SM clock are read in the same run.  Prints one JSON line.
    python profiles/bench_null_depth.py [--batches 16] [--rounds 5] [--iters 200]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time
from argparse import Namespace

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nunif_b200 import synth  # noqa: E402
from nunif_b200.iw3 import MLBW, NullDepthModel, RowFlowV3, bind_batch_frame_callback  # noqa: E402

SHAPES = {"1080p": (4, 1080, 1920), "4k": (2, 2160, 3840)}
METHODS = ("forward_fill", "backward", "row_flow_v3", "mlbw_l2")
R = 392
HBM_BYTES_PER_S = 3.35e12           # H100 SXM data sheet


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True)
    return {"torch_device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def tap_index(n_in, n_out):
    """ATen's bilinear source indices i0, i1 (align_corners=False) for every output index, in fp32 as on the device."""
    s = np.float32(n_in) / np.float32(n_out)
    r = (s.astype(np.float64) * (np.arange(n_out, dtype=np.float32) + np.float32(0.5)) - 0.5).astype(np.float32)
    i0 = np.maximum(r, 0).astype(np.int64)
    return i0, i0 + (i0 < n_in - 1)


def null_depth_bytes(B, H, W):
    """(bytes read, bytes written): the 32-byte sectors of the B,3,H,W fp32 frames that hold a tap, and the B,1,R,R output."""
    rows = np.unique(np.concatenate(tap_index(H, R)))
    cols = np.unique(np.concatenate(tap_index(W, R)))
    sectors = 0
    for r in rows:
        sectors += np.unique((r * W + cols) * 4 // 32).size
    return int(sectors) * 32 * 3 * B, B * R * R * 4


def make_args(method, batch_size, dev):
    return Namespace(method=method, divergence=2.0, convergence=0.5, synthetic_view="both", ipd_offset=0, mapper="none",
                     edge_dilation=2, tta=False, low_vram=False, disable_amp=False, depth_aa=False, rotate_left=False,
                     rotate_right=False, max_output_height=None, max_output_width=None, keep_aspect_ratio=False, pad=None,
                     pad_mode=None, vr180=False, half_sbs=False, tb=False, half_tb=False, cross_eyed=False, anaglyph=None,
                     rgbd=False, half_rgbd=False, debug_depth=False, preserve_screen_border=False, pix_fmt="yuv420p",
                     batch_size=batch_size, cuda_stream=False, stereo_width=None, warp_steps=None,
                     state={"device": dev, "convergence_model": None})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--batches", type=int, default=16, help="batches per timed run")
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--iters", type=int, default=200, help="launches per NULL kernel timing")
    opt = ap.parse_args()
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    dev = torch.device("cuda:0")
    result = {"card": card(), "resolution": R, "edge_dilation": 2, "output": "sbs", "batches_per_run": opt.batches,
              "rounds": opt.rounds, "fps": {}, "null_kernel": {}}
    dm = NullDepthModel("NULL").load(gpu=0, resolution=R)
    dm.disable_ema()
    side = {"row_flow_v3": RowFlowV3(synth.row_flow_v3_state_dict(0), dev), "mlbw_l2": MLBW(synth.mlbw_state_dict(0, num_layers=2), dev)}
    for shape, (B, H, W) in SHAPES.items():
        src = torch.stack([synth.synth_image(60 + i, 3, H, W, smooth=True) for i in range(2 * B)]).to(dev)
        batches = [src[(i % 2) * B:(i % 2 + 1) * B] for i in range(opt.batches)]

        def run(method):
            cb = bind_batch_frame_callback(dm, side.get(method), set(), make_args(method, B, dev))
            n = 0
            for i, x in enumerate(batches):
                y = cb(x, list(range(i * B, (i + 1) * B)), False)
                n += y.shape[0]
            assert cb(None, None, True) is None and n == len(batches) * B
            return n

        for m in METHODS:               # warm every method at this shape
            run(m)
        torch.cuda.synchronize()
        fps = {m: [] for m in METHODS}
        for _ in range(opt.rounds):
            for m in METHODS:
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                n = run(m)
                torch.cuda.synchronize()
                fps[m].append(n / (time.perf_counter() - t0))
        result["fps"][shape] = {m: {"median": statistics.median(v), "min": min(v), "max": max(v)} for m, v in fps.items()}

        net = dm.get_model()
        x = src[:B].contiguous()
        for _ in range(10):
            net(x)
        ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
        ev[0].record()
        for _ in range(opt.iters):
            net(x)
        ev[1].record()
        torch.cuda.synchronize()
        us = ev[0].elapsed_time(ev[1]) * 1e3 / opt.iters
        rd, wr = null_depth_bytes(B, H, W)
        floor_us = (rd + wr) / HBM_BYTES_PER_S * 1e6
        result["null_kernel"][shape] = {"B": B, "frame": [3, H, W], "us": us, "floor_bytes_read": rd, "floor_bytes_written": wr,
                                        "frame_bytes": B * 3 * H * W * 4, "floor_us_at_3.35TB/s": floor_us,
                                        "achieved_GB/s_of_floor_bytes": (rd + wr) / (us * 1e-6) / 1e9,
                                        "floor_over_time": floor_us / us}
        del src, batches, x
        torch.cuda.empty_cache()
    print(json.dumps(result))


if __name__ == "__main__":
    main()
