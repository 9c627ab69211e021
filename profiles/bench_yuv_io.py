"""YUV frame I/O on the H100.

kernels   ms per frame of yuv_to_rgb / rgb_to_yuv (csrc/yuv.cu) at 1920x1080 in, 3840x1080 (SBS out) and 3840x2160, 8-bit
          (yuv420p <-> rgb24) and 10-bit (yuv420p10le <-> rgb48), B = 4, CUDA events over ITERS calls, median of ROUNDS.
          Bytes are the planes read plus the HWC frame written (or the reverse); their rate is set against the H100 SXM
          data-sheet 3.35 TB/s.
pipeline  iw3 1080p as bench.py's iw3_1080p row (Depth-Anything-V2-S seeded weights, forward_fill, SBS, B = 4) from host
          frames through FrameBatchPipeline: rgb24 frames in and out, against yuv420p BT.709 planes in and out
          (source= / target=), alternated in the same run.  H2D and D2H bytes per frame of each.
host      CPU ms per frame of cv2.cvtColor RGB <-> I420 at the same sizes, one thread: a stand-in for the libswscale work
          that the reference does per frame on the host and that these stages move to the GPU (not swscale itself).
Prints the card name, power limit and max SM clock, then one JSON line.
    python profiles/bench_yuv_io.py [--iters 50] [--rounds 5] [--frames 200] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

import bench  # noqa: E402
from nunif_b200.nunif.video import FrameBatchPipeline, plane_shape, rgb_to_yuv, yuv_to_rgb  # noqa: E402

PEAK_BPS = 3.35e12
SIZES = {"1080p": (1080, 1920), "sbs1080p": (1080, 3840), "4k": (2160, 3840)}
B = 4


def card():
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def timed(fn, iters):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(iters):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / iters


def kernels(iters, rounds):
    out = {}
    for name, (H, W) in SIZES.items():
        for bits, pix_fmt in ((8, "yuv420p"), (10, "yuv420p10le")):
            dt = torch.uint16 if bits > 8 else torch.uint8
            rgb = torch.randint(0, 1 << (16 if bits > 8 else 8), (B, H, W, 3), dtype=torch.int32, device="cuda").to(dt)
            planes = rgb_to_yuv(rgb, pix_fmt, 1, 1)
            fns = {"yuv_to_rgb": lambda: yuv_to_rgb(planes, pix_fmt, 1, 1, use_16bit=bits > 8),
                   "rgb_to_yuv": lambda: rgb_to_yuv(rgb, pix_fmt, 1, 1)}
            nbytes = (planes[0].numel() + rgb[0].numel()) * rgb.element_size()
            for fn in fns.values():
                timed(fn, 3)
            ms = {k: [] for k in fns}
            for _ in range(rounds):
                for k, fn in fns.items():
                    ms[k].append(timed(fn, iters) / B)
            for k, v in ms.items():
                med = statistics.median(v)
                out[f"{k}/{name}/{bits}bit"] = {"ms_per_frame": med, "spread_ms": [min(v), max(v)], "bytes_per_frame": nbytes,
                                                "share_of_3.35TBps": nbytes / (med / 1e3) / PEAK_BPS}
    return out


def pipeline(n_frames):
    wl = bench.IW3_WORKLOADS["iw3_1080p"]
    dev = torch.device("cuda:0")
    H, W = bench.FRAME[wl["frame"]]
    _, dm = bench._iw3_models(wl, dev)
    from nunif_b200 import synth
    from nunif_b200.iw3 import stereo_sbs

    def frames_to_stereo(xf):
        depth = dm.infer(xf, edge_dilation=wl["edge_dilation"])
        return stereo_sbs(xf, depth, 2.0, 0.5, method=wl["method"], mapper=wl["mapper"], edge_dilation=0, anaglyph=wl["anaglyph"])

    c = torch.stack([synth.synth_image(50 + i, 3, H, W, smooth=False) for i in range(B)]).to(dev)
    u8 = (c.permute(0, 2, 3, 1) * 255.0).round().to(torch.uint8).contiguous()
    host = {"rgb24": [f.cpu().pin_memory() for f in u8],
            "yuv420p": [p.cpu().pin_memory() for p in rgb_to_yuv(u8, "yuv420p", 1, 1)]}
    fmt = ("yuv420p", 1, 1)
    kw = {"rgb24": {}, "yuv420p": {"source": fmt, "target": fmt}}
    pipes = {k: FrameBatchPipeline(frames_to_stereo, B, dev, depth=3, copy_output=False, **v) for k, v in kw.items()}
    res = {k: [] for k in kw}
    out_shape = {}
    for _ in range(3):
        for k, pipe in pipes.items():
            fr = host[k]
            got = 0
            for _ in range(3 * B):
                got += len(pipe(fr[got % B]))
            got += len(pipe.finish())
            t0 = time.perf_counter()
            done = 0
            for i in range(n_frames):
                out = pipe(fr[i % B])
                done += len(out)
                if out:
                    out_shape[k] = tuple(out[-1].shape)
            done += len(pipe.finish())
            torch.cuda.synchronize()
            res[k].append(n_frames / (time.perf_counter() - t0))
            assert done == n_frames
    o_h, o_w = H, 2 * W
    return {k: {"frames_per_s": statistics.median(v), "runs": v,
                "h2d_bytes_per_frame": host[k][0].numel() * host[k][0].element_size(),
                "d2h_bytes_per_frame": int(np.prod(out_shape[k])),
                "out_frame_shape": out_shape[k]} for k, v in res.items()} | {"sbs_out": [o_h, o_w]}


def host_cost(reps):
    import cv2
    cv2.setNumThreads(1)
    out = {}
    for name, (H, W) in SIZES.items():
        rgb = np.random.default_rng(0).integers(0, 256, (H, W, 3), dtype=np.uint8)
        i420 = cv2.cvtColor(rgb, cv2.COLOR_RGB2YUV_I420)
        for k, fn in (("rgb_to_i420", lambda: cv2.cvtColor(rgb, cv2.COLOR_RGB2YUV_I420)),
                      ("i420_to_rgb", lambda: cv2.cvtColor(i420, cv2.COLOR_YUV2RGB_I420))):
            fn()
            t0 = time.perf_counter()
            for _ in range(reps):
                fn()
            out[f"{k}/{name}"] = {"cpu_ms_per_frame": (time.perf_counter() - t0) / reps * 1e3}
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=50)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--frames", type=int, default=200)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_yuv_io needs a CUDA device")
    info = card()
    print("card, power limit, max SM clock:", info)
    res = {"card": info, "plane_shape_1080p_yuv420p": plane_shape("yuv420p", 1080, 1920)}
    res["kernels"] = kernels(a.iters, a.rounds)
    for k, v in res["kernels"].items():
        print(f"{k:32s} {v['ms_per_frame'] * 1e3:8.1f} us/frame  {v['bytes_per_frame'] / 1e6:6.2f} MB  "
              f"{v['share_of_3.35TBps'] * 100:5.1f} % of 3.35 TB/s")
    res["pipeline_iw3_1080p"] = pipeline(a.frames)
    for k, v in res["pipeline_iw3_1080p"].items():
        if k != "sbs_out":
            print(f"pipeline {k:8s} {v['frames_per_s']:7.1f} frames/s  H2D {v['h2d_bytes_per_frame']} B/frame  "
                  f"D2H {v['d2h_bytes_per_frame']} B/frame  runs {[round(r) for r in v['runs']]}")
    try:
        res["host_cv2_stand_in"] = host_cost(20)
        for k, v in res["host_cv2_stand_in"].items():
            print(f"cv2 {k:24s} {v['cpu_ms_per_frame']:7.2f} CPU ms/frame (1 thread; stand-in for libswscale)")
    except ImportError as e:
        res["host_cv2_stand_in"] = f"not measured: {e}"
    line = json.dumps(res)
    print(line)
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "bench_yuv_io.json"), "w") as fh:
            fh.write(line + "\n")


if __name__ == "__main__":
    main()
