#!/usr/bin/env python
"""Throughput of iw3's `mlbw_l2_inpaint` (image mode, both eyes: the mask-MLBW warp with its hole head, the hole mask and
light_inpaint_v1): the engine (nunif_b200.iw3.MLBWInpaint) against PyTorch + cuDNN running the oracle (oracle.mask_mlbw) under fp16
autocast, the reference's CUDA numerics, in the same process with the legs alternating.  Both legs use the engine's MLBW warp
(the oracle's backward warp is CPU code), so the comparison is of the hole mask and the inpainting network.

    python profiles/bench_mlbw_inpaint.py --out DIR

Workloads: 1080p with batch 4 and 4K with batch 1, each with a 392 x 686 depth map (Depth-Anything's output for a 16:9 frame).
Seeded frames and depth maps, divergence 2, convergence 0.5.  WARMUP untimed calls of each leg, then CALLS timed calls of each
(host clock around work that ends in a device synchronise).  Reported: ms per frame (median, min, max), frames/s, the largest
difference between the legs, and - in a separate pass with the engine's event profiler on - ms per kernel class, with the hole
mask kernel (`hole_mask`) against its algorithmic bytes (read h * w * 4, write H * W * 4 per frame and eye).  Also the card's
name, power limit and max SM clock.  Writes result.json.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

WORKLOADS = [("1080p_b4", 4, 1080, 1920), ("4k_b1", 1, 2160, 3840)]
DEPTH_HW = (392, 686)


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,driver_version", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for result.json")
    ap.add_argument("--calls", type=int, default=8)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    from nunif_b200 import synth, _lib
    from nunif_b200.iw3 import MLBW, MLBWInpaint, LightInpaintV1, apply_divergence_nn_delta_weight
    from oracle import light_inpaint as oli
    from oracle import mask_mlbw as omm
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    os.makedirs(args.out, exist_ok=True)
    dev = "cuda:0"
    torch.backends.cudnn.benchmark = True
    lib = _lib.lib()
    sd_inp, sd_mask = synth.light_inpaint_v1_state_dict(0), synth.mask_mlbw_state_dict(0)
    sdc = {k: v.to(dev) for k, v in sd_inp.items()}
    mm = MLBW(sd_mask, dev)
    side = MLBWInpaint(LightInpaintV1(sd_inp, dev), mm, dev)
    result = {"card": card(), "divergence": 2.0, "convergence": 0.5, "depth": list(DEPTH_HW), "workloads": {}}
    for tag, B, H, W in WORKLOADS:
        x = torch.stack([synth.synth_image(100 + i, 3, H, W) for i in range(B)]).to(dev)
        depth = synth.synth_depth(100, B, *DEPTH_HW).to(dev)

        def engine():
            return side.infer(x, depth, 2.0, 0.5)

        def torch_ref():
            # the same warp (the engine's), then the reference's hole mask and network in PyTorch
            left, lm = apply_divergence_nn_delta_weight(mm, x, depth, 2.0, 0.5, 1, -1, return_mask=True)
            right, rm = apply_divergence_nn_delta_weight(mm, x, depth, 2.0, 0.5, 1, 1, return_mask=True)
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
                left = oli.infer(sdc, left.flip(-1), omm.postprocess_hole_mask(lm.flip(-1), (H, W))).flip(-1)
                right = oli.infer(sdc, right, omm.postprocess_hole_mask(rm, (H, W)))
            return left.float(), right.float()

        legs = {"engine": engine, "torch_cudnn_amp": torch_ref}
        times = {k: [] for k in legs}
        outs = {}
        for i in range(args.warmup + args.calls):
            for k, f in legs.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                outs[k] = f()
                torch.cuda.synchronize()
                if i >= args.warmup:
                    times[k].append((time.perf_counter() - t0) * 1e3 / B)
        diff = max(float((a.float() - b.float()).abs().max()) for a, b in zip(outs["engine"], outs["torch_cudnn_amp"]))
        mean = max(float((a.float() - b.float()).abs().mean()) for a, b in zip(outs["engine"], outs["torch_cudnn_amp"]))
        r = {"batch": B, "frame": [3, H, W], "max_abs_engine_vs_amp": diff, "mean_abs_engine_vs_amp": mean}
        for k, ts in times.items():
            med = statistics.median(ts)
            r[k] = {"ms_per_frame": med, "ms_min": min(ts), "ms_max": max(ts), "frames_per_s": 1e3 / med, "calls": len(ts)}
        r["engine_speedup_vs_torch"] = r["torch_cudnn_amp"]["ms_per_frame"] / r["engine"]["ms_per_frame"]
        _lib.check(lib.nb200_profile_enable(1))
        engine()
        buf = ctypes.create_string_buffer(16384)
        _lib.check(lib.nb200_profile_report(buf, 16384))
        _lib.check(lib.nb200_profile_enable(0))
        prof = json.loads(buf.value.decode())
        r["profile"] = prof
        hm = prof.get("hole_mask")
        if hm:
            nbytes = 2 * B * 4.0 * (DEPTH_HW[0] * DEPTH_HW[1] + H * W)          # both eyes
            r["hole_mask_kernel"] = {"launches": hm["launches"], "ms": hm["ms"], "algorithmic_bytes": nbytes,
                                     "achieved_GB_per_s": nbytes / (hm["ms"] / 1e3) / 1e9}
        result["workloads"][tag] = r
        print(tag, json.dumps({k: r[k] for k in ("engine", "torch_cudnn_amp", "engine_speedup_vs_torch", "max_abs_engine_vs_amp",
                                                 "mean_abs_engine_vs_amp")}), flush=True)
        print(tag, "hole_mask", json.dumps(r.get("hole_mask_kernel")), flush=True)
        print(tag, "profile", json.dumps(prof), flush=True)
        del outs, x, depth
        torch.cuda.empty_cache()
    with open(os.path.join(args.out, "result.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
