#!/usr/bin/env python
"""Throughput of iw3's `forward_inpaint` (image mode, both eyes: forward warp + mask chain + light_inpaint_v1): the engine
(nunif_b200.iw3.ForwardInpaint) against PyTorch + cuDNN running the oracle (oracle.light_inpaint.forward_inpaint) under fp16
autocast, the reference's CUDA numerics, in the same process with the legs alternating.  Both legs use the engine's forward
warp (the oracle's warp is CPU code), so the comparison is of the mask chain and the network.

    python profiles/bench_forward_inpaint.py --out DIR

Workloads: 1080p with batch 4 and 4K with batch 1 (what a user converting video frames or photos runs).  Seeded frames and box
depth maps (holes behind every box edge), divergence 2, convergence 0.5.  WARMUP untimed calls of each leg, then CALLS timed calls
of each (host clock around work that ends in a device synchronise).  Reported: ms per frame (median, min, max), frames/s,
TFLOP/s of the two network forwards per frame (oracle.light_inpaint.flops: 233 GFLOP per eye at 1080p, 905 at 4K), the
largest difference between the legs, and - in a separate pass with the engine's event profiler on - ms per kernel class.
Also the card's name, power limit and max SM clock.  Writes result.json.
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
    from nunif_b200.iw3 import ForwardInpaint, LightInpaintV1, apply_divergence_forward_warp
    from oracle import light_inpaint as oli
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    os.makedirs(args.out, exist_ok=True)
    dev = "cuda:0"
    torch.backends.cudnn.benchmark = True
    lib = _lib.lib()
    sd = synth.light_inpaint_v1_state_dict(0)
    sdc = {k: v.to(dev) for k, v in sd.items()}
    fi = ForwardInpaint(LightInpaintV1(sd, dev), dev)
    result = {"card": card(), "divergence": 2.0, "convergence": 0.5, "workloads": {}}
    for tag, B, H, W in WORKLOADS:
        x = torch.stack([synth.synth_image(100 + i, 3, H, W) for i in range(B)]).to(dev)
        depth = synth.synth_depth(100, B, H, W).to(dev)
        flop = 2 * oli.flops(H, W) * B

        def engine():
            return fi.infer(x, depth, 2.0, 0.5)

        def torch_ref():
            # the same warp (the engine's; oracle.iw3's is CPU code), then the reference's mask chain and network in PyTorch
            left, right, lm, rm = apply_divergence_forward_warp(x, depth, 2.0, 0.5, return_mask=True, width_base=False)
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
                return (oli.forward_left(sdc, left, lm, 0, 0, W).float(), oli.forward_right(sdc, right, rm, 0, 0, W).float())

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
        r = {"batch": B, "frame": [3, H, W], "tflop_per_frame": flop / B / 1e12, "max_abs_engine_vs_amp": diff}
        for k, ts in times.items():
            med = statistics.median(ts)
            r[k] = {"ms_per_frame": med, "ms_min": min(ts), "ms_max": max(ts), "frames_per_s": 1e3 / med,
                    "tflop_per_s": flop / B / 1e12 / (med / 1e3), "calls": len(ts)}
        r["engine_speedup_vs_torch"] = r["torch_cudnn_amp"]["ms_per_frame"] / r["engine"]["ms_per_frame"]
        _lib.check(lib.nb200_profile_enable(1))
        engine()
        buf = ctypes.create_string_buffer(8192)
        _lib.check(lib.nb200_profile_report(buf, 8192))
        _lib.check(lib.nb200_profile_enable(0))
        r["profile"] = json.loads(buf.value.decode())
        result["workloads"][tag] = r
        print(tag, json.dumps({k: r[k] for k in ("engine", "torch_cudnn_amp", "engine_speedup_vs_torch", "max_abs_engine_vs_amp")}),
              flush=True)
        print(tag, "profile", json.dumps(r["profile"]), flush=True)
        del outs, x, depth
        torch.cuda.empty_cache()
    with open(os.path.join(args.out, "result.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
