#!/usr/bin/env python
"""Throughput of the learned row-flow stereo warps on 1080p frames with a 392 x 686 depth map (what Depth-Anything-V2 at
lower_bound = 392 gives for 16:9), batch 4: the engine against PyTorch + cuDNN running the oracle under fp16 autocast (the
reference's CUDA numerics), in the same process, alternating call by call after warm-up.

    python profiles/bench_row_flow.py --out DIR

Rows:
  v2_delta       the sbs.row_flow_v2 delta network alone (ms, and TFLOP/s from 33,152 FLOP per depth pixel)
  v2_lr          apply_divergence_nn_LR with row_flow_v2, both eyes
  v3_sym_lr      apply_divergence_nn_LR with row_flow_v3_sym (one delta, both eyes in one warp), both eyes
  v3_lr          apply_divergence_nn_LR with row_flow_v3, both eyes (the reference point of the symmetric model's "2x")
Each row: ms per call (median, min, max) of each leg, the engine's speed-up, and the fraction of 8-bit output samples that
differ between the two legs (for v2_delta: the max |delta| difference).  Also the card's name, power limit and max SM clock,
read in the same run.  Writes result.json.
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

B, H, W, h, w = 4, 1080, 1920, 392, 686
V2_FLOP_PER_PIXEL = 2 * (144 + 16 + 2304 + 4608 + 9216 + 288)   # MACs x 2 = 33,152 FLOP


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,driver_version", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for result.json")
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--warmup", type=int, default=3)
    args = ap.parse_args()
    import torch
    from nunif_b200 import synth
    from nunif_b200.iw3 import RowFlowV2, RowFlowV3, apply_divergence_nn_LR
    from nunif_b200.iw3.row_flow import make_input
    from oracle import row_flow as orf, row_flow_v2 as orf2
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    os.makedirs(args.out, exist_ok=True)
    dev = "cuda:0"
    torch.backends.cudnn.benchmark = True
    c = torch.stack([synth.synth_image(500 + i, 3, H, W) for i in range(B)]).to(dev)
    d = synth.synth_depth(510, B, h, w).to(dev)
    sd2, sd3s, sd3 = synth.row_flow_v2_state_dict(0), synth.row_flow_v3_state_dict(2), synth.row_flow_v3_state_dict(0)
    m2, m3s, m3 = RowFlowV2(sd2, dev), RowFlowV3(sd3s, dev, symmetric=True), RowFlowV3(sd3, dev)
    sdc2, sdc3s, sdc3 = ({k: v.to(dev) for k, v in s.items()} for s in (sd2, sd3s, sd3))
    x = make_input(d, 2.0, 0.5)

    def amp(fn, sdc, cast):
        def f(xx):
            with torch.autocast("cuda", dtype=torch.float16):
                y = fn(sdc, xx)
            return y.float() if cast else y
        return f

    def v3_ref_lr(sdc):
        def f():
            return orf2.apply_divergence_nn_delta_LR(amp(orf.row_flow_delta, sdc, True), c, d, 2.0, 0.5)
        return f

    rows = {
        "v2_delta": {"engine": lambda: m2.delta_x(x), "torch_cudnn_amp": lambda: amp(orf2.row_flow_v2_delta, sdc2, False)(x).float()},
        "v2_lr": {"engine": lambda: apply_divergence_nn_LR(m2, c, d, 2.0, 0.5),
                  "torch_cudnn_amp": lambda: orf2.apply_divergence_nn_delta_LR(amp(orf2.row_flow_v2_delta, sdc2, False), c, d, 2.0, 0.5)},
        "v3_sym_lr": {"engine": lambda: apply_divergence_nn_LR(m3s, c, d, 2.0, 0.5),
                      "torch_cudnn_amp": lambda: orf2.apply_divergence_nn_symmetric(amp(orf.row_flow_delta, sdc3s, True), c, d, 2.0, 0.5)},
        "v3_lr": {"engine": lambda: apply_divergence_nn_LR(m3, c, d, 2.0, 0.5), "torch_cudnn_amp": v3_ref_lr(sdc3)},
    }
    result = {"card": card(), "batch": B, "frame": [3, H, W], "depth": [h, w], "v2_flop_per_depth_pixel": V2_FLOP_PER_PIXEL,
              "rows": {}}
    with torch.no_grad():
        for name, legs in rows.items():
            times = {k: [] for k in legs}
            outs = {}
            for i in range(args.warmup + args.iters):
                for k, f in legs.items():
                    torch.cuda.synchronize()
                    t0 = time.perf_counter()
                    outs[k] = f()
                    torch.cuda.synchronize()
                    if i >= args.warmup:
                        times[k].append((time.perf_counter() - t0) * 1e3)
            r = {}
            for k, ts in times.items():
                med = statistics.median(ts)
                r[k] = {"ms": med, "ms_min": min(ts), "ms_max": max(ts), "iters": len(ts)}
                if name == "v2_delta":
                    r[k]["tflop_per_s"] = V2_FLOP_PER_PIXEL * B * h * w / (med / 1e3) / 1e12
            r["engine_speedup_vs_torch"] = r["torch_cudnn_amp"]["ms"] / r["engine"]["ms"]
            a, b = outs["engine"], outs["torch_cudnn_amp"]
            if name == "v2_delta":
                r["max_abs_delta_engine_vs_amp"] = float((a - b).abs().max())
                r["frac_delta_differs"] = float((a != b).double().mean())
            else:
                qa = torch.cat([(e * 255).round().clamp(0, 255) for e in a])
                qb = torch.cat([(e * 255).round().clamp(0, 255) for e in b])
                r["q8_mismatch_engine_vs_amp"] = float((qa != qb).double().mean())
                r["max_abs_engine_vs_amp"] = float(max((ea - eb).abs().max() for ea, eb in zip(a, b)))
            result["rows"][name] = r
            print(name, json.dumps(r), flush=True)
            del outs, a, b
            torch.cuda.empty_cache()
    with open(os.path.join(args.out, "result.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
