"""Auto-convergence (--convergence-mode sod_v1) on the engine against PyTorch + cuDNN running oracle/sod.py under fp16 autocast:
ms per frame of the whole estimator (SODV1.infer + depth_position_from_ratio), alternating the two, at B = 4 and 8 on 1080p and
4K frames with a 392 x 686 depth map.  Prints the card and its power limit, the network FLOPs from shapes, the achieved rate
and the engine's launches per call.  Results go to stdout and, with --out, to DIR/result.json.
    python profiles/bench_sod_convergence.py [--iters 20] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nunif_b200 import synth, _lib  # noqa: E402
from nunif_b200.iw3 import ConvergenceEstimator  # noqa: E402
from oracle import sod as osod  # noqa: E402


def flops_per_frame():
    """2 * MACs of every conv at its level (192 >> level) for U2NETP(in_ch=6); side and head convs included."""
    total, S = 0, 192
    for stage, n, _ in synth.SOD_STAGES:
        lvl = {"stage1": 0, "stage2": 1, "stage3": 2, "stage4": 3, "stage5": 4, "stage6": 5, "stage5d": 4, "stage4d": 3,
               "stage3d": 2, "stage2d": 1, "stage1d": 0}[stage]
        s = S >> lvl
        for name, cin, cout, _ in synth.sod_rebnconvs():
            if f".{stage}." not in name:
                continue
            k = name.rsplit("rebnconv", 1)[1].rstrip("d")
            depth = 0 if (n == 0 or k in ("in", "1")) else min(int(k), n - 1) - 1
            ss = s >> depth
            total += 2 * ss * ss * 9 * cin * cout
    total += sum(2 * (S >> l) ** 2 * 9 * 64 for l in range(6)) + 2 * S * S * 6
    return total


def timed(fn, iters):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(iters):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / iters


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--out", default=None, help="directory for result.json")
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    print("card:", q)
    dev = "cuda:0"
    sd = synth.sod_v1_state_dict(0)
    sdc = {k: v.to(dev) for k, v in sd.items()}
    est = ConvergenceEstimator(0.5, 0, state_dict=sd)
    F = flops_per_frame()
    print(f"network FLOPs per frame: {F / 1e9:.3f} G")
    rows = []
    for (H, W) in ((1080, 1920), (2160, 3840)):
        for B in (4, 8):
            rgb = torch.rand(B, 3, H, W, device=dev)
            d = synth.synth_depth(1, B, 392, 686).to(dev)

            def eng():
                est(rgb, d)

            def ref():
                with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
                    s, d192 = osod.sod_infer(sdc, rgb, d)
                osod.depth_position(s, d192, 0.5)

            for f in (eng, ref):
                f(); f()
            torch.cuda.synchronize()
            n0 = _lib.lib().nb200_launch_count()
            eng()
            launches = _lib.lib().nb200_launch_count() - n0
            te = tr = 0.0
            for _ in range(3):       # alternate the two
                te += timed(eng, a.iters) / 3
                tr += timed(ref, a.iters) / 3
            row = dict(H=H, W=W, B=B, engine_ms_per_frame=te / B, torch_ms_per_frame=tr / B, speedup=tr / te,
                       engine_tflops=F * B / (te * 1e-3) / 1e12, launches_per_call=int(launches))
            rows.append(row)
            print(json.dumps(row))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "result.json"), "w") as fh:
            json.dump(dict(card=q, flops_per_frame=F, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
