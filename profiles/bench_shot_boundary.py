"""Scene detection (iw3 --scene-detect) on the engine against PyTorch running oracle/transnetv2.py with torch's default GPU
settings (TF32 convolutions, fp32 linears), one window per forward and one host sync per window as the reference does:
  * frames/s of the whole detector over N seeded 27 x 48 uint8 frames (host frames in, segment set out), the two alternated;
  * network ms per 100-frame window at B = 1 and batched (B = 8).
Prints the card, its power limit and max SM clock, and the FLOPs from shapes.  With --out, also DIR/result.json.
    python profiles/bench_shot_boundary.py [--frames 10000] [--reps 3] [--out DIR]
"""
import argparse
import json
import os
import subprocess
import sys
import time
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nunif_b200 import synth  # noqa: E402
from nunif_b200.nunif.transnetv2 import TransNetV2  # noqa: E402
from nunif_b200.nunif.shot_boundary_detection import detect_boundary  # noqa: E402
from oracle import transnetv2 as otn  # noqa: E402

DEV = "cuda:0"


def flops_per_window_frame():
    """2 * MACs per frame of one window: the (1,3,3) and (3,1,1) convs, the projections, fc1 and the heads."""
    total, h, w = 0, 27, 48
    for s in range(3):
        F = 16 << s
        for j in range(2):
            cin = 4 * F if j == 1 else (3 if s == 0 else 2 * F)
            total += 2 * h * w * (9 * cin * 8 * F + 4 * 3 * 2 * F * F)
        h, w = h // 2, w // 2
    return total + 2 * (448 * 128 + 2 * 101 * 128 + 4864 * 1024 + 2 * 1024)


def reference_detect(frames, pts, sd):
    """The reference's loop with the oracle network: per window, upload, forward, sigmoid and .cpu()."""
    probs, kept = [], []
    for w in otn.windows(pts):
        x = torch.from_numpy(frames[w]).to(DEV).permute(0, 3, 1, 2).float() / 255
        with torch.inference_mode():
            p = torch.sigmoid(otn.forward(sd, x.unsqueeze(0))[0][0])[25:75].cpu()
        probs.append(p)
        kept += [pts[i] for i in w[25:75]]
    prob = torch.cat(probs)[:len(pts)]
    return set(p for p, q in zip(kept[:len(pts)], (prob > 0.5).tolist()) if q)


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
    ap.add_argument("--frames", type=int, default=10000)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    card = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                          capture_output=True, text=True).stdout.strip()
    print("card:", card)
    # torch's default precision, as the reference runs: TF32 cuDNN convolutions, fp32 matmuls
    torch.backends.cuda.matmul.allow_tf32, torch.backends.cudnn.allow_tf32 = False, True
    sd = synth.transnetv2_state_dict(0)
    sdg = {k: v.to(DEV) for k, v in sd.items()}
    model = TransNetV2(sd, DEV)
    frames = np.concatenate([synth.shot_sequence(1000 + k, 1000) for k in range(args.frames // 1000)])
    n = frames.shape[0]
    pts = [1001 * i + 7 for i in range(n)]
    fpf = flops_per_window_frame()
    print(f"{n} frames; {fpf / 1e9:.3f} GFLOP per window-frame, {2 * fpf / 1e9:.3f} per output frame (windows overlap 2x)")

    # warm-up of both paths (module load, cuDNN algorithm choice)
    e_set = detect_boundary(zip(frames[:300], pts[:300]), device=DEV, model=model)
    r_set = reference_detect(frames[:300], pts[:300], sdg)
    res = {"card": card, "frames": n, "gflop_per_window_frame": fpf / 1e9, "engine_fps": [], "torch_fps": []}
    for _ in range(args.reps):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        e_set = detect_boundary(zip(frames, pts), device=DEV, model=model)
        t1 = time.perf_counter()
        r_set = reference_detect(frames, pts, sdg)
        t2 = time.perf_counter()
        res["engine_fps"].append(n / (t1 - t0))
        res["torch_fps"].append(n / (t2 - t1))
        print(f"detector frames/s: engine {n / (t1 - t0):.0f}  pytorch {n / (t2 - t1):.0f}")
    res["sets_equal"] = e_set == r_set
    res["set_sizes"] = [len(e_set), len(r_set), len(e_set ^ r_set)]
    print(f"segment sets: engine {len(e_set)}, pytorch {len(r_set)}, symmetric difference {len(e_set ^ r_set)}")

    x = torch.from_numpy(frames[:800]).to(DEV).permute(0, 3, 1, 2).float().div(255).view(8, 100, 3, 27, 48)
    for B in (1, 8):
        xb = x[:B].contiguous()
        model(xb)
        with torch.inference_mode():
            otn.forward(sdg, xb)
        for _ in range(args.reps):
            te = timed(lambda: model(xb), 20) / B
            with torch.inference_mode():
                tr = timed(lambda: otn.forward(sdg, xb), 5) / B
            print(f"network ms per window, B = {B}: engine {te:.3f} ({fpf * 100 / te / 1e9:.1f} TFLOP/s)  pytorch {tr:.3f}")
            res.setdefault(f"ms_per_window_B{B}", []).append([te, tr])
    if args.out:
        os.makedirs(args.out, exist_ok=True)
        with open(os.path.join(args.out, "result.json"), "w") as fh:
            json.dump(res, fh, indent=1)


if __name__ == "__main__":
    main()
