"""Film-grain output stage at 3840 x 2160, B = 4 frames per call, 8- and 16-bit output: ms per frame of
  fused       the temporal grain + quantise kernel FrameBatchPipeline(grain=...) runs (csrc/rgb_noise.cu: noise generated in
              the kernel, buffer blended in a register across the batch, uint8 / uint16 HWC written in the same pass);
  plain       the conversion the pipeline runs without grain (nb200_chw_f32_to_hwc, no grain at all);
  torch_ops   the reference's sequence on the same GPU, frame by frame (waifu2x/ui_utils.py:167-175 with rgb_noise.py and
              from_tensor's quantisation, without its device -> host copy): randn_like, randn, nearest interpolate, the
              buffer blend, apply_rgb_noise, * scale, round, cast.
GB/s counts the bytes the fused stage must move per frame - the 12 B/px float frame in, 3 or 6 B/px out, and the 12 B/px
buffer read and written once per call (24 / B B/px) - set against the H100 SXM data-sheet 3.35 TB/s; the other two rows are
charged the same bytes, so theirs is only a speed ratio.  CUDA events, the three calls round-robin ROUNDS times after a
warm-up; median and spread are printed, with the card and its power limit.
    python profiles/bench_grain.py [--iters 10] [--rounds 5] [--out DIR]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nunif_b200.iw3.frames import chw_float_to_hwc  # noqa: E402
from nunif_b200.nunif.rgb_noise import TemporalGrain  # noqa: E402
from oracle import rgb_noise as orn  # noqa: E402

H, W, B = 2160, 3840, 4
PEAK_BPS = 3.35e12
STRENGTH, SPEED = 0.2, 0.8


def timed(fn, iters):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(iters):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / iters


def reference_noise_like(base):
    """rgb_noise.py:5-17 for a CHW frame."""
    noise = torch.randn_like(base)
    noise2 = torch.randn(base.shape[:-2] + (base.shape[-2] // 2, base.shape[-1] // 2), dtype=base.dtype, device=base.device)
    noise2 = F.interpolate(noise2.unsqueeze(0), size=(base.shape[-2], base.shape[-1]), mode="nearest").squeeze(0)
    return noise.mul_(0.5).add_(noise2, alpha=0.5)


def reference_frames(x, state, bits):
    dtype, scale = (torch.uint16, 65535.0) if bits == 16 else (torch.uint8, 255.0)
    outs = []
    for f in x:
        noise = reference_noise_like(f)
        if noise.shape != state["buf"].shape:
            state["buf"].resize_(noise.shape)
            state["buf"].copy_(noise)
        else:
            state["buf"].mul_(1.0 - SPEED)
            state["buf"].add_(noise.mul_(SPEED))
        y = orn.apply_rgb_noise(f, state["buf"], strength=STRENGTH)
        outs.append((y.permute(1, 2, 0).contiguous() * scale).round_().to(dtype))
    return outs


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for result.json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_grain needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    print("card:", q)
    dev = "cuda:0"
    x = torch.rand(B, 3, H, W, generator=torch.Generator().manual_seed(1)).to(dev)
    rows = []
    for bits in (8, 16):
        dtype = torch.uint16 if bits == 16 else torch.uint8
        grain = TemporalGrain(STRENGTH, SPEED, seed=1)
        state = {"buf": torch.zeros((0,), device=dev)}
        calls = {
            "fused": lambda: grain(x, dtype=dtype),
            "plain": lambda: chw_float_to_hwc(x, use_16bit=bits == 16),
            "torch_ops": lambda: reference_frames(x, state, bits),
        }
        for f in calls.values():
            f(); f()
        torch.cuda.synchronize()
        samples = {k: [] for k in calls}
        for _ in range(a.rounds):
            for k, f in calls.items():
                samples[k].append(timed(f, a.iters) / B)
        bytes_per_frame = H * W * (12 + 3 * bits // 8 + 24 / B)
        for k, ms in samples.items():
            med = statistics.median(ms)
            gbps = bytes_per_frame / (med * 1e-3) / 1e9
            row = dict(bits=bits, B=B, step=k, ms_per_frame=round(med, 4), ms_min=round(min(ms), 4), ms_max=round(max(ms), 4),
                       gbps=round(gbps, 1), pct_of_3350=round(100 * gbps * 1e9 / PEAK_BPS, 1))
            rows.append(row)
            print(json.dumps(row))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "result.json"), "w") as fh:
            json.dump(dict(card=q, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
