"""Depth export and import per frame at 1920 x 1080 and 3840 x 2160: ms per frame, and bytes moved between host and device.

Export (nunif_b200/iw3/depth_io.export_depth_u16, csrc/depth_io.cu), from a normalised depth at the depth model's
resolution (518 x 920, the size of a Depth-Anything output for a 16:9 frame) to the uint16 map on the host:
  nofit        mapper none, no fit: the engine kernel vs the same ops in eager torch on the GPU (clamp, * 0xffff, cast);
  fit          --export-depth-fit to the frame size (align_corners=True, the image path), mapper none;
  fit+MAPPER   --export-disparity with div_6 and with the softplus blend mul_1+mul_2=0.5:
                 fused      the mapper evaluated on every tap of the resize (what the engine runs),
                 separate   a source pass (nb200_mapper_apply) into a buffer, then the fit without a mapper,
                 torch      the mapper's torch ops (oracle/mapper.py), F.interpolate(antialias=True), clamp, * 0xffff, cast;
  down+MAPPER  the same three with a depth at twice the frame size, where the fit downsamples and each source pixel is
               read by several outputs.
Before timing, every engine export is checked to be within one code of the same ops in torch on the CPU (ATen's CPU
antialiased resize, which the engine follows; the torch GPU kernel computes the weights differently), and each row
reports its largest code difference from that.  Every export row includes the device -> host copy of the uint16 map (2 B/px of the frame with fit); "fp32_to_host"
gives the 4 B/px a caller moves when it copies the float map instead.

Import (depth_io.import_depth and the iw3_export.yml image path), from the decoded 16-bit PNG map in host memory:
  decode       upload (2 B/px) + nb200_depth_import vs upload + load_depth's ops in eager torch on the GPU;
  full         upload + decode + the inverted edge dilation (-dilate_edge(-d, 2)) + forward_fill warp + SBS compose on
               the engine; the warp and dilation have no eager-torch counterpart in this tree, so this row is the engine's
               alone.

CUDA events around each call, ROUNDS round-robin repetitions after a warm-up; median, min and max are printed with the
card and its power limit.
    python profiles/bench_depth_export.py [--iters 20] [--rounds 5] [--out DIR]
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys
from argparse import Namespace

import torch
import torch.nn.functional as F

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nunif_b200 import _lib  # noqa: E402
from nunif_b200.iw3.depth_io import export_depth_u16, import_depth  # noqa: E402
from nunif_b200.iw3.dilation import dilate_edge  # noqa: E402
from nunif_b200.iw3.mapper import descriptor  # noqa: E402
from nunif_b200.iw3.postprocess import postprocess_image  # noqa: E402
from nunif_b200.iw3.utils import apply_divergence  # noqa: E402
from oracle.mapper import mapper as torch_mapper  # noqa: E402

FRAMES = {"1080p": (1080, 1920), "4k": (2160, 3840)}
DEPTH = (518, 920)
MAPPERS = ("div_6", "mul_1+mul_2=0.5")


def timed(fn, iters):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(iters):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / iters


def separate(d, mapper, size):
    """The alternative to the fused mapper: one source pass, then the fit."""
    m = torch.empty_like(d)
    _lib.check(_lib.lib().nb200_mapper_apply(_lib.ptr(d), d.numel(), ctypes.byref(descriptor(mapper)), _lib.ptr(m),
                                             _lib.stream_ptr(d.device)))
    return export_depth_u16(m, size=size)


def torch_export(d, mapper, size, align_corners=True):
    if mapper is not None:
        d = torch_mapper(d, mapper)
    if size is not None:
        d = F.interpolate(d.unsqueeze(0), size=size, mode="bilinear", antialias=True, align_corners=align_corners).squeeze(0)
    return (0xffff * torch.clamp(d, 0, 1)).to(torch.uint16)


def torch_decode(u16):
    return torch.clamp(u16.to(torch.float32) / 0xffff, 0, 1).unsqueeze(0)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=20)
    ap.add_argument("--rounds", type=int, default=5)
    ap.add_argument("--out", default=None, help="directory for result.json")
    a = ap.parse_args()
    if not torch.cuda.is_available():
        raise SystemExit("bench_depth_export needs a CUDA device")
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    print("card:", q)
    dev = torch.device("cuda:0")
    g = torch.Generator().manual_seed(1)
    rows = []
    args = Namespace(method="forward_fill", mapper="none", divergence=2.0, convergence=0.5, synthetic_view="both",
                     disable_amp=False, state={"convergence_model": None}, ipd_offset=0, pad=None, pad_mode=None, vr180=False,
                     half_sbs=False, tb=False, half_tb=False, cross_eyed=False, anaglyph=None, rgbd=False, half_rgbd=False,
                     max_output_height=None, max_output_width=None, keep_aspect_ratio=False)
    for fname, (H, W) in FRAMES.items():
        size = (H, W)
        d = torch.rand((1,) + DEPTH, generator=g).to(dev)
        d_big = torch.rand((1, 2 * H, 2 * W), generator=g).to(dev)
        # step -> (source depth, mapper, fit size)
        spec = {"nofit": (d, None, None), "fit": (d, None, size)}
        for m in MAPPERS:
            spec[f"fit+{m}"] = (d, m, size)
            spec[f"down+{m}"] = (d_big, m, size)
        calls = {}
        for step, (src, m, sz) in spec.items():
            if m is None:
                calls[(step, "engine")] = lambda src=src, sz=sz: export_depth_u16(src, size=sz).cpu()
            else:
                calls[(step, "fused")] = lambda src=src, m=m, sz=sz: export_depth_u16(src, mapper=m, size=sz).cpu()
                calls[(step, "separate")] = lambda src=src, m=m, sz=sz: separate(src, m, sz).cpu()
            calls[(step, "torch")] = lambda src=src, m=m, sz=sz: torch_export(src, m, sz).cpu()
        u16_host = (torch.rand((H, W), generator=g) * 65535).to(torch.int32).to(torch.uint16).pin_memory()
        x = torch.rand((3, H, W), generator=g).to(dev)

        def full():
            depth = import_depth(u16_host.numpy(), dev)
            depth = -dilate_edge(-depth.unsqueeze(0), 2).squeeze(0)
            left, right = apply_divergence(depth, x, args, None)
            return postprocess_image(left, right, args)
        calls[("decode", "engine")] = lambda: import_depth(u16_host.numpy(), dev)
        calls[("decode", "torch")] = lambda: torch_decode(u16_host.to(dev))
        calls[("full", "engine")] = full

        # before anything is timed: every export agrees within one code with the same ops in torch on the CPU (ATen's CPU
        # antialiased resize, the kernel the engine follows); the torch rows report how far the GPU ops are from it
        code_diff = {}
        for step, (src, m, sz) in spec.items():
            want = torch_export(src.cpu(), m, sz).to(torch.int64)
            for impl in ("engine", "fused", "separate", "torch"):
                if (step, impl) in calls:
                    code_diff[(step, impl)] = (calls[(step, impl)]().to(torch.int64) - want).abs().max().item()
            for impl in ("engine", "fused", "separate"):
                if (step, impl) in calls:
                    assert code_diff[(step, impl)] <= 1, (fname, step, impl, code_diff[(step, impl)])
        decode_diff = (calls[("decode", "engine")]().cpu() - torch_decode(u16_host)).abs().max().item()
        assert decode_diff == 0.0, decode_diff
        for f in calls.values():
            f(); f()
        torch.cuda.synchronize()
        samples = {k: [] for k in calls}
        for _ in range(a.rounds):
            for k, f in calls.items():
                samples[k].append(timed(f, a.iters))
        for (step, impl), ms in samples.items():
            if step == "decode" or step == "full":
                to_host, to_device = 0, 2 * H * W
            else:
                to_host, to_device = 2 * (H * W if step != "nofit" else DEPTH[0] * DEPTH[1]), 0
            row = dict(frame=fname, step=step, impl=impl, ms_per_frame=round(statistics.median(ms), 4), ms_min=round(min(ms), 4),
                       ms_max=round(max(ms), 4), bytes_to_host=to_host, bytes_to_device=to_device)
            if to_host:
                row["fp32_to_host"] = 2 * to_host
                row["max_code_diff_vs_torch_cpu"] = code_diff[(step, impl)]
            rows.append(row)
            print(json.dumps(row))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "result.json"), "w") as fh:
            json.dump(dict(card=q, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
