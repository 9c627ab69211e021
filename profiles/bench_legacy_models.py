#!/usr/bin/env python
"""4K-frame throughput of waifu2x.upconv_7 (2x) and waifu2x.vgg_7 (1x): the engine's tiled_render against PyTorch + cuDNN
running the oracle under fp16 autocast (the reference's CUDA numerics) through the reference's tiling loop
(oracle.seam_blending.tiled_render), in the same process, alternating frame by frame.

    python profiles/bench_legacy_models.py --out DIR

Per model: a seeded 3x2160x3840 frame, tile 256, batch 16 (9 x 16 = 144 tiles), WARMUP untimed frames of each leg, then FRAMES
timed frames of each (host clock around work that ends in a device synchronise).  Reported: ms per frame (median, min, max),
input MP/s, TFLOP/s from the per-tile FLOP count of the network (tile_flops below), the fraction of output samples whose 8-bit
value differs between the two legs, and - in a separate pass with the engine's event profiler on - ms per kernel class
with the HBM bytes each class must move.  Also the card's name, power limit and max SM clock.  Writes result.json.
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

H, W, TILE, BATCH = 2160, 3840, 256, 16
UPCONV_7 = [3, 16, 32, 64, 128, 128, 256]
VGG_7 = [3, 32, 32, 64, 64, 128, 128]


def tile_flops(widths, up, T=TILE):
    """Multiply-adds x 2 of one T x T tile: six 3x3 valid convs, then the 3-channel head (ConvTranspose 4x4 s2 p3: each output
    pixel sees 2 x 2 taps, i.e. 16 taps per input pixel; or a 3x3 conv)."""
    f, s = 0, T
    for i in range(6):
        s -= 2
        f += 2 * widths[i] * widths[i + 1] * 9 * s * s
    if up:
        f += 2 * widths[6] * 3 * 16 * s * s
    else:
        f += 2 * widths[6] * 3 * 9 * (s - 2) * (s - 2)
    return f


def card():
    import torch
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,driver_version", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return {"torch_device": torch.cuda.get_device_name(0), "nvidia_smi": q.stdout.strip() or q.stderr.strip()}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--out", required=True, help="directory for result.json")
    ap.add_argument("--frames", type=int, default=6)
    ap.add_argument("--warmup", type=int, default=2)
    args = ap.parse_args()
    import torch
    import ctypes
    from nunif_b200 import synth, _lib
    from nunif_b200.nunif.models import create_model
    from nunif_b200.nunif.render import tiled_render
    from oracle import legacy as ol, seam_blending as osb
    assert torch.cuda.is_available(), "this benchmark needs a GPU"
    os.makedirs(args.out, exist_ok=True)
    dev = "cuda:0"
    torch.backends.cudnn.benchmark = True
    lib = _lib.lib()
    img = synth.synth_image(1000, 3, H, W, smooth=False).to(dev)
    result = {"card": card(), "frame": [3, H, W], "tile_size": TILE, "batch_size": BATCH, "models": {}}
    for name, sdf, fn, spec, widths, up in [
            ("waifu2x.upconv_7", synth.upconv7_state_dict, ol.upconv7_forward, ol.UPCONV_7, UPCONV_7, True),
            ("waifu2x.vgg_7", synth.vgg7_state_dict, ol.vgg7_forward, ol.VGG_7, VGG_7, False)]:
        sd = sdf(0)
        m = create_model(name, sd, dev)
        sdc = {k: v.to(dev) for k, v in sd.items()}
        cfg = osb.create_config(H, W, spec["scale"], spec["offset"], TILE, 0)
        ntiles = cfg["h_blocks"] * cfg["w_blocks"]
        flop = tile_flops(widths, up) * ntiles

        def engine():
            with torch.no_grad():
                return tiled_render(img, m, tile_size=TILE, batch_size=BATCH)

        def amp_model(b):
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
                return fn(sdc, b)

        def torch_ref():
            with torch.no_grad():
                return osb.tiled_render(img, amp_model, spec["scale"], spec["offset"], 0, TILE, BATCH)

        legs = {"engine": engine, "torch_cudnn_amp": torch_ref}
        times = {k: [] for k in legs}
        outs = {}
        for i in range(args.warmup + args.frames):
            for k, f in legs.items():
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                outs[k] = f()
                torch.cuda.synchronize()
                if i >= args.warmup:
                    times[k].append((time.perf_counter() - t0) * 1e3)
        a, b = outs["engine"], outs["torch_cudnn_amp"]
        qa, qb = (a * 255).round().clamp(0, 255), (b * 255).round().clamp(0, 255)
        r = {"tiles": ntiles, "tflop_per_frame": flop / 1e12, "gflop_per_tile": tile_flops(widths, up) / 1e9,
             "q8_mismatch_engine_vs_amp": float((qa != qb).double().mean()), "max_abs_engine_vs_amp": float((a - b).abs().max())}
        for k, ts in times.items():
            med = statistics.median(ts)
            r[k] = {"ms_per_frame": med, "ms_min": min(ts), "ms_max": max(ts), "input_mp_per_s": H * W / 1e6 / (med / 1e3),
                    "tflop_per_s": flop / 1e12 / (med / 1e3), "frames": len(ts)}
        r["engine_speedup_vs_torch"] = r["torch_cudnn_amp"]["ms_per_frame"] / r["engine"]["ms_per_frame"]
        # profiled pass (events around every launch; a run of its own)
        _lib.check(lib.nb200_profile_enable(1))
        engine()
        buf = ctypes.create_string_buffer(8192)
        _lib.check(lib.nb200_profile_report(buf, 8192))
        _lib.check(lib.nb200_profile_enable(0))
        prof = json.loads(buf.value.decode())
        for c in prof.values():
            c["gb_per_s"] = c["hbm_bytes"] / (c["ms"] / 1e3) / 1e9 if c["ms"] > 0 else None
        r["profile"] = prof
        result["models"][name] = r
        print(name, json.dumps({k: r[k] for k in ("engine", "torch_cudnn_amp", "engine_speedup_vs_torch", "q8_mismatch_engine_vs_amp")}),
              flush=True)
        print(name, "profile", json.dumps(prof), flush=True)
        del m, outs, a, b
        torch.cuda.empty_cache()
    with open(os.path.join(args.out, "result.json"), "w") as fh:
        json.dump(result, fh, indent=1)
    print(json.dumps(result["card"]))


if __name__ == "__main__":
    main()
