#!/usr/bin/env python
"""Kernel-level A/B of the fused Swin-block tail (`nb200_swin_mlp_fused_f16` with att, swin_mlp_fused_kernel<C>) between two
builds of libnunif_b200.so, loaded side by side into one process with ctypes.

The comparison build is made from a git revision into the git-ignored profiles/_bin/ (the copy needs no git to run):

    mkdir -p profiles/_bin/parent && git archive HEAD~1 | tar -x -C profiles/_bin/parent
    python profiles/_bin/parent/nunif_b200/build.py
    python profiles/ab_swin_mlp.py --base profiles/_bin/parent/nunif_b200/libnunif_b200.so

At the four production shapes of the swin_unet 4x model (batch 16: 240^2 x 96, 120^2 x 192, 60^2 x 192, 240^2 x 192) both
builds run on the same seeded inputs.  The call updates x in place (x <- x1 + mlp(x1)), so the output check runs each build once
on its own copy of the same x; the timed windows then keep updating that copy (the weights are small, so x stays finite).  Per
shape: warm-up, then REPS repetitions with the order of the two builds alternating, each a CUDA-event window of N back-to-back
calls (N chosen so that a window is ~WINDOW_MS).  Reported: the median ms per call and the max-min spread of each build, the
ratio of medians, and whether the two outputs are bit-identical.  Also printed: the device, its power limit and SM clocks
sampled during the timed region, and per kernel the registers, the dynamic shared memory of its launches (from a torch.profiler
trace) and the CTAs per SM that cuOccupancyMaxActiveBlocksPerMultiprocessor reports for the kernel's cubin at that launch
configuration.
"""
import argparse
import ctypes
import json
import os
import re
import statistics
import subprocess
import sys
import tempfile

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

SHAPES = [(240, 96), (120, 192), (60, 192), (240, 192)]   # (H = W, C) of the swin blocks of swin_unet 4x on 256^2 tiles
BATCH = 16
REPS = 7
WINDOW_MS = 60.0
KERNEL_RE = rb"_ZN5nb20021swin_mlp_fused_kernelILi%dE[A-Za-z0-9_]*"


def load(path):
    from nunif_b200 import _lib
    lib = ctypes.CDLL(os.path.abspath(path))   # RTLD_LOCAL: each build keeps its own symbols and its own static cudart
    for name in ("nb200_last_error", "nb200_check_device", "nb200_swin_mlp_fused_f16"):
        res, args = _lib.SIGNATURES[name]
        getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
    return lib


def check(lib, rc):
    if rc != 0:
        raise RuntimeError(lib.nb200_last_error().decode("utf-8", "replace"))


def call(lib, x, w):
    import torch
    att, wp, bp, w1, b1, w2, b2 = w
    B, H, W, C = x.shape
    p = lambda v: ctypes.c_void_p(v.data_ptr())   # noqa: E731
    check(lib, lib.nb200_swin_mlp_fused_f16(p(x), p(att), B * H * W, C, p(wp), p(bp), p(w1), p(b1), p(w2), p(b2),
                                            ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))


def inputs(H, C, dev):
    import torch
    g = torch.Generator(device="cpu").manual_seed(H * 1000 + C)
    x = torch.randn(BATCH, H, H, C, generator=g).half().to(dev)
    att = torch.randn(BATCH, H, H, C, generator=g).half().to(dev)
    wp = (0.5 * torch.randn(C, C, generator=g) / C ** 0.5).half().to(dev)
    bp = (0.1 * torch.randn(C, generator=g)).to(dev)
    w1 = (torch.randn(2 * C, C, generator=g) / C ** 0.5).half().to(dev)
    b1 = (0.1 * torch.randn(2 * C, generator=g)).to(dev)
    w2 = (0.05 * torch.randn(C, 2 * C, generator=g) / (2 * C) ** 0.5).half().to(dev)
    b2 = (0.01 * torch.randn(C, generator=g)).to(dev)
    return x, (att, wp, bp, w1, b1, w2, b2)


def window_ms(lib, x, w, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        call(lib, x, w)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def launch_smem(libs, dev):
    """shared memory and block size of each build's swin_mlp_fused_kernel<C> launches (torch.profiler trace)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    out = {}
    with tempfile.TemporaryDirectory() as d:
        for tag, lib in libs.items():
            for C in (96, 192):
                x, w = inputs(12, C, dev)
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    call(lib, x, w)
                    torch.cuda.synchronize()
                path = os.path.join(d, f"{tag}{C}.json")
                prof.export_chrome_trace(path)
                ev = [e for e in json.load(open(path))["traceEvents"]
                      if e.get("cat") == "kernel" and "swin_mlp_fused_kernel" in e.get("name", "")]
                a = ev[0]["args"]
                out[(tag, C)] = (int(a["shared memory"]), int(a["block"][0]))
    return out


def occupancy(so_path, C, smem, threads):
    """registers and CTAs per SM of the build's swin_mlp_fused_kernel<C> that takes att, from its own cubin (driver API)."""
    cuobjdump = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    with tempfile.TemporaryDirectory() as d:
        subprocess.run([cuobjdump, "-xelf", "all", os.path.abspath(so_path)], cwd=d, check=True, capture_output=True)
        for f in sorted(os.listdir(d)):
            image = open(os.path.join(d, f), "rb").read()
            names = sorted(n for n in set(re.findall(KERNEL_RE % C, image)) if b"_param_" not in n)
            if names:
                break
        else:
            raise RuntimeError(f"swin_mlp_fused_kernel<{C}> not found in {so_path}")
    # this tree instantiates <C, PROJ>: take the PROJ = true one; older builds have a single kernel per C
    name = next((n for n in names if b"Lb1E" in n), names[0])
    cu = ctypes.CDLL("libcuda.so.1")

    def ck(rc):
        if rc != 0:
            raise RuntimeError(f"CUDA driver error {rc}")
    mod, fn = ctypes.c_void_p(), ctypes.c_void_p()
    ck(cu.cuModuleLoadData(ctypes.byref(mod), ctypes.c_char_p(image)))
    try:
        ck(cu.cuModuleGetFunction(ctypes.byref(fn), mod, name))
        ck(cu.cuFuncSetAttribute(fn, 8, ctypes.c_int(smem)))   # CU_FUNC_ATTRIBUTE_MAX_DYNAMIC_SHARED_SIZE_BYTES
        regs, n = ctypes.c_int(), ctypes.c_int()
        ck(cu.cuFuncGetAttribute(ctypes.byref(regs), 4, fn))   # CU_FUNC_ATTRIBUTE_NUM_REGS
        ck(cu.cuOccupancyMaxActiveBlocksPerMultiprocessor(ctypes.byref(n), fn, threads, ctypes.c_size_t(smem)))
    finally:
        cu.cuModuleUnload(mod)
    return regs.value, n.value


def device_info(index):
    q = subprocess.run(["nvidia-smi", "-i", str(index), "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                       capture_output=True, text=True)
    return q.stdout.strip()


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--base", required=True, help="the build to compare against (libnunif_b200.so)")
    ap.add_argument("--new", default=os.path.join(ROOT, "nunif_b200", "libnunif_b200.so"), help="default: this tree's build")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()
    for p in (args.base, args.new):
        if not os.path.isfile(p):
            ap.error(f"no such library: {p}")
    import torch
    from bench import ClockSampler
    if not torch.cuda.is_available():
        raise SystemExit("ab_swin_mlp.py needs a CUDA device")
    dev = torch.device("cuda:0")
    torch.cuda.init()
    torch.zeros(1, device=dev)
    paths = {"base": args.base, "new": args.new}
    libs = {k: load(v) for k, v in paths.items()}
    for lib in libs.values():
        check(lib, lib.nb200_check_device(0))
    info = {"device": torch.cuda.get_device_name(dev), "nvidia_smi": device_info(0), "paths": paths}
    print(f"# {info['device']} | name, power limit, max SM clock: {info['nvidia_smi']}")

    kern = []
    try:
        for (tag, C), (smem, threads) in sorted(launch_smem(libs, dev).items()):
            regs, ctas = occupancy(paths[tag], C, smem, threads)
            kern.append({"build": tag, "C": C, "threads": threads, "regs": regs, "dyn_smem": smem, "ctas_per_sm": ctas})
            print(f"# {tag:4s} swin_mlp_fused_kernel<{C}>: {threads} threads, {regs} registers at launch, {smem} B shared memory/CTA, "
                  f"{ctas} CTA(s)/SM")
    except Exception as e:  # noqa: BLE001  (the timing below does not depend on it)
        kern.append({"error": f"{type(e).__name__}: {e}"})
        print(f"# occupancy query failed: {type(e).__name__}: {e}")

    rows = []
    with torch.inference_mode(), ClockSampler(0) as clocks:
        for H, C in SHAPES:
            x0, w = inputs(H, C, dev)
            xs = {k: x0.clone() for k in libs}
            for k, lib in libs.items():
                call(lib, xs[k], w)
            torch.cuda.synchronize()
            equal = torch.equal(xs["base"], xs["new"])
            diff = float((xs["base"].float() - xs["new"].float()).abs().max())
            for k, lib in libs.items():
                for _ in range(2):
                    call(lib, xs[k], w)
            est = max(window_ms(libs["base"], xs["base"], w, 2), window_ms(libs["new"], xs["new"], w, 2))
            n = max(3, int(WINDOW_MS / max(est, 1e-3)))
            ms = {k: [] for k in libs}
            for r in range(REPS):
                for k in (("base", "new") if r % 2 == 0 else ("new", "base")):
                    ms[k].append(window_ms(libs[k], xs[k], w, n))
            row = {"B": BATCH, "H": H, "W": H, "C": C, "calls_per_window": n, "equal": equal, "max_abs_diff": diff}
            for k in libs:
                row[k] = {"median_ms": statistics.median(ms[k]), "min_ms": min(ms[k]), "max_ms": max(ms[k])}
            row["new_over_base"] = row["new"]["median_ms"] / row["base"]["median_ms"]
            rows.append(row)
            b, nw = row["base"], row["new"]
            print(f"{BATCH}x{H}x{H}x{C}: base {b['median_ms']:.4f} ms [{b['min_ms']:.4f}, {b['max_ms']:.4f}]  "
                  f"new {nw['median_ms']:.4f} ms [{nw['min_ms']:.4f}, {nw['max_ms']:.4f}]  new/base {row['new_over_base']:.3f}  "
                  f"outputs {'identical' if equal else f'DIFFER (max |d| {diff:g})'}", flush=True)
            del xs, x0, w
    result = {"info": info, "clocks": clocks.summary(), "kernels": kern, "shapes": rows,
              "all_equal": all(r["equal"] for r in rows)}
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)
    return 0 if result["all_equal"] else 1


if __name__ == "__main__":
    sys.exit(main())
