#!/usr/bin/env python
"""Kernel-level A/B of the fused Swin-block head (`nb200_swin_attn_fused_f16`, swin_attn_fused_kernel<C>) between two builds
of libnunif_b200.so, loaded side by side into one process with ctypes.

The comparison build is made from a git revision into the git-ignored profiles/_bin/ (the copy needs no git to run):

    mkdir -p profiles/_bin/parent && git archive HEAD~1 | tar -x -C profiles/_bin/parent
    python profiles/_bin/parent/nunif_b200/build.py
    python profiles/ab_swin_attn.py --base profiles/_bin/parent/nunif_b200/libnunif_b200.so

At the four production shapes of the swin_unet 4x model (batch 16: 240^2 x 96, 120^2 x 192, 60^2 x 192, 240^2 x 192), each
with shift 0 and 3, both builds run on the same seeded inputs.  Per shape: warm-up, then REPS repetitions with the order of the
two builds alternating, each a CUDA-event window of N back-to-back calls (N chosen so that a window is ~WINDOW_MS).  A call
includes what the C ABI does around the kernel (a stream-ordered allocation and the small relative-position-bias packing
kernel, the same in both builds).  Reported: the
median ms per call and the max-min spread of each build, the ratio of medians, and whether the two outputs are bit-identical.
Also printed: the device, its power limit and SM clocks sampled during the timed region, and per kernel the registers, the
dynamic shared memory of its launches (from a torch.profiler trace) and the CTAs per SM that
cuOccupancyMaxActiveBlocksPerMultiprocessor (the driver form of cudaOccupancyMaxActiveBlocksPerMultiprocessor) reports for
the kernel's cubin at that launch configuration (block size and shared memory as the trace recorded them, so each build is
queried at its own).
"""
import argparse
import ctypes
import json
import os
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
KERNEL = "_ZN5nb20022swin_attn_fused_kernelILi{C}EEEv14CUtensorMap_stPK6__halfPKfPK6float4PS2_iiii"


def load(path):
    from nunif_b200 import _lib
    lib = ctypes.CDLL(os.path.abspath(path))   # RTLD_LOCAL: each build keeps its own symbols and its own static cudart
    for name in ("nb200_last_error", "nb200_check_device", "nb200_swin_attn_fused_f16"):
        res, args = _lib.SIGNATURES[name]
        getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
    return lib


def check(lib, rc):
    if rc != 0:
        raise RuntimeError(lib.nb200_last_error().decode("utf-8", "replace"))


def call(lib, t, shift):
    import torch
    x, wqkv, bqkv, table, att = t
    B, H, W, C = x.shape
    p = lambda v: ctypes.c_void_p(v.data_ptr())   # noqa: E731
    check(lib, lib.nb200_swin_attn_fused_f16(p(x), p(wqkv), p(bqkv), p(table), p(att), B, H, W, C, shift,
                                             ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)))


def inputs(H, C, shift, dev):
    import torch
    g = torch.Generator(device="cpu").manual_seed(H * 1000 + C + shift)
    x = torch.randn(BATCH, H, H, C, generator=g).half().to(dev)
    wqkv = (torch.randn(3 * C, C, generator=g) / C ** 0.5).half().to(dev)
    bqkv = (0.1 * torch.randn(3 * C, generator=g)).to(dev)
    table = (0.5 * torch.randn(121, 6, generator=g)).to(dev)
    return x, wqkv, bqkv, table


def window_ms(lib, t, shift, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        call(lib, t, shift)
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def launch_smem(libs, dev):
    """shared memory, registers and block size of each build's swin_attn_fused_kernel<C> launches (torch.profiler trace)."""
    import torch
    from torch.profiler import ProfilerActivity, profile
    out = {}
    with tempfile.TemporaryDirectory() as d:
        for tag, lib in libs.items():
            for C in (96, 192):
                x, wqkv, bqkv, table = inputs(12, C, 0, dev)
                t = (x, wqkv, bqkv, table, torch.empty_like(x))
                with profile(activities=[ProfilerActivity.CUDA]) as prof:
                    call(lib, t, 0)
                    torch.cuda.synchronize()
                path = os.path.join(d, f"{tag}{C}.json")
                prof.export_chrome_trace(path)
                ev = [e for e in json.load(open(path))["traceEvents"]
                      if e.get("cat") == "kernel" and "swin_attn_fused_kernel" in e.get("name", "")]
                a = ev[0]["args"]
                out[(tag, C)] = {"smem": int(a["shared memory"]), "regs_trace": int(a["registers per thread"]),
                                 "threads": a["block"][0] * a["block"][1] * a["block"][2]}
    return out


def occupancy(so_path, C, smem, threads):
    """CTAs per SM of swin_attn_fused_kernel<C> from the build's own cubin, loaded with the driver API into the current context."""
    name = KERNEL.format(C=C)
    cuobjdump = os.path.join(os.environ.get("CUDA_HOME", "/usr/local/cuda"), "bin", "cuobjdump")
    with tempfile.TemporaryDirectory() as d:
        subprocess.run([cuobjdump, "-xelf", "all", os.path.abspath(so_path)], cwd=d, check=True, capture_output=True)
        image = next(b for b in (open(os.path.join(d, f), "rb").read() for f in sorted(os.listdir(d))) if name.encode() in b)
    cu = ctypes.CDLL("libcuda.so.1")

    def ck(rc):
        if rc != 0:
            raise RuntimeError(f"CUDA driver error {rc}")
    mod, fn = ctypes.c_void_p(), ctypes.c_void_p()
    ck(cu.cuModuleLoadData(ctypes.byref(mod), ctypes.c_char_p(image)))
    try:
        ck(cu.cuModuleGetFunction(ctypes.byref(fn), mod, name.encode()))
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
    import torch
    from bench import ClockSampler
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
        for (tag, C), s in sorted(launch_smem(libs, dev).items()):
            regs, ctas = occupancy(paths[tag], C, s["smem"], s["threads"])
            kern.append({"build": tag, "C": C, "regs": regs, "dyn_smem": s["smem"], "threads": s["threads"], "ctas_per_sm": ctas})
            print(f"# {tag:4s} swin_attn_fused_kernel<{C}>: {s['threads']} threads, {regs} registers, {s['smem']} B shared memory/CTA, "
                  f"{ctas} CTA(s)/SM")
    except Exception as e:  # noqa: BLE001  (the timing below does not depend on it)
        kern.append({"error": f"{type(e).__name__}: {e}"})
        print(f"# occupancy query failed: {type(e).__name__}: {e}")

    rows = []
    with torch.inference_mode(), ClockSampler(0) as clocks:
        for H, C in SHAPES:
            for shift in (0, 3):
                x, wqkv, bqkv, table = inputs(H, C, shift, dev)
                t = {k: (x, wqkv, bqkv, table, torch.full_like(x, 7.0)) for k in libs}
                for k, lib in libs.items():
                    for _ in range(3):
                        call(lib, t[k], shift)
                torch.cuda.synchronize()
                equal = torch.equal(t["base"][4], t["new"][4])
                diff = float((t["base"][4].float() - t["new"][4].float()).abs().max())
                est = max(window_ms(libs["base"], t["base"], shift, 2), window_ms(libs["new"], t["new"], shift, 2))
                n = max(3, int(WINDOW_MS / max(est, 1e-3)))
                ms = {k: [] for k in libs}
                for r in range(REPS):
                    for k in (("base", "new") if r % 2 == 0 else ("new", "base")):
                        ms[k].append(window_ms(libs[k], t[k], shift, n))
                row = {"B": BATCH, "H": H, "W": H, "C": C, "shift": shift, "calls_per_window": n, "equal": equal, "max_abs_diff": diff}
                for k in libs:
                    row[k] = {"median_ms": statistics.median(ms[k]), "min_ms": min(ms[k]), "max_ms": max(ms[k])}
                row["new_over_base"] = row["new"]["median_ms"] / row["base"]["median_ms"]
                rows.append(row)
                b, nw = row["base"], row["new"]
                print(f"{BATCH}x{H}x{H}x{C} shift {shift}: base {b['median_ms']:.4f} ms [{b['min_ms']:.4f}, {b['max_ms']:.4f}]  "
                      f"new {nw['median_ms']:.4f} ms [{nw['min_ms']:.4f}, {nw['max_ms']:.4f}]  new/base {row['new_over_base']:.3f}  "
                      f"outputs {'identical' if equal else f'DIFFER (max |d| {diff:g})'}", flush=True)
                del t, x
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
