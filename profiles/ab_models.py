#!/usr/bin/env python
"""Model-level A/B of every model kind between two builds of libnunif_b200.so, loaded side by side into one process with
ctypes.  For changes that must not move any output bit: host-side restructuring of the forwards, workspace layout, packing.

The comparison build is made from a git revision into the git-ignored profiles/_bin/ (the copy needs no git to run):

    mkdir -p profiles/_bin/parent && git archive HEAD~1 | tar -x -C profiles/_bin/parent
    python profiles/_bin/parent/nunif_b200/build.py
    python profiles/ab_models.py --base profiles/_bin/parent/nunif_b200/libnunif_b200.so

Both builds get the same seeded weights (nunif_b200.synth) and inputs through each model's C ABI entry, at production sizes:
swin_unet 1x / 2x / 4x (and 4x's to_2x) and UpCUNet / CUNet / UpConv7 / VGG7 on 256^2 tiles in batches of 16, Depth-Anything-V2
S / B / L at the iw3_1080p network input (4 x 392x686), ZoeD_N at 384x512 and 384x704 (batch 2), and row_flow_v3, mlbw
(2 and 4 layers, and 2 layers `small`: two blocks shifted along x only), depth_aa (all three modes) and light_inpaint_v1 (with
and without the mirror) on 1080p frames.  Every output must be bit-identical, and so must ZoeD_N's debug taps 0..14 and
light_inpaint_v1's taps 100..173; Depth-Anything must leave an armed ZoeD_N tap buffer untouched.  Then the cases in TIMED
are timed: REPS CUDA-event windows per build, the order of the two builds alternating (a depth_aa call runs its three modes).
The device name and its power limit are printed with the timings.
"""
import argparse
import ctypes
import json
import os
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

TILE, TILE_BATCH = 256, 16
FRAME = (1080, 1920)
REPS = 7
WINDOW_MS = 150.0
TAP_BYTES = 256 << 20
TIMED = ("depth_anything_v2_vits", "zoedepth_n_384x512", "row_flow_v3", "mlbw_2", "mlbw_4", "depth_aa")
INPAINT_TAPS = [100, 101] + [110 + 10 * k + s for k in range(6) for s in range(8)] + [170, 171, 172, 173]


def load(path):
    from nunif_b200 import _lib
    lib = ctypes.CDLL(os.path.abspath(path))   # RTLD_LOCAL: each build keeps its own symbols and its own static cudart
    for name, (res, args) in _lib.SIGNATURES.items():
        if hasattr(lib, name):
            getattr(lib, name).restype, getattr(lib, name).argtypes = res, args
    return lib


def check(lib, rc):
    if rc != 0:
        raise RuntimeError(lib.nb200_last_error().decode("utf-8", "replace"))


def p(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else None


def stream():
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream().cuda_stream)


def create(lib, kind, sd):
    import torch
    items = [(k, v.detach().to("cpu", torch.float32).contiguous()) for k, v in sd.items()]
    n = len(items)
    names = (ctypes.c_char_p * n)(*[k.encode() for k, _ in items])
    datas = (ctypes.c_void_p * n)(*[v.data_ptr() for _, v in items])
    numels = (ctypes.c_int64 * n)(*[v.numel() for _, v in items])
    h = ctypes.c_void_p()
    check(lib, lib.nb200_model_create(kind, n, names, datas, numels, 0, ctypes.byref(h)))
    return h


def i2i_case(kind, sd_fn, scale, offset, down=1):
    """(weights, inputs, call) of an image-to-image model on one batch of tiles (nb200_model_forward)."""
    import torch

    def inputs(dev):
        g = torch.Generator().manual_seed(kind * 10 + down)
        x = torch.zeros(TILE_BATCH, TILE, TILE, 8, dtype=torch.float16)
        x[..., :3] = torch.rand(TILE_BATCH, TILE, TILE, 3, generator=g).half()
        return {"x": x.to(dev)}

    def call(lib, h, t):
        s = 4 // down if down > 1 else scale
        S = TILE * s - 2 * (32 // down if down > 1 else offset)
        z = torch.full((TILE_BATCH, 3, S, S), 7.0, device=t["x"].device, dtype=torch.float32 if down > 1 else torch.float16)
        check(lib, lib.nb200_model_forward(h, p(t["x"]), TILE_BATCH, TILE, down, p(z), stream()))
        return [z]
    return sd_fn, inputs, call


def depth_case(entry, B, H, W):
    import torch

    def inputs(dev):
        g = torch.Generator().manual_seed(B * H + W)
        return {"x": torch.randn(B, 3, H, W, generator=g).to(dev)}

    def call(lib, h, t):
        out = torch.full((B, H, W), 7.0, device=t["x"].device)
        check(lib, getattr(lib, entry)(h, p(t["x"]), B, H, W, p(out), stream()))
        return [out]
    return inputs, call


def stereo_input(dev, B, C):
    """depth, divergence feature, convergence feature planes as the learned warps take them (C = 3), or the depth alone"""
    import torch
    from nunif_b200 import synth
    d = synth.synth_depth(5, B, *FRAME).reshape(B, 1, *FRAME)
    if C == 1:
        return d.contiguous().to(dev)
    return torch.cat([d, torch.full_like(d, 0.25), torch.full_like(d, 0.5)], 1).contiguous().to(dev)


def cases():
    import torch
    from nunif_b200 import synth
    B, (H, W) = 2, FRAME
    out = []
    for kind, r, off in ((3, 1, 8), (4, 2, 16), (5, 4, 32)):
        out.append((f"swin_unet_{r}x", kind, *i2i_case(kind, lambda r=r: synth.swin_unet_state_dict(0, r), r, off)))
    out.append(("swin_unet_4x.to_2x", 5, *i2i_case(5, lambda: synth.swin_unet_state_dict(0, 4), 4, 32, down=2)))
    out.append(("upcunet", 1, *i2i_case(1, lambda: synth.upcunet_state_dict(0), 2, 36)))
    out.append(("cunet", 2, *i2i_case(2, lambda: synth.cunet_state_dict(0), 1, 28)))
    out.append(("upconv_7", 13, *i2i_case(13, lambda: synth.upconv7_state_dict(0), 2, 14)))
    out.append(("vgg_7", 14, *i2i_case(14, lambda: synth.vgg7_state_dict(0), 1, 7)))
    for enc, kind in (("vits", 6), ("vitb", 8), ("vitl", 9)):
        out.append((f"depth_anything_v2_{enc}", kind, lambda enc=enc: synth.depth_anything_v2_state_dict(0, enc),
                    *depth_case("nb200_depth_anything_forward", 4, 392, 686)))
    for h, w in ((384, 512), (384, 704)):
        out.append((f"zoedepth_n_{h}x{w}", 12, lambda: synth.zoedepth_state_dict(0), *depth_case("nb200_zoedepth_forward", 2, h, w)))

    def row_flow(lib, h, t):
        d = torch.full((B, 1, H, W), 7.0, device=t["x"].device)
        check(lib, lib.nb200_row_flow_delta(h, p(t["x"]), B, H, W, p(d), stream()))
        return [d]
    out.append(("row_flow_v3", 7, lambda: synth.row_flow_v3_state_dict(0), lambda dev: {"x": stereo_input(dev, B, 3)}, row_flow))

    for L in (2, 4):
        def mlbw(lib, h, t, L=L):
            d = torch.full((B, L, H, W), 7.0, device=t["x"].device)
            lw = torch.full_like(d, 7.0)
            check(lib, lib.nb200_mlbw_delta(h, p(t["x"]), B, H, W, p(d), p(lw), stream()))
            return [d, lw]
        out.append((f"mlbw_{L}", 11, lambda L=L: synth.mlbw_state_dict(0, L), lambda dev: {"x": stereo_input(dev, B, 3)}, mlbw))
        if L == 2:   # `small` is read off the missing lv2.2 / lv2.3: shifted blocks pad along x only (pad_y = 0, pad_x = 2)
            small = lambda: {k: v for k, v in synth.mlbw_state_dict(0, 2).items() if not k.startswith(("lv2.2.", "lv2.3."))}
            out.append(("mlbw_2_small", 11, small, lambda dev: {"x": stereo_input(dev, B, 3)}, mlbw))

    def depth_aa(lib, h, t):
        res = []
        for mode in (0, 1, 2):
            o = torch.full((B, 1, H, W), 7.0, device=t["x"].device)
            check(lib, lib.nb200_depth_aa(h, p(t["x"]), B, H, W, mode, p(o), stream()))
            res.append(o)
        return res
    out.append(("depth_aa", 10, lambda: synth.depth_aa_state_dict(0), lambda dev: {"x": stereo_input(dev, B, 1)}, depth_aa))

    def inpaint_inputs(dev):
        g = torch.Generator().manual_seed(15)
        x = torch.rand(B, 3, H, W, generator=g)
        holes = torch.nn.functional.interpolate((torch.rand(B, 1, H // 8, W // 8, generator=g) > 0.8).float(), size=(H, W))
        return {"x": x.to(dev), "mask": holes.contiguous().to(dev)}

    def inpaint(lib, h, t, mirrors=(0, 1)):
        res = []
        for mirror in mirrors:
            o = torch.full_like(t["x"], 7.0)
            check(lib, lib.nb200_light_inpaint(h, p(t["x"]), p(t["mask"]), B, H, W, mirror, p(o), stream()))
            res.append(o)
        return res
    out.append(("light_inpaint_v1", 15, lambda: synth.light_inpaint_v1_state_dict(0), inpaint_inputs, inpaint))
    return out


def tapped(lib, tap_id, buf, fn):
    """fn() with debug tap `tap_id` armed into a zeroed buf; returns (buf copy, fn's outputs)"""
    buf.zero_()
    check(lib, lib.nb200_debug_tap(tap_id, p(buf), buf.numel()))
    try:
        outs = fn()
    finally:
        lib.nb200_debug_tap(-1, None, 0)
    return buf.clone(), outs


def window_ms(fn, n):
    import torch
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    for _ in range(n):
        fn()
    e1.record()
    e1.synchronize()
    return e0.elapsed_time(e1) / n


def time_ab(fns):
    """median / min / max ms per call of each build, REPS windows in alternating order"""
    import torch
    for fn in fns.values():
        for _ in range(3):
            fn()
    torch.cuda.synchronize()
    est = max(window_ms(fn, 2) for fn in fns.values())
    n = max(3, int(WINDOW_MS / max(est, 1e-3)))
    ms = {k: [] for k in fns}
    for r in range(REPS):
        for k in (("base", "new") if r % 2 == 0 else ("new", "base")):
            ms[k].append(window_ms(fns[k], n))
    row = {k: {"median_ms": statistics.median(v), "min_ms": min(v), "max_ms": max(v)} for k, v in ms.items()}
    row["calls_per_window"] = n
    row["new_over_base"] = row["new"]["median_ms"] / row["base"]["median_ms"]
    return row


def main():
    ap = argparse.ArgumentParser(description=__doc__, formatter_class=argparse.RawDescriptionHelpFormatter)
    ap.add_argument("--base", required=True, help="the build to compare against (libnunif_b200.so)")
    ap.add_argument("--new", default=os.path.join(ROOT, "nunif_b200", "libnunif_b200.so"), help="default: this tree's build")
    ap.add_argument("--out", default=None, help="also write the JSON result here")
    args = ap.parse_args()
    import torch
    dev = torch.device("cuda:0")
    torch.cuda.init()
    torch.zeros(1, device=dev)
    libs = {"base": load(args.base), "new": load(args.new)}
    for lib in libs.values():
        check(lib, lib.nb200_check_device(0))
    smi = subprocess.run(["nvidia-smi", "-i", "0", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    info = {"device": torch.cuda.get_device_name(dev), "nvidia_smi": smi}
    print(f"# {info['device']} | name, power limit, max SM clock: {smi}", flush=True)
    taps = {k: torch.empty(TAP_BYTES, dtype=torch.uint8, device=dev) for k in libs}

    rows, timings = [], {}
    with torch.inference_mode():
        for name, kind, sd_fn, inputs, call in cases():
            sd = sd_fn()
            t = inputs(dev)
            h = {k: create(lib, kind, sd) for k, lib in libs.items()}
            del sd
            try:
                got = {k: call(lib, h[k], t) for k, lib in libs.items()}
                torch.cuda.synchronize()
                equal = all(torch.equal(a, b) for a, b in zip(got["base"], got["new"]))
                row = {"case": name, "outputs": len(got["base"]), "equal": equal}
                tap_ids = list(range(15)) if kind == 12 else INPAINT_TAPS if kind == 15 else []
                if tap_ids:
                    differ = []
                    for i in tap_ids:
                        fn = (lambda k: call(libs[k], h[k], t)) if kind == 12 else (lambda k: call(libs[k], h[k], t, (0,)))
                        r = {k: tapped(libs[k], i, taps[k], lambda k=k: fn(k)) for k in libs}
                        if not (torch.equal(r["base"][0], r["new"][0]) and not torch.equal(r["new"][0], torch.zeros_like(r["new"][0]))
                                and torch.equal(r["new"][1][0], got["new"][0])):
                            differ.append(i)
                    row["taps"] = len(tap_ids)
                    row["taps_differ"] = differ
                    row["equal"] = row["equal"] and not differ
                if kind == 6:   # Depth-Anything answers no ZoeD_N tap id
                    row["zoe_taps_answered"] = [i for i in range(15)
                                                if bool(tapped(libs["new"], i, taps["new"], lambda: call(libs["new"], h["new"], t))[0].any())]
                    row["equal"] = row["equal"] and not row["zoe_taps_answered"]
                if name in TIMED:
                    timings[name] = time_ab({k: (lambda k=k: call(libs[k], h[k], t)) for k in libs})
                    tr = timings[name]
                    row["timing"] = tr
                rows.append(row)
                msg = f"{name}: {row['outputs']} output(s) {'identical' if equal else 'DIFFER'}"
                if "taps" in row:
                    msg += f", {row['taps']} taps {'identical' if not row['taps_differ'] else 'DIFFER at ' + str(row['taps_differ'])}"
                if "zoe_taps_answered" in row:
                    msg += f", ZoeD_N tap ids answered: {row['zoe_taps_answered'] or 'none'}"
                if "timing" in row:
                    b, nw = tr["base"], tr["new"]
                    msg += (f"\n    base {b['median_ms']:.3f} ms [{b['min_ms']:.3f}, {b['max_ms']:.3f}]  new {nw['median_ms']:.3f} ms "
                            f"[{nw['min_ms']:.3f}, {nw['max_ms']:.3f}]  new/base {tr['new_over_base']:.3f} ({tr['calls_per_window']} calls/window)")
                print(msg, flush=True)
            finally:
                for k, lib in libs.items():
                    lib.nb200_model_destroy(h[k])
                del t
                torch.cuda.empty_cache()
    result = {"info": info, "cases": rows, "all_equal": all(r["equal"] for r in rows)}
    print(json.dumps(result))
    if args.out:
        os.makedirs(os.path.dirname(os.path.abspath(args.out)), exist_ok=True)
        with open(args.out, "w") as fh:
            json.dump(result, fh, indent=1)
    return 0 if result["all_equal"] else 1


if __name__ == "__main__":
    sys.exit(main())
