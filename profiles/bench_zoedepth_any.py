"""ZoeD_Any_N (iw3's default depth model) on the engine against PyTorch running oracle/zoedepth_any.py under fp16 autocast, with
seeded full-size weights (ViT-L/14).  Per case (1080p frames at B = 4, 4K frames at B = 2; both become 392 x 700 network inputs):
  * network ms per call, engine vs PyTorch, alternated, and the outputs of both against the fp32 oracle at the timed size;
  * ZoeDepthAnythingModel.infer ms per frame (preprocess, network, crop, negation);
  * the iw3 frame path in frames/s: infer (dilate_edge 2) -> minmax normalise with the div_6 mapper -> apply_divergence
    (forward_fill) -> SBS.
Prints the card, its power limit and max SM clock.  Results go to stdout and, with --out, to DIR/result.json.
    python profiles/bench_zoedepth_any.py [--iters 10] [--out DIR]
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
from nunif_b200.iw3 import create_depth_model, apply_divergence  # noqa: E402
from nunif_b200.iw3.zoedepth_preprocess import batch_preprocess  # noqa: E402
from oracle import zoedepth_any as oza  # noqa: E402


def timed(fn, iters):
    ev = [torch.cuda.Event(enable_timing=True) for _ in range(2)]
    ev[0].record()
    for _ in range(iters):
        fn()
    ev[1].record()
    torch.cuda.synchronize()
    return ev[0].elapsed_time(ev[1]) / iters


def err(a, b):
    d = (a.float() - b.float()).abs()
    return dict(max=float(d.max()), mean=float(d.mean()))


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--iters", type=int, default=10)
    ap.add_argument("--out", default=None, help="directory for result.json")
    a = ap.parse_args()
    q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv,noheader"], capture_output=True,
                       text=True).stdout.strip()
    print("card:", q)
    dev = "cuda:0"
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    sd = synth.zoedepth_any_state_dict(0, None, normed=False)
    sdc = {k: v.to(dev) for k, v in sd.items()}
    model = create_depth_model("ZoeD_Any_N").load_state_dict(sd, gpu=0)
    model.disable_ema()
    args = argparse.Namespace(method="forward_fill", mapper="div_6", convergence=0.5, divergence=2.0, synthetic_view="both",
                              state={"convergence_model": None}, preserve_screen_border=False, stereo_width=None, warp_steps=None)
    rows = []
    for (H, W, B) in ((1080, 1920, 4), (2160, 3840, 2)):
        x = synth.synth_image(1, 3, H, W, smooth=False).to(dev).unsqueeze(0).repeat(B, 1, 1, 1).contiguous()
        xp, pad_h, pad_w = batch_preprocess(x, h_height=392, v_height=518, ensure_multiple_of=14)

        def net_eng():
            return model.model(xp)

        def net_ref():
            with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
                return oza.zoedepth_any_forward(sdc, xp, oza.ZOED_ANY)

        def infer():
            with torch.inference_mode():
                return model.infer(x, tta=False, edge_dilation=0)

        def frame_path():
            with torch.inference_mode():
                depth = model.infer(x, tta=False, edge_dilation=2)
                depth = torch.stack(model.minmax_normalize(depth))
                left, right = apply_divergence(depth, x, args, None)
                return torch.cat([left, right], dim=3).clamp_(0, 1)

        for f in (net_eng, net_ref, infer, frame_path):
            f(); f()
        torch.cuda.synchronize()
        with torch.no_grad():
            got, amp = net_eng(), net_ref().float()
            ref32 = oza.zoedepth_any_forward(sdc, xp.float(), oza.ZOED_ANY)
        e_eng, e_amp = err(got, ref32), err(amp, ref32)
        n0 = _lib.lib().nb200_launch_count()
        net_eng()
        launches = _lib.lib().nb200_launch_count() - n0
        te = tr = 0.0
        for _ in range(3):       # alternate the two
            te += timed(net_eng, a.iters) / 3
            tr += timed(net_ref, a.iters) / 3
        ti = timed(infer, a.iters)
        tf = timed(frame_path, a.iters)
        row = dict(H=H, W=W, B=B, net_input=list(xp.shape[-2:]), pads=[pad_h, pad_w], engine_net_ms=te, torch_amp_net_ms=tr,
                   speedup=tr / te, infer_ms_per_frame=ti / B, iw3_frame_fps=1000.0 * B / tf, launches_per_call=int(launches),
                   engine_vs_fp32=e_eng, torch_amp_vs_fp32=e_amp, depth_range=[float(ref32.min()), float(ref32.max())])
        rows.append(row)
        print(json.dumps(row))
    if a.out:
        os.makedirs(a.out, exist_ok=True)
        with open(os.path.join(a.out, "result.json"), "w") as fh:
            json.dump(dict(card=q, rows=rows), fh, indent=1)


if __name__ == "__main__":
    main()
