"""Generate tests/golden/mask_mlbw.npz by running the REAL reference (nagadomi/nunif, a checkout given by --reference or
$NUNIF_REFERENCE, imported read-only) on the CPU in fp32:
    python oracle/gen_golden_mask_mlbw.py --reference PATH/TO/nunif

Weights: nunif_b200.synth.mask_mlbw_state_dict(0) (sbs.mlbw with hole_mask=True) and synth.light_inpaint_v1_state_dict(0).
  net{i}_{x,delta,lw,logits}       MLBW._forward_delta_only at two sizes (one width not a multiple of 32); x = make_input_tensor
  pp{i}_{cfg,closed,sigmoid,mask}  postprocess_hole_mask on net0_logits (or their flip): the final mask and, for the cases
                                   without dilation, the closed logits and the sigmoid at the target size before the threshold;
                                   cfg = flip, H, W, inner, outer
  lr_{d,c,left,right}              `--method mask_mlbw_l2`: apply_divergence_nn_LR (hole fill of backward_warp.py:329-341)
  drv{i}_{cfg,corner,left,right}   MLBWInpaintImage.forward on a 24 x 96 frame with a 16 x 48 depth map; an eye the view does
                                   not synthesise is the input frame and is not stored;
                                   cfg = seed, divergence, convergence, view (0 both, 1 left, 2 right), inner, outer, max_width,
                                   preserve_screen_border
The sizes are small so that the file stays small; every stage still runs with a depth map smaller than the frame.
The script checks that the thresholded masks cover 3-30 % of the pixels, so the inpainting stage is exercised.
"""
import argparse
import os
import sys
import tempfile
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nunif_b200 import synth  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "mask_mlbw.npz")
NET_CASES = [(3, 1, 48, 100), (4, 1, 20, 96)]                   # (depth seed, B, h, w); divergence 2, convergence 0.5
# flip, H, W, inner, outer: upsampling to a non-integer ratio, the same at equal size, dilations, and the flipped logits
PP_CASES = [(0, 71, 147, 0, 0), (0, 48, 100, 0, 0), (0, 71, 147, 2, 3), (1, 71, 147, 0, 0), (1, 71, 147, 1, 2)]
VIEWS = ["both", "left", "right"]
# seed, divergence, convergence, view, inner, outer, max_width (0 = None), preserve_screen_border
DRV_CASES = [(11, 4.0, 0.5, 0, 0, 0, 0, 0), (11, 4.0, 0.5, 1, 0, 0, 0, 0), (11, 4.0, 0.5, 2, 0, 0, 0, 0),
             (12, 3.0, 0.0, 0, 2, 3, 0, 1), (13, 4.0, 1.0, 0, 1, 1, 96, 0)]
DRV_HW, DRV_DEPTH_HW = (24, 96), (16, 48)
LR_CASE = (5, 1, 24, 48, 32, 64)                                 # seed, B, h, w, H, W


def net_depth(seed, B, h, w):
    return synth.synth_depth(seed, B, h, w)


def drv_inputs(seed, max_width):
    H, W = DRV_HW
    if max_width:
        H, W = H + 8, W + 32      # resized to an even max_width x even height (mlbw_inpaint.py:120-127)
    x = synth.synth_image(seed, 3, H, W).unsqueeze(0)
    depth = synth.synth_depth(seed, 1, *DRV_DEPTH_HW)
    return x, depth


def lr_inputs():
    seed, B, h, w, H, W = LR_CASE
    d = synth.synth_depth(seed, B, h, w)
    c = torch.stack([synth.synth_image(seed * 16 + i, 3, H, W) for i in range(B)])
    return d, c


def _frac(m):
    f = float(m.float().mean())
    assert 0.03 <= f <= 0.30, f"hole mask covers {f:.3f} of the pixels: pick synth.MASK_MLBW_HOLE_BIAS for 3-30 %"
    return f


def main():
    import torch.nn as nn
    import torch.nn.functional as F
    import iw3.models  # noqa: F401
    from nunif.models import create_model
    from iw3 import dilation
    from iw3.backward_warp import apply_divergence_nn_LR, make_input_tensor, postprocess_hole_mask
    from iw3.mlbw_inpaint import MLBWInpaintImage, MASK_MLBW_THRESHOLD
    sd = synth.mask_mlbw_state_dict(0)
    mm = create_model("sbs.mlbw", hole_mask=True).eval()
    mm.load_state_dict(sd, strict=True)
    mm.delta_output = True
    out = {}
    for i, (seed, B, h, w) in enumerate(NET_CASES):
        d = net_depth(seed, B, h, w)
        x = torch.stack([make_input_tensor(None, d[j], divergence=2.0, convergence=0.5, image_width=max(h, w)) for j in range(B)])
        delta, lw, logits = mm(x)
        out.update({f"net{i}_x": x, f"net{i}_delta": delta, f"net{i}_lw": lw, f"net{i}_logits": logits})
        print(f"net{i}: thresholded closed logits cover", _frac(torch.sigmoid(dilation.closing(logits, n_iter=1)) > MASK_MLBW_THRESHOLD))
    for i, cfg in enumerate(PP_CASES):
        flip, H, W, inner, outer = cfg
        lg = out["net0_logits"].flip(-1) if flip else out["net0_logits"]
        closed = dilation.closing(lg, n_iter=1)                                         # backward_warp.py:384-388
        z = closed if (H, W) == tuple(lg.shape[-2:]) else F.interpolate(closed, size=(H, W), mode="bilinear", align_corners=True,
                                                                         antialias=False)
        mask = postprocess_hole_mask(lg, (H, W), MASK_MLBW_THRESHOLD, inner_dilation=inner, outer_dilation=outer)
        out.update({f"pp{i}_cfg": np.array(cfg), f"pp{i}_mask": mask.to(torch.uint8)})
        if inner == 0 and outer == 0:
            out.update({f"pp{i}_closed": closed, f"pp{i}_sigmoid": torch.sigmoid(z)})
        print(f"pp{i}: thresholded mask covers", _frac(torch.sigmoid(z) > MASK_MLBW_THRESHOLD), "dilated", float(mask.float().mean()))
    d, c = lr_inputs()
    left, right = apply_divergence_nn_LR(mm, c, d, 2.0, 0.5, steps=1, synthetic_view="both", enable_amp=False)
    out.update(lr_d=d, lr_c_corner=c[..., :8, :8], lr_left=left, lr_right=right)
    inp = create_model("inpaint.light_inpaint_v1").eval()
    inp.load_state_dict(synth.light_inpaint_v1_state_dict(0), strict=True)
    fi = MLBWInpaintImage.__new__(MLBWInpaintImage)
    nn.Module.__init__(fi)
    fi.model, fi.mask_mlbw, fi.device = inp, mm, torch.device("cpu")
    for i, cfg in enumerate(DRV_CASES):
        seed, div, conv, view, inner, outer, max_width, psb = cfg
        x, depth = drv_inputs(seed, max_width)
        left, right = fi.forward(x, depth, divergence=div, convergence=conv, preserve_screen_border=bool(psb),
                                 synthetic_view=VIEWS[view], inner_dilation=inner, outer_dilation=outer, max_width=max_width or None,
                                 enable_amp=False)
        out.update({f"drv{i}_cfg": np.array(cfg, dtype=np.float64), f"drv{i}_corner": x[..., :8, :8]})
        for tag, eye in (("left", left), ("right", right)):
            if VIEWS[view] in ("both", tag):
                out[f"drv{i}_{tag}"] = eye
            else:
                assert torch.equal(eye, x)
    np.savez_compressed(OUT, **{k: (v.numpy() if torch.is_tensor(v) else np.asarray(v)) for k, v in out.items()})
    print("wrote", OUT, os.path.getsize(OUT) // 1024, "KiB")


if __name__ == "__main__":
    ap = argparse.ArgumentParser()
    ap.add_argument("--reference", default=os.environ.get("NUNIF_REFERENCE"), help="checkout of nagadomi/nunif")
    args = ap.parse_args()
    if not args.reference:
        ap.error("give the reference checkout with --reference or $NUNIF_REFERENCE")
    # the reference creates its home directory on import; keep it out of the (read-only) reference tree
    os.environ.setdefault("NUNIF_HOME", tempfile.mkdtemp(prefix="nunif_home_"))
    sys.path.insert(0, os.path.abspath(args.reference))
    torch.set_grad_enabled(False)
    torch.manual_seed(0)
    main()
