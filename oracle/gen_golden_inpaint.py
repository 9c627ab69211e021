"""Generate tests/golden/light_inpaint.npz by running the REAL reference (nagadomi/nunif, a checkout given by --reference or
$NUNIF_REFERENCE, imported read-only) on the CPU in fp32:
    python oracle/gen_golden_inpaint.py --reference PATH/TO/nunif

Weights: nunif_b200.synth.light_inpaint_v1_state_dict(0).  Inputs are not stored: the tests rebuild them from the seeds
(oracle.light_inpaint.net_inputs, synth.synth_image / synth_depth) and an 8 x 8 corner of each pins them against drift.
  net{i}_{seed,hw,corner,z,blur}   LightInpaintV1.infer(x, mask) at an odd size, a size with W % 64 == 0 and a wide one;
                                   blur = the preprocessed mask clamp(blur15(mask) + mask, 0, 1)
  mask_{src,closing,outer,inner}   mask_closing(mask > 0), dilate_outer(., 3, base_width), dilate_inner(., 2, base_width)
                                   on a 37 x 90 mask with base_width 45 (run lengths 6 and 4)
  drv{i}_{cfg,left,right}          ForwardInpaintImage.forward on a 32 x 128 frame with a 32 x 64 depth map (base_width != W);
                                   cfg = seed, divergence, convergence, view (0 both, 1 left, 2 right), inner, outer, max_width
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
from oracle import light_inpaint as oli  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "light_inpaint.npz")
NET_CASES = [(3, 45, 70), (4, 36, 128), (5, 33, 200)]          # (seed, H, W), batch 1
MASK_CASE = (7, 37, 90, 45)                                      # seed, H, W, base_width
VIEWS = ["both", "left", "right"]
# seed, divergence, convergence, view, inner, outer, max_width (0 = None)
DRV_CASES = [(11, 10.0, 0.5, 0, 0, 0, 0), (11, 10.0, 0.5, 1, 0, 0, 0), (11, 10.0, 0.5, 2, 0, 0, 0),
             (12, 8.0, 0.0, 0, 2, 3, 0), (13, 10.0, 1.0, 0, 1, 1, 128)]
DRV_HW, DRV_DEPTH_HW = (32, 128), (32, 64)


def drv_inputs(seed, max_width):
    H, W = DRV_HW
    if max_width:
        H, W = H + 8, W + 32      # resized to an even max_width x even height (forward_inpaint.py:74-81)
    x = synth.synth_image(seed, 3, H, W).unsqueeze(0)
    depth = synth.synth_depth(seed, 1, *DRV_DEPTH_HW)
    return x, depth


def main():
    import torch.nn as nn
    import iw3.models  # noqa
    from nunif.models import create_model
    from iw3 import dilation
    from iw3.forward_inpaint import ForwardInpaintImage
    sd = synth.light_inpaint_v1_state_dict(0)
    m = create_model("inpaint.light_inpaint_v1").eval()
    m.load_state_dict(sd, strict=True)
    out = {}
    for i, (seed, h, w) in enumerate(NET_CASES):
        x, mask = oli.net_inputs(seed, 1, h, w)
        _, blur = m.preprocess(x, mask)
        out.update({f"net{i}_seed": seed, f"net{i}_hw": np.array([h, w]), f"net{i}_corner": x[..., :8, :8],
                    f"net{i}_z": m.infer(x, mask), f"net{i}_blur": blur})
    seed, h, w, bw = MASK_CASE
    src = oli.hole_mask(seed, 1, h, w, frac=0.05)
    closed = dilation.mask_closing(src > 0)
    outer = dilation.dilate_outer(closed, n_iter=3, base_width=bw)
    inner = dilation.dilate_inner(outer, n_iter=2, base_width=bw)
    out.update(mask_case=np.array(MASK_CASE), mask_src=src.to(torch.uint8), mask_closing=closed.to(torch.uint8),
               mask_outer=outer.to(torch.uint8), mask_inner=inner.to(torch.uint8))
    fi = ForwardInpaintImage.__new__(ForwardInpaintImage)
    nn.Module.__init__(fi)
    fi.model = m
    for i, cfg in enumerate(DRV_CASES):
        seed, div, conv, view, inner_d, outer_d, max_width = cfg
        x, depth = drv_inputs(seed, max_width)
        left, right = fi.forward(x, depth, divergence=div, convergence=conv, synthetic_view=VIEWS[view],
                                 inner_dilation=inner_d, outer_dilation=outer_d, max_width=max_width or None)
        out.update({f"drv{i}_cfg": np.array(cfg, dtype=np.float64), f"drv{i}_corner": x[..., :8, :8],
                    f"drv{i}_left": left, f"drv{i}_right": right})
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
