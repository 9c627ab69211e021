"""Generate tests/golden/sod_v1.npz by running the REAL reference (nagadomi/nunif, a checkout given by --reference or
$NUNIF_REFERENCE, imported read-only) on the CPU in fp32:
    python oracle/gen_golden_sod.py --reference PATH/TO/nunif

ConvergenceEstimator.__init__ is never called (it downloads the release checkpoint): SODV1 is built with create_model, loaded
with synth.sod_v1_state_dict(0) (strict) and put in eval mode after .fuse(); the estimator is an instance made with __new__
around it.  On the CPU the reference's autocast is disabled, so everything runs in fp32.  Inputs are regenerated from synth:
  net{i}_{sal,cfg}        SODV1.infer's saliency for NET_CASES (frame seeds, H, W, depth seed, h, w): a 1080p landscape
                          frame and a portrait frame, both with a low-resolution depth map
  net{i}_d192c            the top-left 16 x 16 of SODV1.infer's depth_192 (the whole map is F.interpolate of the regenerated
                          depth, which the tests recompute; the corner pins it to the reference)
  net{i}_zpos             depth_position_from_ratio(sal, d192, pos) for pos in POS, [len(POS)][B]
  bg_zpos, flat_zpos      an all-background saliency (-> 0.5) and a constant depth (-> q01) at pos 0.3
  ema_{a,b}, ema_reset    __call__ with enable_ema on EMA_FRAMES in two calls, reset_pts in the first
  e2e_{method}_{left,right}, e2e_conv
                          apply_divergence's path with the estimator (convergence = estimator(im, depth), mapper "none")
                          for E2E_METHODS on E2E frames (B = 3), and the convergences
"""
import argparse
import os
import sys
import tempfile
from types import SimpleNamespace
import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from nunif_b200 import synth  # noqa: E402

OUT = os.path.join(ROOT, "tests", "golden", "sod_v1.npz")
NET_CASES = [((11,), 1080, 1920, 13, 98, 172), ((14,), 640, 360, 15, 60, 34)]
POS = [0.0, 0.3, 0.5, 1.0]
EMA_FRAMES = ((31, 32, 33, 34, 35), 54, 96, 36, 24, 42)
EMA_RESET = [False, True, False, False, False]
E2E = ((41, 42, 43), 24, 40, 44, 24, 40)
E2E_METHODS = ("backward", "forward_fill")
E2E_ARGS = dict(divergence=2.5, convergence=0.3, synthetic_view="both", mapper="none")


def frames(seeds, H, W, dseed, h, w):
    rgb = torch.stack([synth.synth_image(s, 3, H, W) for s in seeds])
    return rgb, synth.synth_depth(dseed, len(seeds), h, w)


def main():
    import iw3.models  # noqa: F401
    from nunif.models import create_model
    from iw3.convergence_estimator import ConvergenceEstimator
    from iw3.backward_warp import apply_divergence_grid_sample
    from iw3.forward_warp import apply_divergence_forward_warp
    model = create_model("iw3.sod_v1").eval()
    model.load_state_dict(synth.sod_v1_state_dict(0), strict=True)
    model = model.fuse()

    def estimator(pos, enable_ema=False):
        est = ConvergenceEstimator.__new__(ConvergenceEstimator)
        est.model, est.convergence, est.device = model, pos, torch.device("cpu")
        est.enable_ema, est.decay, est.convergence_ema = enable_ema, 0.9, None
        return est

    out = {}
    for i, case in enumerate(NET_CASES):
        rgb, d = frames(*case)
        sal, d192 = model.infer(rgb, d)
        frac = float((sal > 0.5).float().mean())
        print(f"net{i}: salient fraction {frac:.3f}")
        assert 0.05 < frac < 0.95
        zp = torch.stack([ConvergenceEstimator.depth_position_from_ratio(sal, d192, p).flatten() for p in POS])
        out.update({f"net{i}_sal": sal, f"net{i}_d192c": d192[..., :16, :16].clone(), f"net{i}_zpos": zp,
                    f"net{i}_cfg": np.array([len(case[0]), *case[1:]], dtype=np.int64)})
        print(f"net{i}: zpos {zp.tolist()}")
        if i == 0:
            out["bg_zpos"] = ConvergenceEstimator.depth_position_from_ratio(torch.zeros_like(sal), d192, 0.3)
            out["flat_zpos"] = ConvergenceEstimator.depth_position_from_ratio(sal, torch.full_like(d192, 0.37), 0.3)
    rgb, d = frames(*EMA_FRAMES)
    est = estimator(0.3, enable_ema=True)
    out["ema_a"] = est(rgb, d, reset_pts=EMA_RESET)
    out["ema_b"] = est(rgb.flip(0), d.flip(0))
    out["ema_raw"] = estimator(0.3)(rgb, d)
    rgb, d = frames(*E2E)
    # apply_divergence with args.state["convergence_model"] (iw3/utils.py:303-340, mapper "none"); iw3.utils itself imports
    # the video stack, so its two branches are called directly
    conv = estimator(E2E_ARGS["convergence"])(rgb, d)
    a = SimpleNamespace(**E2E_ARGS)
    for method in E2E_METHODS:
        if method == "backward":
            left, right = apply_divergence_grid_sample(rgb, d, a.divergence, convergence=conv, synthetic_view=a.synthetic_view)
        else:
            left, right = apply_divergence_forward_warp(rgb, d, a.divergence, convergence=conv, method=method,
                                                        synthetic_view=a.synthetic_view, width_base=False)
        out[f"e2e_{method}_left"], out[f"e2e_{method}_right"] = left, right
    out["e2e_conv"] = conv
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
