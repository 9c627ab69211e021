"""Generate tests/golden/row_flow_v2.npz by running the REAL reference (nagadomi/nunif, a checkout given by --reference or
$NUNIF_REFERENCE, imported read-only) on the CPU in fp32 (enable_amp=False):
    python oracle/gen_golden_row_flow_v2.py --reference PATH/TO/nunif

Weights: nunif_b200.synth.row_flow_v2_state_dict(0) for `sbs.row_flow_v2`, and synth.row_flow_v3_state_dict(2) for
`sbs.row_flow_v3` with symmetric = True (the row_flow_v3_sym network: the same module, its own weights), both loaded with
strict=True.
  net{i}_{x,delta}              RowFlowV2._forward_delta_only (x component) at (B, h, w) = NET_CASES, including h = 1 and a
                                width (5) narrower than the receptive field; x = make_input_tensor (image_width = max(h, w))
  v2_{d,c}_corner               8 x 8 corners of the LR cases' depth (1, 1, 20, 40) and larger frame (1, 3, 30, 64), which
                                lr_inputs() regenerates from synth
  v2lr{i}_{cfg,left,right}      apply_divergence_nn_LR(row_flow_v2) for LR_CASES; cfg = divergence, convergence, view
                                (0 both, 1 left, 2 right), steps, preserve_screen_border.  An eye the view does not synthesise
                                is the input frame and is not stored.
  sym{i}_{cfg,d,c,left,right}   apply_divergence_nn_LR(row_flow_v3_sym) for SYM_CASES; cfg = divergence, convergence, view,
                                depth h, depth w, frame H, frame W; d and c are 8 x 8 corners of sym_inputs(i, ...).  One case has a portrait depth map (H > W), which pins the
                                symmetric driver's image_width = W.
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

OUT = os.path.join(ROOT, "tests", "golden", "row_flow_v2.npz")
NET_CASES = [(1, 2, 70, 130), (2, 1, 1, 40), (3, 1, 9, 5), (4, 2, 17, 111)]        # (depth seed, B, h, w)
VIEWS = ["both", "left", "right"]
LR_CASES = [(2.0, 0.5, 0, 1, 0), (2.5, 0.3, 2, 1, 0), (3.0, 0.5, 1, 1, 0), (4.0, 0.5, 0, 2, 0), (3.0, 0.4, 0, 1, 1),
            (4.0, 0.5, 2, 2, 1)]
SYM_CASES = [(2.0, 0.5, 0, 20, 40, 30, 64), (2.5, 0.3, 1, 20, 40, 30, 64), (2.5, 0.3, 2, 20, 40, 30, 64),
             (3.0, 0.5, 0, 40, 24, 60, 36)]


def lr_inputs():
    return synth.synth_depth(7, 1, 20, 40), synth.synth_image(70, 3, 30, 64).unsqueeze(0)


def sym_inputs(i, h, w, H, W):
    return synth.synth_depth(80 + i, 1, h, w), synth.synth_image(90 + i, 3, H, W).unsqueeze(0)


def main():
    import iw3.models  # noqa: F401
    from nunif.models import create_model
    from iw3.backward_warp import apply_divergence_nn_LR, make_input_tensor
    v2 = create_model("sbs.row_flow_v2").eval()
    v2.load_state_dict(synth.row_flow_v2_state_dict(0), strict=True)
    v2.delta_output = True
    v3s = create_model("sbs.row_flow_v3").eval()
    v3s.load_state_dict(synth.row_flow_v3_state_dict(2), strict=True)
    v3s.symmetric, v3s.delta_output = True, True     # stereo_model_factory.load_row_flow_model, row_flow_v3_sym
    out = {}
    for i, (seed, B, h, w) in enumerate(NET_CASES):
        d = synth.synth_depth(seed, B, h, w)
        x = torch.stack([make_input_tensor(None, d[j], divergence=2.0, convergence=0.5, image_width=max(h, w)) for j in range(B)])
        delta = v2(x)
        assert float(delta[:, 1].abs().max()) == 0.0
        out.update({f"net{i}_x": x, f"net{i}_delta": delta[:, :1]})
        print(f"net{i}: |delta| max {float(delta.abs().max()):.3f} mean {float(delta.abs().mean()):.3f}")
    d, c = lr_inputs()
    out.update(v2_d_corner=d[..., :8, :8], v2_c_corner=c[..., :8, :8])
    for i, cfg in enumerate(LR_CASES):
        div, conv, view, steps, psb = cfg
        left, right = apply_divergence_nn_LR(v2, c, d, div, conv, steps, synthetic_view=VIEWS[view], preserve_screen_border=bool(psb),
                                             enable_amp=False)
        out[f"v2lr{i}_cfg"] = np.array(cfg, dtype=np.float64)
        for tag, eye in (("left", left), ("right", right)):
            if VIEWS[view] in ("both", tag):
                out[f"v2lr{i}_{tag}"] = eye
            else:
                assert torch.equal(eye, c)
    for i, cfg in enumerate(SYM_CASES):
        div, conv, view, h, w, H, W = cfg
        d, c = sym_inputs(i, h, w, H, W)
        left, right = apply_divergence_nn_LR(v3s, c, d, div, conv, None, synthetic_view=VIEWS[view], enable_amp=False)
        out.update({f"sym{i}_cfg": np.array(cfg, dtype=np.float64), f"sym{i}_d": d[..., :8, :8], f"sym{i}_c": c[..., :8, :8]})
        for tag, eye in (("left", left), ("right", right)):
            if VIEWS[view] in ("both", tag):
                out[f"sym{i}_{tag}"] = eye
            else:
                assert torch.equal(eye, c)
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
