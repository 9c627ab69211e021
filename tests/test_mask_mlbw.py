"""CPU: the mask_mlbw_l2 / mlbw_l2_inpaint oracle against the goldens the real reference produced (tests/golden/mask_mlbw.npz,
oracle/gen_golden_mask_mlbw.py), and the host contract of the engine's mlbw_l2_inpaint side model."""
import os
import sys
import pytest
import torch

from tests.util import load_golden, t
from nunif_b200 import synth
from oracle import mask_mlbw as omm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import gen_golden_mask_mlbw as gg  # noqa: E402


@pytest.fixture(scope="module")
def g():
    return load_golden("mask_mlbw")


@pytest.fixture(scope="module")
def sd():
    return synth.mask_mlbw_state_dict(0)


def test_state_dict_extends_mlbw_l2(sd):
    """The hole head is a fifth lv1_out row; every other tensor is mlbw_state_dict(0, 2)'s."""
    base = synth.mlbw_state_dict(0, 2)
    assert set(sd) == set(base)
    for k, v in base.items():
        if k.startswith("lv1_out.1."):
            assert sd[k].shape[0] == 5 and torch.equal(sd[k][:4], v)
        else:
            assert torch.equal(sd[k], v)


@pytest.mark.parametrize("i", range(len(gg.NET_CASES)))
def test_oracle_network_golden(g, sd, i):
    seed, B, h, w = gg.NET_CASES[i]
    x = t(g[f"net{i}_x"])
    assert torch.equal(x[:, :1], gg.net_depth(seed, B, h, w))
    with torch.inference_mode():
        delta, lw, logits = omm.mask_mlbw_delta(sd, x)
    assert (delta - t(g[f"net{i}_delta"])).abs().max() <= 1e-4
    assert (lw - t(g[f"net{i}_lw"])).abs().max() <= 1e-5
    assert (logits - t(g[f"net{i}_logits"])).abs().max() <= 1e-5


@pytest.mark.parametrize("i", range(len(gg.PP_CASES)))
def test_oracle_postprocess_hole_mask_golden(g, i):
    flip, H, W, inner, outer = gg.PP_CASES[i]
    lg = t(g["net0_logits"])
    lg = lg.flip(-1) if flip else lg
    if f"pp{i}_closed" in g:
        closed, sig, _ = omm.hole_mask_stages(lg, (H, W))
        assert torch.equal(closed, t(g[f"pp{i}_closed"]))
        assert (sig - t(g[f"pp{i}_sigmoid"])).abs().max() <= 1e-6
    assert torch.equal(omm.postprocess_hole_mask(lg, (H, W), omm.THRESHOLD, inner, outer).to(torch.uint8), t(g[f"pp{i}_mask"]))


def test_oracle_mask_mlbw_l2_golden(g, sd):
    d, c = gg.lr_inputs()
    assert torch.equal(d, t(g["lr_d"])) and torch.equal(c[..., :8, :8], t(g["lr_c_corner"]))
    with torch.inference_mode():
        left, right = omm.apply_divergence_nn_LR(sd, c, d, 2.0, 0.5)
    assert (left - t(g["lr_left"])).abs().max() <= 1e-5
    assert (right - t(g["lr_right"])).abs().max() <= 1e-5


@pytest.mark.parametrize("i", range(len(gg.DRV_CASES)))
def test_oracle_mlbw_inpaint_golden(g, sd, i):
    seed, div, conv, view, inner, outer, mw, psb = gg.DRV_CASES[i]
    x, depth = gg.drv_inputs(seed, mw)
    assert torch.equal(x[..., :8, :8], t(g[f"drv{i}_corner"]))
    with torch.inference_mode():
        left, right = omm.mlbw_inpaint(synth.light_inpaint_v1_state_dict(0), sd, x, depth, div, conv, gg.VIEWS[view], inner, outer,
                                       mw or None, bool(psb))
    for tag, eye in (("left", left), ("right", right)):
        if gg.VIEWS[view] in ("both", tag):
            assert (eye - t(g[f"drv{i}_{tag}"])).abs().max() <= 1e-5
        else:
            assert f"drv{i}_{tag}" not in g and torch.equal(eye, x)     # the frame itself: not stored


def test_goldens_exercise_the_inpainting(g):
    """Every eye of the driver goldens has holes to paint: the masks the generator checked cover 3-30 % of the pixels."""
    for i in range(len(gg.PP_CASES)):
        if f"pp{i}_sigmoid" in g:
            f = float((t(g[f"pp{i}_sigmoid"]) > omm.THRESHOLD).float().mean())
            assert 0.03 <= f <= 0.30, (i, f)


def _ckpt(tmp_path, **data):
    p = tmp_path / "m.pth"
    torch.save(data, p)
    return str(p)


def test_mask_mlbw_checkpoint_checks(tmp_path, sd):
    from nunif_b200.iw3.mlbw_inpaint import load_mask_mlbw_state_dict
    with pytest.raises(FileNotFoundError):
        load_mask_mlbw_state_dict(str(tmp_path / "iw3_mask_mlbw_l2_d1_20250903.pth"))
    with pytest.raises(ValueError, match="name"):
        load_mask_mlbw_state_dict(_ckpt(tmp_path, name="sbs.row_flow_v3", kwargs={"hole_mask": True}, state_dict=sd))
    with pytest.raises(ValueError, match="hole_mask"):
        load_mask_mlbw_state_dict(_ckpt(tmp_path, name="sbs.mlbw", kwargs={"num_layers": 2}, state_dict=sd))
    with pytest.raises(ValueError, match="hole_mask"):
        load_mask_mlbw_state_dict(_ckpt(tmp_path, name="sbs.mlbw", kwargs={"hole_mask": False}, state_dict=sd))
    got = load_mask_mlbw_state_dict(_ckpt(tmp_path, name="sbs.mlbw", kwargs={"num_layers": 2, "hole_mask": True}, state_dict=sd))
    assert set(got) == set(sd)


def test_default_mask_mlbw_checkpoint_path():
    from nunif_b200.iw3.mlbw_inpaint import default_mask_mlbw_checkpoint
    from nunif_b200.iw3.base_depth_model import HUB_MODEL_DIR
    assert default_mask_mlbw_checkpoint() == os.path.join(HUB_MODEL_DIR, "checkpoints", "iw3_mask_mlbw_l2_d1_20250903.pth")


def test_mlbw_inpaint_surface():
    from nunif_b200.iw3.mlbw_inpaint import MLBWInpaint
    mi = object.__new__(MLBWInpaint)
    mi.mode = "image"
    with pytest.raises(NotImplementedError, match="video"):
        mi.set_mode("video")
    mi.set_mode("image")
    assert mi.flush() == (None, None)
    with mi.compile_context():
        pass
    with pytest.raises(NotImplementedError):
        mi.infer(torch.rand(1, 3, 8, 8), torch.rand(1, 1, 8, 8), 2.0, 0.5, enable_amp=False)
