"""CPU: the forward_inpaint oracle against the goldens the real reference produced (tests/golden/light_inpaint.npz,
oracle/gen_golden_inpaint.py), and the host contract of the engine's forward_inpaint side model."""
import os
import sys
import types
import pytest
import torch

from tests.util import load_golden, t
from nunif_b200 import synth
from oracle import light_inpaint as oli

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import gen_golden_inpaint as gg  # noqa: E402


@pytest.fixture(scope="module")
def g():
    return load_golden("light_inpaint")


@pytest.fixture(scope="module")
def sd():
    return synth.light_inpaint_v1_state_dict(0)


def test_state_dict_matches_reference_keys(sd):
    assert len(sd) == 81
    assert sd["mask_bias"].abs().mean() > 0.1


@pytest.mark.parametrize("i", range(3))
def test_oracle_network_golden(g, sd, i):
    h, w = (int(v) for v in g[f"net{i}_hw"])
    x, mask = oli.net_inputs(int(g[f"net{i}_seed"]), 1, h, w)
    assert torch.equal(x[..., :8, :8], t(g[f"net{i}_corner"]))
    _, blur = oli.prepare_mask(mask, x)
    assert (blur - t(g[f"net{i}_blur"])).abs().max() <= 1e-6
    z = oli.infer(sd, x, mask)
    assert (z - t(g[f"net{i}_z"])).abs().max() <= 1e-5
    # every stage shows: the holes get values far from the hole-zeroed input, and the output spans [0, 1]
    assert z.min() == 0 and z.max() == 1


def test_oracle_mask_ops_golden(g):
    seed, h, w, bw = (int(v) for v in g["mask_case"])
    src = oli.hole_mask(seed, 1, h, w, frac=0.05)
    assert torch.equal(src.to(torch.uint8), t(g["mask_src"]))
    c = oli.mask_closing(src > 0)
    assert torch.equal(c.to(torch.uint8), t(g["mask_closing"]))
    o = oli.dilate_outer(c, 3, bw)
    assert torch.equal(o.to(torch.uint8), t(g["mask_outer"]))
    assert torch.equal(oli.dilate_inner(o, 2, bw).to(torch.uint8), t(g["mask_inner"]))


@pytest.mark.parametrize("i", range(len(gg.DRV_CASES)))
def test_oracle_driver_golden(g, sd, i):
    seed, div, conv, view, inner, outer, mw = gg.DRV_CASES[i]
    x, depth = gg.drv_inputs(seed, mw)
    assert torch.equal(x[..., :8, :8], t(g[f"drv{i}_corner"]))
    left, right = oli.forward_inpaint(sd, x, depth, div, conv, gg.VIEWS[view], inner, outer, mw or None)
    assert (left - t(g[f"drv{i}_left"])).abs().max() <= 1e-5
    assert (right - t(g[f"drv{i}_right"])).abs().max() <= 1e-5


def test_flop_count():
    """233 GFLOP per eye at 1080p, 905 at 4K (torch.utils.flop_counter on the reference)."""
    assert round(oli.flops(1080, 1920) / 1e9) == 233
    assert round(oli.flops(2160, 3840) / 1e9) == 905


def test_missing_checkpoint_raises(tmp_path):
    from nunif_b200.iw3.forward_inpaint import load_state_dict
    with pytest.raises(FileNotFoundError):
        load_state_dict(str(tmp_path / "iw3_light_inpaint_v1_20250919.pth"))


def test_wrong_checkpoint_name_raises(tmp_path, sd):
    from nunif_b200.iw3.forward_inpaint import load_state_dict
    p = tmp_path / "x.pth"
    torch.save({"name": "sbs.row_flow_v3", "state_dict": sd}, p)
    with pytest.raises(ValueError):
        load_state_dict(str(p))
    torch.save({"name": "inpaint.light_inpaint_v1", "state_dict": sd}, p)
    assert set(load_state_dict(str(p))) == set(sd)


def test_default_checkpoint_path():
    from nunif_b200.iw3.forward_inpaint import default_checkpoint
    from nunif_b200.iw3.base_depth_model import HUB_MODEL_DIR
    assert default_checkpoint() == os.path.join(HUB_MODEL_DIR, "checkpoints", "iw3_light_inpaint_v1_20250919.pth")


def test_mlbw_l2_inpaint_raises():
    from nunif_b200.iw3 import apply_divergence
    args = types.SimpleNamespace(method="mlbw_l2_inpaint", mapper="none", convergence=0.5, divergence=2.0, synthetic_view="both")
    with pytest.raises(NotImplementedError, match="mlbw_l2_inpaint"):
        apply_divergence(torch.rand(1, 8, 8), torch.rand(3, 8, 8), args, None)


def test_video_mode_and_fp32_raise():
    from nunif_b200.iw3.forward_inpaint import ForwardInpaint
    fi = object.__new__(ForwardInpaint)
    fi.mode = "image"
    with pytest.raises(NotImplementedError, match="video"):
        fi.set_mode("video")
    fi.set_mode("image")
    assert fi.flush() == (None, None)
    with fi.compile_context():
        pass
    with pytest.raises(NotImplementedError):
        fi.infer(torch.rand(1, 3, 8, 8), torch.rand(1, 1, 8, 8), 2.0, 0.5, enable_amp=False)
