"""waifu2x.upconv_7 / waifu2x.vgg_7 on the CPU: the oracle pinned to the reference's goldens (tests/golden/upconv_7.npz,
vgg_7.npz, written by oracle/gen_golden_legacy.py), the tile planner and tile-size contract, and the host-side surface
(model table, hub table, refusals).  No GPU needed."""
import ctypes

import pytest
import torch

from nunif_b200 import synth
from oracle import legacy as ol, seam_blending as osb
from tests.util import load_golden, t

torch.set_grad_enabled(False)

MODELS = [("upconv_7", synth.upconv7_state_dict, ol.upconv7_forward, ol.UPCONV_7),
          ("vgg_7", synth.vgg7_state_dict, ol.vgg7_forward, ol.VGG_7)]
IDS = [m[0] for m in MODELS]


def maxdiff(a, b):
    return float((t(a).double() - t(b).double()).abs().max())


def inputs(g):
    """The forward inputs and the rendered image of a golden file, rebuilt from the seeds it stores."""
    x = torch.stack([synth.synth_image(int(s), 3, 104, 104, smooth=bool(sm)) for s, sm in g["x_seeds"]])
    x_odd = torch.stack([synth.synth_image(int(s), 3, 61, 61, smooth=bool(sm)) for s, sm in g["x_odd_seeds"]])
    img = synth.synth_image(int(g["img_seed"]), 3, *(int(v) for v in g["img_hw"]))
    return {"x": x, "x_odd": x_odd, "img": img}


@pytest.mark.parametrize("name,sdf,fn,spec", MODELS, ids=IDS)
def test_oracle_matches_reference_goldens(name, sdf, fn, spec):
    g = load_golden(name)
    sd = sdf(0)
    inp = inputs(g)
    for k in ("x", "x_odd", "img"):                                                # synth drift shows here
        assert torch.equal(inp[k][..., :16, :16], t(g[k + "_corner"])), k
    for xk, zk in (("x", "z"), ("x_odd", "z_odd")):
        z = fn(sd, inp[xk])
        assert z.shape == t(g[zk]).shape
        assert maxdiff(z, g[zk]) < 2e-5, (name, xk)
    y = osb.tiled_render(inp["img"], lambda b: fn(sd, b), spec["scale"], spec["offset"], spec["blend_size"],
                         int(g["tile_size"]), int(g["batch_size"]))
    assert y.shape == t(g["render"]).shape
    assert maxdiff(y, g["render"]) < 2e-5
    # the render covers 2 x 2 tiles in two batches (the second one ragged), so it has seams in both directions
    p = osb.create_config(*inp["img"].shape[1:], spec["scale"], spec["offset"], int(g["tile_size"]), 0)
    assert (p["h_blocks"], p["w_blocks"]) == (2, 2) and 4 % int(g["batch_size"]) != 0


@pytest.mark.parametrize("name", IDS)
def test_golden_outputs_exercise_both_clamps(name):
    g = load_golden(name)
    for k in ("z", "z_odd", "render"):
        z = t(g[k])
        assert float(((z > 0) & (z < 1)).double().mean()) >= 0.2, (name, k)
        assert bool((z == 0).any()) and bool((z == 1).any()), (name, k)


@pytest.mark.parametrize("name,spec", [("upconv_7", ol.UPCONV_7), ("vgg_7", ol.VGG_7)])
def test_seam_planner_bit_exact(name, spec):
    """The oracle planner and the library's planner (the one nb200_tiled_render uses) against SeamBlending.create_config."""
    from nunif_b200 import _lib
    g = load_golden(name)
    assert (int(g["scale"]), int(g["offset"])) == (spec["scale"], spec["offset"])
    for case, want in zip(g["cases"], g["configs"]):
        h, w, scale, offset, tile, blend = (int(v) for v in case)
        p = osb.create_config(h, w, scale, offset, tile, blend)
        got = [p["y_h"], p["y_w"], p["h_blocks"], p["w_blocks"], *p["pad"],
               p["y_buffer_h"], p["y_buffer_w"], p["input_tile_step"], p["output_tile_step"]]
        assert got == [int(v) for v in want], (case, got, want)
        cfg = _lib.TileConfig()
        _lib.check(_lib.lib().nb200_tile_config_create(h, w, scale, offset, tile, blend, ctypes.byref(cfg)))
        d = cfg.as_dict()
        assert [d["h_blocks"], d["w_blocks"], d["input_tile_step"], d["output_tile_step"]] == [int(v) for v in (want[2], want[3], want[10], want[11])]


@pytest.mark.parametrize("name", IDS)
def test_every_tile_size_is_valid(name):
    from nunif_b200.nunif import models
    g = load_golden(name)
    validator = models._validator_for("waifu2x." + name)
    for q, want in zip(g["query"], g["tile"]):
        assert osb.find_valid_tile_size(ol.any_tile_validator, int(q)) == int(want)
        assert int(want) == int(q)
        assert validator(int(q))


def test_model_table():
    from nunif_b200.nunif import models
    assert models.KINDS["waifu2x.upconv_7"] == 13 and models.KINDS["waifu2x.vgg_7"] == 14
    # the swin and cunet validators are unchanged
    assert models._validator_for("waifu2x.cunet") is models._cunet_validator
    assert models._validator_for("waifu2x.upcunet") is models._cunet_validator
    assert models._validator_for("waifu2x.swin_unet_4x") is models._swin_validator


def test_hub_tables():
    from os import path
    from nunif_b200.waifu2x import hub
    table = hub._types("/models")
    for style in ("art", "photo"):
        assert table[f"upconv_7/{style}"] == path.join("/models", "upconv_7", style)
        assert f"upconv_7/{style}" in hub.NO_4X_MODELS
    assert "upconv_7" not in table          # bare style names stay swin_unet
    assert table["art"] == path.join("/models", "swin_unet", "art")


@pytest.mark.parametrize("model_type", ["upconv_7/art", "upconv_7/photo"])
def test_hub_refuses_4x_methods(model_type):
    from nunif_b200.waifu2x import hub
    m = object.__new__(hub.Waifu2xImageModel)          # the mode table only; no checkpoints are loaded
    m.model_type = model_type
    for method in ("scale4x", "noise_scale4x"):
        with pytest.raises(ValueError, match="does not support"):
            m.set_mode(method, 1 if method.startswith("noise") else -1)
    m.set_mode("noise_scale", 3)
    assert (m.method, m.noise_level) == ("noise_scale", 3)


@pytest.mark.parametrize("name,sdf", [("waifu2x.upconv_7", synth.upconv7_state_dict), ("waifu2x.vgg_7", synth.vgg7_state_dict)])
def test_create_model_refuses_other_channel_counts(name, sdf, monkeypatch):
    from nunif_b200 import _lib
    from nunif_b200.nunif.models import create_model

    def no_cuda(*a, **k):
        raise AssertionError("the refusal must come before any CUDA call")
    monkeypatch.setattr(_lib, "lib", no_cuda)
    for k in ("in_channels", "out_channels"):
        with pytest.raises(NotImplementedError, match=k):
            create_model(name, sdf(0), **{k: 1})
