"""CPU-only checks of host-side logic of the Python mirror (no CUDA calls): checkpoint-directory rules of Waifu2x
(waifu2x/utils.py:128-216), method normalisation (waifu2x/hub.py:151-163), edge_dilation parsing (iw3/dilation.py:5-27),
the learned-warp feature values (iw3/backward_warp.py:8-15) and the launch-list summariser."""
import os
import types
import pytest


class _Fake:
    def __init__(self, tag):
        self.tag = tag

    def to_2x(self):
        return _Fake(self.tag + "->2x")

    def to_1x(self):
        return _Fake(self.tag + "->1x")


def _ctx(tmp_path, files):
    from nunif_b200.waifu2x.utils import Waifu2x
    for f in files:
        open(os.path.join(tmp_path, f), "w").close()
    w = Waifu2x(str(tmp_path), [0])
    w.load_model_by_name = lambda filename: _Fake(filename)      # no GPU: record which file would be loaded
    return w


def test_waifu2x_checkpoint_rules_4x_only_directory(tmp_path):
    w = _ctx(tmp_path, ["scale4x.pth", "noise0_scale4x.pth", "noise1_scale4x.pth", "noise2_scale4x.pth", "noise3_scale4x.pth"])
    w.load_model_all(load_4x=True)
    assert w.scale4x_model.tag == "scale4x.pth" and w.scale_model.tag == "scale4x.pth->2x"
    for n in range(4):
        assert w.noise_scale4x_models[n].tag == f"noise{n}_scale4x.pth"
        assert w.noise_scale_models[n].tag == f"noise{n}_scale4x.pth->2x"
        assert w.noise_models[n].tag == f"noise{n}_scale4x.pth->1x"


def test_waifu2x_checkpoint_rules_prefer_native_files_and_errors(tmp_path):
    w = _ctx(tmp_path, ["scale2x.pth", "noise2.pth", "noise2_scale2x.pth"])
    w.load_model("noise_scale", 2)
    assert w.noise_scale_models[2].tag == "noise2_scale2x.pth" and w.scale_model.tag == "scale2x.pth"   # companion scale model
    w.load_model("noise", 2)
    assert w.noise_models[2].tag == "noise2.pth"
    with pytest.raises(FileNotFoundError):
        w.load_model("scale4x", -1)
    with pytest.raises(FileNotFoundError):
        w.load_model("noise", 1)                 # neither noise1.pth nor noise1_scale4x.pth
    with pytest.raises(AssertionError):
        w.load_model("noise", 7)
    with pytest.raises(ValueError):
        w._load_model("bogus", 0)
    first = w.noise_models[2]
    w.load_model("noise", 2)
    assert w.noise_models[2] is first            # cached


def test_normalize_method_and_dilation_parse():
    from nunif_b200.waifu2x.hub import Waifu2xImageModel
    nm = Waifu2xImageModel.normalize_method
    assert nm("scale2x", -1) == "scale" and nm("scale", 1) == "noise_scale" and nm("scale4x", 0) == "noise_scale4x"
    assert nm("noise_scale2x", 2) == "noise_scale" and nm(None, 0) is None and nm("noise", 3) == "noise"
    from nunif_b200.iw3.dilation import edge_dilation_parse, edge_dilation_is_enabled
    assert edge_dilation_parse(2) == (2, 2) or tuple(edge_dilation_parse(2)) == (2, 2)
    assert tuple(edge_dilation_parse([2, 1])) == (2, 1)
    assert edge_dilation_is_enabled([0, 1]) and not edge_dilation_is_enabled(0) and not edge_dilation_is_enabled([0, 0])
    with pytest.raises((ValueError, TypeError)):
        edge_dilation_parse("x")


def test_row_flow_feature_values():
    from nunif_b200.iw3.row_flow import make_divergence_feature_value
    d, c = make_divergence_feature_value(2.0, 0.5, 1920)
    assert d == pytest.approx(2.0 * 0.5 * 0.01 * 1920 / 32.0) and c == pytest.approx(-2.0 * 0.5 * 0.01 * 1920 * 0.5 / 32.0)


@pytest.mark.parametrize("g,ph,pw", [(24, 24, 32), (24, 24, 44), (6, 4, 6), (6, 6, 6), (5, 9, 3)])
def test_zoe_relative_position_table_resample_matches_oracle(g, ph, pw):
    """Host logic of the ZoeD_N path (no GPU): the BEiT relative-position table resampled for a non-training token grid
    (csrc/zoe_model.cu zoe_resample_table) against the oracle's F.interpolate restatement of MiDaS `_get_rel_pos_bias`."""
    import ctypes
    import torch
    import torch.nn.functional as F
    from nunif_b200 import _lib
    heads = 4
    S = 2 * g - 1
    tab = torch.randn(S * S + 3, heads, generator=torch.Generator().manual_seed(g * 100 + ph * 10 + pw))
    nh, nw = 2 * ph - 1, 2 * pw - 1
    out = torch.empty(nh * nw + 3, heads)
    _lib.check(_lib.lib().nb200_zoe_rel_pos_table(ctypes.c_void_p(tab.data_ptr()), g, heads, ph, pw, ctypes.c_void_p(out.data_ptr())))
    sub = tab[:S * S].reshape(1, S, S, heads).permute(0, 3, 1, 2)
    want = F.interpolate(sub, size=(nh, nw), mode="bilinear").permute(0, 2, 3, 1).reshape(nh * nw, heads)
    want = torch.cat([want, tab[S * S:]])
    assert float((out - want).abs().max()) < 2e-6
    if (ph, pw) == (g, g):
        assert torch.equal(out, tab)


def test_zoedepth_model_host_contract():
    """ZoeDepthModel host-side contract (iw3/zoedepth_model.py:151-233) without a GPU: supported types, checkpoint path,
    metric flag, loud errors for the checkpoints the engine does not implement, checkpoint dict unwrapping."""
    import torch
    from nunif_b200.iw3 import ZoeDepthModel
    from nunif_b200.iw3 import zoedepth_model as zm
    assert ZoeDepthModel.supported("ZoeD_N") and not ZoeDepthModel.supported("ZoeD_K") and not ZoeDepthModel.supported("ZoeD_Any_N")
    assert ZoeDepthModel.get_name() == "ZoeDepth"
    assert ZoeDepthModel.get_model_path("ZoeD_N").endswith(os.path.join("checkpoints", "ZoeD_M12_N.pt"))
    m = ZoeDepthModel("ZoeD_N")
    assert m.is_metric() and not m.loaded()
    for bad in ("ZoeD_K", "ZoeD_NK", "ZoeD_Any_K", "Any_V2_S"):
        with pytest.raises(ValueError):
            ZoeDepthModel(bad)
    with pytest.raises(FileNotFoundError):
        m.load_model("ZoeD_N", device=torch.device("cuda", 0))        # no checkpoint on disk, never downloads
    sd = {"a": torch.zeros(1)}
    assert zm._strip_checkpoint({"model": sd, "epoch": 3}) is sd and zm._strip_checkpoint(sd) is sd
    with pytest.raises(RuntimeError):
        zm.ZoeDepthNet(sd, "cpu")                                      # no CPU path


def test_iw3_workloads_are_declared_for_both_bench_arms():
    import bench
    for key, wl in bench.IW3_WORKLOADS.items():
        assert wl["frame"] in bench.FRAME and wl["batch"] > 0 and wl["depth"] in ("Any_V2_S", "ZoeD_N")
        assert wl["method"] in ("forward_fill", "backward")
    assert "iw3_4k_zoe" in bench.IW3_WORKLOADS and "swin4x_4k" in bench.WORKLOADS


def test_create_model_refuses_unbuilt_variants_loudly():
    """Constructor arguments that change the arithmetic are never ignored (VERDICT r1: no silent no-ops); all of these raise
    before any CUDA call."""
    import torch
    from nunif_b200.nunif.models import create_model
    sd = {"x": torch.zeros(1)}
    for name in ("waifu2x.swin_unet_8x", "waifu2x.swin_unet_4xl"):
        with pytest.raises(NotImplementedError):
            create_model(name, sd, "cuda:0")
    with pytest.raises(NotImplementedError, match="pre_antialias"):
        create_model("waifu2x.swin_unet_4x", sd, "cuda:0", pre_antialias=True)
    with pytest.raises(NotImplementedError):
        create_model("waifu2x.swin_unet_4x", sd, "cuda:0", base_dim=192, layer_norm=True)
    with pytest.raises(NotImplementedError):
        create_model("waifu2x.upcunet", sd, "cuda:0", in_channels=1)
    with pytest.raises(AssertionError):
        create_model("waifu2x.swin_unet_downscaled", sd, "cuda:0", downscale_factor=3)
    with pytest.raises(ValueError, match="Unknown model name"):
        create_model("waifu2x.no_such_model", sd, "cuda:0")
    with pytest.raises(RuntimeError, match="no CPU path"):
        create_model("waifu2x.swin_unet_downscaled", sd, "cpu", downscale_factor=2)      # name accepted; the engine needs CUDA
