"""GPU: every disparity mapper of iw3/mapper.py on the engine (csrc/mapper.cuh) against tests/golden/mapper.npz (generated
by the real reference), the fused per-frame min/max + mapper pass, the float mapper_c entries, apply_divergence with
--foreground-scale names on a relative and a metric model and with auto-convergence, and --stereo-width.

Bounds: 2e-6 for a mapper against the reference.  The reference's own fp32 error against float64 is at most 5.2e-7
(div_25), so two fp32 evaluations of the same op sequence agree well inside it."""
import argparse
import ctypes

import pytest
import torch
import torch.nn.functional as F

from tests.util import load_golden, t, stats, log_metric
from nunif_b200 import synth, _lib

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
TOL = 2e-6
DIV = {"none": -1.0, "div_25": 2.5, "div_10": 1.0, "div_6": 0.6, "div_4": 0.4, "div_2": 0.2, "div_1": 0.1}


@pytest.fixture(scope="module")
def g():
    return load_golden("mapper")


def _err(got, want):
    return float((got.double().cpu() - t(want).double()).abs().max())


def test_every_name_ladder_and_chain_matches_reference(g):
    from nunif_b200.iw3 import get_mapper, depth_mapper
    pts, conv = t(g["pts"], DEV), t(g["conv"], DEV)
    worst = {}
    for n in map(str, g["names"]):
        f = get_mapper(n)
        worst[n] = max(_err(f(pts), g["pts/" + n]), _err(f(conv), g["conv/" + n]), _err(depth_mapper(pts, n), g["pts/" + n]))
    for c in map(str, g["cases"]):
        worst[c] = max(_err(get_mapper(c)(pts), g["pts/" + c]), _err(depth_mapper(pts, c), g["pts/" + c]))
    lpts = pts[::16].contiguous()
    for i, n in enumerate(map(str, g["ladder_names"])):
        worst[n] = _err(get_mapper(n)(lpts), g["ladder"][i])
    top = max(worst, key=worst.get)
    log_metric("mapper_vs_reference", names=len(worst), worst_name=top, worst=worst[top],
               late_bound=worst["mul_1+mul_2=0.5:div_6+div_1=0.25"])
    bad = {k: v for k, v in worst.items() if v > TOL}
    assert not bad, bad


def test_fused_minmax_mapper_is_minmax_then_mapper(g):
    from nunif_b200.iw3 import minmax_normalize, depth_mapper
    raw = t(g["raw"], DEV)
    plain = minmax_normalize(raw, "none")
    worst = 0.0
    for n in list(map(str, g["names"])) + list(map(str, g["cases"])):
        fused = minmax_normalize(raw, mapper=n)
        assert torch.equal(fused, depth_mapper(plain, n)), n
        if "mm/" + n in g:
            worst = max(worst, _err(fused, g["mm/" + n]))
    log_metric("mapper_fused_minmax", worst=worst)
    assert worst <= TOL, worst


def test_none_and_div_bit_identical_through_old_and_new_entries():
    from nunif_b200.iw3.mapper import descriptor
    x = synth.synth_depth(11, 2, 50, 70).to(DEV) * 3 - 1
    x01 = synth.synth_depth(12, 2, 50, 70).to(DEV)
    B, n = x.shape[0], x[0].numel()
    L, st = _lib.lib(), _lib.stream_ptr()
    for name, c in DIV.items():
        d = ctypes.byref(descriptor(name))
        old, new = torch.empty_like(x), torch.empty_like(x)
        mm_old, mm_new = torch.empty(B, 2, device=DEV), torch.empty(B, 2, device=DEV)
        _lib.check(L.nb200_minmax_map(_lib.ptr(x), B, n, c, _lib.ptr(old), _lib.ptr(mm_old), st))
        _lib.check(L.nb200_minmax_mapper(_lib.ptr(x), B, n, d, _lib.ptr(new), _lib.ptr(mm_new), st))
        assert torch.equal(old, new) and torch.equal(mm_old, mm_new), name
        new = torch.empty_like(x01)
        _lib.check(L.nb200_mapper_apply(_lib.ptr(x01), x01.numel(), d, _lib.ptr(new), st))
        if c < 0:
            assert torch.equal(new, x01)
        else:
            old = torch.empty_like(x01)
            _lib.check(L.nb200_depth_mapper(_lib.ptr(x01), x01.numel(), c, _lib.ptr(old), st))
            assert torch.equal(old, new), name


def test_bad_descriptor_is_refused():
    m = _lib.Mapper()
    m.n_stages = 9
    x = torch.rand(16, device=DEV)
    assert _lib.lib().nb200_mapper_apply(_lib.ptr(x), 16, ctypes.byref(m), _lib.ptr(x), _lib.stream_ptr()) != 0
    m.n_stages, m.stage[0].a.kind = 1, 99
    assert _lib.lib().nb200_mapper_apply(_lib.ptr(x), 16, ctypes.byref(m), _lib.ptr(x), _lib.stream_ptr()) != 0
    assert b"unknown mapper function kind" in _lib.lib().nb200_last_error()


def _args(mapper, **kw):
    a = dict(method="backward", mapper=mapper, convergence=0.5, divergence=2.0, synthetic_view="both", tta=False, low_vram=False,
             disable_amp=False, edge_dilation=2, depth_aa=False, state={"convergence_model": None}, warp_steps=None,
             preserve_screen_border=False, stereo_width=None)
    a.update(kw)
    return argparse.Namespace(**a)


def _divergence_against_oracle(dm, x, mapper, tag):
    from nunif_b200.iw3 import apply_divergence
    from oracle import iw3 as oiw
    from oracle.mapper import mapper as omapper
    with torch.inference_mode():
        depth = dm.infer(x, tta=False, edge_dilation=2)
        nd = dm.minmax_normalize_chw(depth)
    dn = depth.cpu()
    want_nd = (dn - dn.min()) / (dn.max() - dn.min())
    le, re = apply_divergence(nd, x, _args(mapper), None)
    mapped = omapper(want_nd.unsqueeze(0), mapper)
    lo, ro = oiw.apply_divergence_grid_sample(x.cpu().unsqueeze(0).double(), mapped.double(), 2.0, 0.5)
    frac = max(stats(le, lo[0])["frac_gt_1e3"], stats(re, ro[0])["frac_gt_1e3"])
    log_metric("mapper_apply_divergence", tag=tag, mapper=mapper, frac_gt_1e3=frac)
    assert frac < 2e-3, (mapper, frac)


def test_apply_divergence_relative_model_foreground_scale():
    from nunif_b200.iw3 import DepthAnythingModel, resolve_mapper_name
    dm = DepthAnythingModel("Any_V2_S")
    dm.load_state_dict(synth.depth_anything_v2_state_dict(0, pos_grid=6), gpu=0, resolution=140)
    dm.disable_ema()
    x = synth.synth_image(5, 3, 96, 160).to(DEV)
    for mtype, want in ((None, "mul_1+mul_2=0.5"), ("shift", "shift_14+shift_20=0.5")):
        name = resolve_mapper_name(None, 1.5, False, mtype)
        assert name == want
        _divergence_against_oracle(dm, x, name, "Any_V2_S")


def test_apply_divergence_metric_model_foreground_scale():
    from nunif_b200.iw3 import ZoeDepthModel, resolve_mapper_name
    dm = ZoeDepthModel("ZoeD_N").load_state_dict(synth.zoedepth_state_dict(2, synth.ZOED_MINI), gpu=0)
    dm.disable_ema()
    name = resolve_mapper_name(None, -0.5, True)
    assert name == "div_6+div_10=0.5"
    _divergence_against_oracle(dm, synth.synth_image(6, 3, 126, 224).to(DEV), name, "ZoeD_N")


def test_auto_convergence_is_mapped(monkeypatch):
    from nunif_b200.iw3 import ConvergenceEstimator, apply_divergence, get_mapper, depth_mapper
    import nunif_b200.iw3.utils as u
    est = ConvergenceEstimator(0.3, 0, state_dict=synth.sod_v1_state_dict(0))
    c = torch.stack([synth.synth_image(50 + i, 3, 54, 96) for i in range(3)]).to(DEV)
    d = synth.synth_depth(53, 3, 24, 42).to(DEV)
    seen = {}

    def warp(im, depth, divergence, convergence, synthetic_view):
        seen["depth"], seen["convergence"] = depth, convergence
        return im, im

    monkeypatch.setattr(u, "apply_divergence_grid_sample", warp)
    apply_divergence(d, c, _args("mul_2", state={"convergence_model": est}), None)
    want = get_mapper("mul_2")(est(c, d))
    assert seen["convergence"].shape == (3, 1, 1, 1) and torch.equal(seen["convergence"], want)
    assert torch.equal(seen["depth"], depth_mapper(d, "mul_2"))


def test_stereo_width_resize_matches_aten(monkeypatch):
    from nunif_b200.iw3 import apply_divergence
    from nunif_b200.iw3.utils import resize_depth_aa
    import nunif_b200.iw3.utils as u
    im = synth.synth_image(7, 3, 180, 320).unsqueeze(0).to(DEV)
    d = synth.synth_depth(8, 1, 96, 172).to(DEV)
    seen = {}
    monkeypatch.setattr(u, "apply_divergence_nn_LR", lambda m, c, depth, *a, **k: (seen.__setitem__("depth", depth), (c, c))[1])
    worst = {}
    for sw in (103, 258, 400):                       # 0.6x and 1.5x the depth width; 400 > W clamps to W = 320
        apply_divergence(d, im, _args("none", method="row_flow_v3", stereo_width=sw), object())
        w = min(320, sw)
        h = int(180 * (w / 320))
        got = seen["depth"]
        assert got.shape == (1, 1, h, w), (sw, got.shape)
        assert torch.equal(got, resize_depth_aa(d, h, w).clamp(0, 1))
        for where in ("cuda", "cpu"):
            want = F.interpolate(d.to(where), size=(h, w), mode="bilinear", align_corners=True, antialias=True).clamp(0, 1)
            worst[f"{where}_w{sw}"] = float((got.to(where) - want).abs().max())
    log_metric("stereo_width_resize_vs_aten", **worst)
    # nb200_depth_resize_aa follows ATen's CPU antialias kernel (bit-exact at these sizes, measured on an H100); ATen's
    # CUDA kernel rounds differently: up to 1.4e-6 from it here.  2e-6 is test_gpu_iw3's bound for this kernel.
    assert max(worst.values()) <= 2e-6, worst
    apply_divergence(d, im, _args("none", method="row_flow_v3", stereo_width=172), object())
    assert seen["depth"] is d


@pytest.mark.parametrize("method", ["row_flow_v3", "mlbw_l2"])
def test_stereo_width_eyes(method):
    from nunif_b200.iw3 import apply_divergence, apply_divergence_nn_LR, RowFlowV3, MLBW
    from nunif_b200.iw3.utils import resize_depth_aa
    model = RowFlowV3(synth.row_flow_v3_state_dict(3), DEV) if method == "row_flow_v3" else MLBW(synth.mlbw_state_dict(0), DEV)
    im = synth.synth_image(9, 3, 180, 320).unsqueeze(0).to(DEV)
    d = synth.synth_depth(10, 1, 96, 172).to(DEV)
    for sw in (103, 258, 172):
        le, re = apply_divergence(d, im, _args("none", method=method, stereo_width=sw), model)
        w = min(320, sw)
        rd = d if w == d.shape[3] else resize_depth_aa(d, int(180 * (w / 320)), w).clamp(0, 1)
        lo, ro = apply_divergence_nn_LR(model, im, rd, 2.0, 0.5, None, synthetic_view="both", preserve_screen_border=False,
                                        enable_amp=True)
        assert torch.equal(le, lo) and torch.equal(re, ro), (method, sw)
