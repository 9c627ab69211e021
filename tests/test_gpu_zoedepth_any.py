"""GPU parity of ZoeD_Any_N / ZoeD_Any_K (Depth-Anything V1 encoder + DPT head + ZoeDepth bins head) and of the Depth-Anything
V1 models Any_S/B/L against the oracle's restatement (oracle/zoedepth_any.py, oracle/depth_anything.py).

Criterion as for ZoeD_N (tests/test_gpu_zoedepth.py): the engine computes in the reference's CUDA numerics (fp16 autocast), so
its error against the fp32 oracle is compared with the error of the oracle itself run under CUDA fp16 autocast."""
import argparse
import ctypes
import pytest
import torch

from tests.util import load_golden, log_metric, stats, t, true_fp32
from tests.test_gpu_zoedepth import _check
from nunif_b200 import synth, _lib
from oracle import zoedepth_any as oza
from oracle import depth_anything as oda

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
KIND = {False: "ZoeD_Any_N", True: "ZoeD_Any_K"}


def _refs(sd, x, cfg, normed, return_all=False):
    sdc = {k: v.to(DEV) for k, v in sd.items()}
    with torch.no_grad():
        with true_fp32():
            ref32 = oza.zoedepth_any_forward(sdc, x.to(DEV).float(), cfg, normed, return_all)
        with torch.autocast("cuda", dtype=torch.float16):
            refamp = oza.zoedepth_any_forward(sdc, x.to(DEV), cfg, normed, return_all)
    if return_all:
        return ref32, refamp
    return ref32.cpu(), refamp.float().cpu()


def _net(sd, normed):
    from nunif_b200.iw3 import ZoeDepthAnythingNet
    return ZoeDepthAnythingNet(sd, DEV, KIND[normed])


@pytest.mark.parametrize("normed", [False, True])
@pytest.mark.parametrize("B,H,W", [(1, 98, 126), (2, 98, 126), (1, 112, 140), (2, 112, 140)])
def test_zoedepth_any_forward_mini(normed, B, H, W):
    """Reduced widths (synth.ZOED_ANY_MINI), same code path; 7 x 9 (odd) and 8 x 10 token grids."""
    sd = synth.zoedepth_any_state_dict(1, synth.ZOED_ANY_MINI, normed)
    x = torch.randn(B, 3, H, W, generator=torch.Generator().manual_seed(H + W + B))
    got = _net(sd, normed)(x.to(DEV)).cpu()
    ref32, refamp = _refs(sd, x, oza.ZOED_ANY_MINI, normed)
    assert got.shape == ref32.shape == (B, 1, H, W)
    assert float(ref32.std()) > 0.05
    _check(f"zoedepth_any_{KIND[normed]}_{B}x{H}x{W}", got, ref32, refamp)


def _tapped(net, tap_id, x, nbytes):
    lib = _lib.lib()
    buf = torch.zeros(nbytes // 4, dtype=torch.float32, device=DEV)
    _lib.check(lib.nb200_debug_tap(tap_id, _lib.ptr(buf), nbytes))
    try:
        out = net(x)
    finally:
        lib.nb200_debug_tap(-1, None, 0)
    torch.cuda.synchronize()
    return out, buf


def test_zoedepth_any_k_sorted_centres_tap():
    """Tap 15: the last level's centres after the per-pixel sort and the clip, against the oracle within the autocast error;
    non-decreasing along the bins and inside [1e-3, 80].  Tap 14 (b_new of the last level, [0, 1] units) sorts into tap 15."""
    sd = synth.zoedepth_any_state_dict(1, synth.ZOED_ANY_MINI, True)
    x = torch.randn(2, 3, 98, 126, generator=torch.Generator().manual_seed(7))
    net = _net(sd, True)
    hp, wp = 8 * 7, 8 * 9
    n = 2 * hp * wp * 64 * 4
    _, c = _tapped(net, 15, x.to(DEV), n)
    _, b = _tapped(net, 14, x.to(DEV), n)
    c = c.view(2, hp, wp, 64).permute(0, 3, 1, 2).cpu()
    b = b.view(2, hp, wp, 64).permute(0, 3, 1, 2).cpu()
    r32, ramp = _refs(sd, x, oza.ZOED_ANY_MINI, True, return_all=True)
    want32, wantamp = r32["centers"].cpu(), ramp["centers"].float().cpu()
    e_our, e_ref = stats(c, want32), stats(wantamp, want32)
    log_metric("zoedepth_any_k_centres", ours_max=e_our["max"], ours_mean=e_our["mean"], refamp_max=e_ref["max"], refamp_mean=e_ref["mean"])
    assert e_our["mean"] <= 1.25 * e_ref["mean"] + 1e-6 and e_our["max"] <= 4.0 * e_ref["max"] + 1e-4, (e_our, e_ref)
    assert float(c.diff(dim=1).min()) >= 0.0
    assert float(c.min()) >= 1e-3 and float(c.max()) <= 80.0
    want = torch.sort((80.0 - 1e-3) * b + 1e-3, dim=1)[0].clip(1e-3, 80.0)
    assert float((c - want).abs().max()) <= 1e-5 * 80.0


@pytest.mark.parametrize("normed,H,W", [(False, 392, 700), (True, 518, 518)])
def test_zoedepth_any_full_size(normed, H, W):
    """The released configuration (ViT-L/14, 24 blocks, 1024 wide): N at the 1080p network input, K at the portrait one."""
    sd = synth.zoedepth_any_state_dict(0, None, normed)
    x = torch.randn(1, 3, H, W, generator=torch.Generator().manual_seed(11)).clamp_(-1, 1)
    got = _net(sd, normed)(x.to(DEV)).cpu()
    ref32, refamp = _refs(sd, x, oza.ZOED_ANY, normed)
    assert got.shape == (1, 1, H, W)
    _check(f"zoedepth_any_full_{KIND[normed]}_{H}x{W}", got, ref32, refamp)


def test_zoedepth_any_batch_invariant_and_grid_change():
    sd = synth.zoedepth_any_state_dict(2, synth.ZOED_ANY_MINI, True)
    net = _net(sd, True)
    x = torch.randn(3, 3, 98, 126, generator=torch.Generator().manual_seed(3)).to(DEV)
    y3 = net(x)
    y1 = net(x[1:2])
    assert torch.equal(y3[1:2], y1)
    z = net(torch.randn(1, 3, 112, 140, generator=torch.Generator().manual_seed(4)).to(DEV))   # position table rebuilt
    assert torch.isfinite(z).all()
    assert torch.equal(net(x[1:2]), y1)                                                         # ... and rebuilt back


def test_zoedepth_any_rejects_bad_input_and_keys():
    from nunif_b200.iw3 import ZoeDepthAnythingNet
    sd_n = synth.zoedepth_any_state_dict(1, synth.ZOED_ANY_MINI, False)
    sd_k = synth.zoedepth_any_state_dict(1, synth.ZOED_ANY_MINI, True)
    net = _net(sd_n, False)
    with pytest.raises(RuntimeError, match="multiples of 14"):
        net(torch.zeros(1, 3, 98, 128, device=DEV))
    bad = dict(sd_n)
    bad.pop("core.core.depth_head.scratch.layer4_rn.weight")
    with pytest.raises(RuntimeError, match="missing key"):
        _net(bad, False)
    bad = dict(sd_k)
    bad["core.core.extra.weight"] = torch.zeros(3)
    with pytest.raises(RuntimeError, match="unexpected key"):
        _net(bad, True)
    with pytest.raises(RuntimeError, match="attractors.0._net.2 has 16 outputs"):
        ZoeDepthAnythingNet(sd_n, DEV, "ZoeD_Any_K")
    with pytest.raises(RuntimeError, match="attractors.0._net.2 has 32 outputs"):
        ZoeDepthAnythingNet(sd_k, DEV, "ZoeD_Any_N")
    from nunif_b200.iw3 import ZoeDepthNet
    with pytest.raises(RuntimeError, match="missing key"):
        ZoeDepthNet(sd_n, DEV)                                  # a ZoeD_Any checkpoint is not a ZoeD_N one


@pytest.mark.parametrize("normed", [False, True])
def test_zoedepth_any_infer_pipeline_1080p(normed):
    """ZoeDepthAnythingModel.infer on 1080p frames: batch_preprocess with prep_mod 14 (392 x 700, pads 22 / 31) -> network ->
    crop -> negate (+ flip TTA, + dilate_edge), against the oracle; then process_image's call sequence."""
    from nunif_b200.iw3 import create_depth_model, dilate_edge
    from nunif_b200.iw3.zoedepth_preprocess import batch_preprocess
    sd = synth.zoedepth_any_state_dict(2, synth.ZOED_ANY_MINI, normed)
    model = create_depth_model(KIND[normed]).load_state_dict(sd, gpu=0)
    assert model.is_metric() and model.get_name() == "ZoeDepth" and model.loaded()
    assert (model.model.prep_mod, model.model.prep_h_height, model.model.prep_v_height) == (14, 392, 518)
    x = torch.stack([synth.synth_image(90 + i, 3, 1080, 1920, smooth=False) for i in range(2)])
    with torch.inference_mode():
        d = model.infer(x.to(DEV), tta=False, edge_dilation=0)
        xp, pad_h, pad_w = batch_preprocess(x.to(DEV), h_height=392, v_height=518, ensure_multiple_of=14)
        assert xp.shape[-2:] == (392, 700) and (pad_h, pad_w) == (22, 31)
        assert d.shape == (2, 1, 392 - 44, 700 - 62) and d.is_cuda and d.dtype == torch.float32
        ref32, refamp = _refs(sd, xp.cpu(), oza.ZOED_ANY_MINI, normed)
        crop = (slice(None), slice(None), slice(22, 392 - 22), slice(31, 700 - 31))
        _check(f"zoedepth_any_1080p_infer_{KIND[normed]}", -d.cpu(), ref32[crop], refamp[crop])
        dt = model.infer(x[0].to(DEV), tta=True, edge_dilation=0)
        assert dt.shape == (1, 392 - 44, 700 - 62)
        xf = torch.cat([xp[:1], torch.flip(xp[:1], dims=[3])], dim=0)
        r32, ramp = _refs(sd, xf.cpu(), oza.ZOED_ANY_MINI, normed)
        want32 = (r32[:1][crop] + torch.flip(r32[1:][crop], dims=[3])) * 0.5
        wantamp = (ramp[:1][crop] + torch.flip(ramp[1:][crop], dims=[3])) * 0.5
        _check(f"zoedepth_any_1080p_tta_{KIND[normed]}", -dt.cpu().unsqueeze(0), want32, wantamp)
        dd = model.infer(x.to(DEV), tta=False, edge_dilation=2)
        assert torch.allclose(dd, dilate_edge(d.clone(), 2), atol=1e-5)
        assert model.get_ema_buffer_size() >= 1
        dn = model.minmax_normalize_chw(model.infer(x[0].to(DEV), tta=False, edge_dilation=2))
        assert dn.shape == d.shape[1:] and float(dn.min()) >= 0.0 and float(dn.max()) <= 1.0


def test_zoedepth_any_infer_matches_reference_batch_infer_golden():
    """ZoeDepthAnythingModel.infer against the REAL iw3/zoedepth_model.batch_infer with prep_mod 14 run on the CPU in fp32 around
    the oracle network (tests/golden/zoedepth_any_infer.npz): N and K, landscape batch and portrait image, flip TTA, dilation.
    Bounds as for ZoeD_N's golden test."""
    from nunif_b200.iw3 import ZoeDepthAnythingModel
    g = load_golden("zoedepth_any_infer")
    from tests.test_zoedepth_any import golden_inputs
    land, port = (v.to(DEV) for v in golden_inputs(g))
    for normed, tag in ((False, "n"), (True, "k")):
        sd = synth.zoedepth_any_state_dict(5, synth.ZOED_ANY_MINI, normed)
        model = ZoeDepthAnythingModel(KIND[normed]).load_state_dict(sd, gpu=0)
        model.model.prep_h_height, model.model.prep_v_height = 56, 70        # the sizes the golden was generated with
        with torch.inference_mode():
            for flip in (0, 1):
                for dil in (0, 2):
                    for name, x in (("land", land), ("port", port)):
                        want = t(g[f"{tag}_{name}_f{flip}_d{dil}"])
                        got = model.infer(x, tta=bool(flip), edge_dilation=dil).cpu()
                        assert got.shape == want.shape, (tag, name, flip, dil, got.shape, want.shape)
                        scale = float(want.abs().max())
                        e = stats(got, want)
                        log_metric(f"zoedepth_any_infer_golden_{tag}_{name}_f{flip}_d{dil}", max=e["max"], mean=e["mean"], p999=e["p999"], scale=scale)
                        assert torch.isfinite(got).all()
                        assert e["mean"] <= 1e-3 * scale and e["p999"] <= 1e-2 * scale and e["max"] <= 0.1 * scale, (tag, name, flip, dil, e, scale)


@pytest.mark.parametrize("model_type,encoder,H,W", [("Any_S", "vits", 14 * 6, 14 * 9), ("Any_B", "vitb", 14 * 7, 14 * 6),
                                                    ("Any_L", "vitl", 14 * 5, 14 * 7)])
def test_depth_anything_v1(model_type, encoder, H, W):
    """Any_S/B/L: the V2 networks with the hooks on the last four blocks, through DepthAnythingModel; depth_aa=True runs
    without AA as in the reference (AA_SUPPORTED_MODELS holds V2 only)."""
    from nunif_b200.iw3 import DepthAnythingModel
    from tests.test_gpu_depth import _check as da_check
    sd = synth.depth_anything_v2_state_dict(6, encoder=encoder, pos_grid=8)
    model = DepthAnythingModel(model_type).load_state_dict(sd, gpu=0)
    x = torch.randn(1, 3, H, W, generator=torch.Generator().manual_seed(H * W))
    got = model.model(x.to(DEV)).cpu()
    sdc = {k: v.to(DEV) for k, v in sd.items()}
    with torch.no_grad():
        with true_fp32():
            ref32 = oda.depth_anything_forward(sdc, x.to(DEV).float(), oza.V1[encoder]).cpu()
        with torch.autocast("cuda", dtype=torch.float16):
            refamp = oda.depth_anything_forward(sdc, x.to(DEV), oza.V1[encoder]).float().cpu()
        v2 = oda.depth_anything_forward(sdc, x.to(DEV).float(), encoder).cpu()
    da_check(f"depth_anything_v1_{encoder}", got, ref32, refamp)
    assert float((v2 - ref32).abs().max()) > 1e-2 * float(ref32.abs().max())
    im = synth.synth_image(3, 3, 120, 200).to(DEV)
    with torch.inference_mode():
        assert torch.equal(model.infer(im, depth_aa=True), model.infer(im, depth_aa=False))


def test_apply_divergence_from_create_depth_model_zoed_any_n():
    """iw3's default path: create_depth_model("ZoeD_Any_N") -> infer (dilate_edge 2) -> minmax_normalize_chw -> apply_divergence
    (forward_fill, div_6) -> SBS, against the oracle warp on the engine's own depth; process_image gives the same frame."""
    from nunif_b200.iw3 import create_depth_model, apply_divergence, process_image
    from oracle import iw3 as oiw
    dm = create_depth_model("ZoeD_Any_N").load_state_dict(synth.zoedepth_any_state_dict(3, synth.ZOED_ANY_MINI, False), gpu=0)
    dm.disable_ema()
    x = synth.synth_image(5, 3, 126, 224).to(DEV)
    args = argparse.Namespace(method="forward_fill", mapper="div_6", convergence=0.5, divergence=2.0, synthetic_view="both",
                              tta=False, low_vram=False, disable_amp=False, edge_dilation=2, depth_aa=False,
                              state={"convergence_model": None}, anaglyph=None, half_sbs=False, warp_steps=None,
                              preserve_screen_border=False, stereo_width=None)
    sbs = process_image(x, args, dm, None)
    assert sbs.shape == (3, 126, 448)
    with torch.inference_mode():
        depth = dm.infer(x, tta=False, edge_dilation=2)
        nd = dm.minmax_normalize_chw(depth)
    dn = depth.cpu()
    want_nd = (dn - dn.min()) / (dn.max() - dn.min())
    assert float((nd.cpu() - want_nd).abs().max()) < 1e-6
    le, re = apply_divergence(nd, x, args, None)
    mapped = oiw.mapper(want_nd.unsqueeze(0), "div_6")
    lo, ro = oiw.forward_warp(x.cpu().unsqueeze(0), mapped, 2.0, 0.5, fill=True, width_base=False)
    frac = max(float(((le.cpu() - lo[0]).abs() > 1e-3).float().mean()), float(((re.cpu() - ro[0]).abs() > 1e-3).float().mean()))
    log_metric("zoedepth_any_apply_divergence", frac_gt_1e3=frac)
    assert frac < 2e-3, frac
    assert torch.equal(sbs, torch.cat([le, re], dim=2).clamp(0, 1))
