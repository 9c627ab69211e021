"""GPU: iw3's NULL depth model on the engine (nb200_null_depth, NullDepthModel) against tests/golden/null_depth.npz (the
real reference on the CPU), against ATen's own composition F.interpolate(...).mean(1, keepdim=True) on the same GPU, and
inside the image and video paths it exists to benchmark."""
import argparse

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from oracle import null_depth as ond
from tests.util import load_golden, log_metric, t

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
G = load_golden("null_depth")


def ulp(a, b):
    """Per-element distance in fp32 units in the last place (both tensors finite and of one sign)."""
    a, b = a.detach().float().contiguous(), b.detach().float().contiguous()
    return (a.view(torch.int32).long() - b.to(a.device).view(torch.int32).long()).abs()


# The reference's CPU resize forms each lerp in another order than ATen's CUDA kernel (products without FMA, and a scalar path
# when single-threaded), so on inputs in [0, 1] the CPU and GPU results differ by up to about one rounding per channel at the
# scale of 1.  The bound against the CPU golden is therefore absolute: 4 * 2^-24.  (Against ATen's composition on the same GPU
# the kernel is compared in ulps below.)  Measured on an H100 80GB HBM3 at 700 W: at most 3 * 2^-24, up to 3 ulp on small
# values; the already-R x R case, where both copy, within 1 ulp (the CPU divides the sum by 3, the GPU multiplies by 1/3).
GOLDEN_ABS = 4 * 2.0 ** -24


@pytest.mark.parametrize("spec", ond.CASES, ids=[c[0] for c in ond.CASES])
def test_matches_reference_golden(spec):
    """The kernel against the reference's CPU result at every golden crop, tta on and off; with edge_dilation=2, the engine's
    dilate_edge within its own golden tolerance (tests/test_gpu_iw3.py test_dilate_edge_minmax_mapper)."""
    from nunif_b200.iw3 import NullDepthModel
    name, B, H, W, res = spec
    x = ond.frames(spec).to(DEV)
    m = NullDepthModel("NULL").load(gpu=0, resolution=res)
    bad = []
    for tta, dil in ond.VARIANTS:
        key = f"{name}/t{tta}_d{dil}"
        y = m.infer(x, tta=bool(tta), edge_dilation=dil)
        assert tuple(y.shape) == tuple(G[f"{key}/shape"]), key
        got = torch.cat([c.flatten() for c in ond.crops(y)])
        want = torch.cat([t(G[f"{key}/crop{i}"], DEV).flatten() for i in range(4)])
        err = float((got.double() - want.double()).abs().max())
        d = ulp(got, want)
        log_metric("null_depth_golden", case=key, max_abs=err, max_ulp=int(d.max()), n_diff=int((d > 0).sum()), n=d.numel())
        if err > (GOLDEN_ABS if dil == 0 else 1e-4):
            bad.append((key, err))
    assert not bad, bad


# (B, H, W, R): 1080p, 4K, portrait, an upscale, R = 1, and an R x R frame (ATen copies it)
ATEN_CASES = [(4, 1080, 1920, 392), (2, 2160, 3840, 518), (3, 1920, 1080, 392), (1, 200, 300, 518), (4, 1080, 1920, 1),
              (2, 720, 1280, 518), (1, 392, 392, 392)]


@pytest.mark.parametrize("B,H,W,R", ATEN_CASES)
def test_matches_aten_on_the_same_gpu(B, H, W, R):
    from nunif_b200.iw3 import NullDepthNet
    x = torch.rand((B, 3, H, W), generator=torch.Generator().manual_seed(B * 7 + R)).to(DEV)
    got = NullDepthNet(R)(x)
    want = F.interpolate(x, size=(R, R), mode="bilinear").mean(dim=1, keepdim=True)
    assert got.shape == want.shape == (B, 1, R, R) and got.dtype == torch.float32
    d = ulp(got, want)
    log_metric("null_depth_aten", B=B, H=H, W=W, R=R, max_ulp=int(d.max()), n_diff=int((d > 0).sum()), n=d.numel())
    assert int(d.max()) <= 1, int(d.max())        # measured: 0 ulp, except R = 1 (2 of 4 pixels 1 ulp apart)


def test_infer_contract():
    from nunif_b200.iw3 import NullDepthModel, dilate_edge
    m = NullDepthModel("NULL").load(gpu=0, resolution=200)
    x = torch.rand((2, 3, 150, 260), generator=torch.Generator().manual_seed(3)).to(DEV)
    y = m.infer(x)
    assert y.shape == (2, 1, 200, 200) and y.device == x.device and y.dtype == torch.float32
    y3 = m.infer(x[1])
    assert y3.shape == (1, 200, 200) and torch.equal(y3, y[1])
    assert torch.equal(m.infer(x, tta=True), y)
    assert torch.equal(m.infer(x, edge_dilation=2), dilate_edge(y, 2))
    assert torch.equal(m.infer(x[0], edge_dilation=2), dilate_edge(y[:1], 2)[0])
    assert torch.equal(m.infer(x, enable_amp=False, low_vram=True), y)
    assert torch.equal(m.infer(x[:, :, 10:110, 20:220]), NullDepthModel("NULL").load(0, 200).infer(x[:, :, 10:110, 20:220].contiguous()))
    with pytest.raises(TypeError):
        m.infer(x.half())
    with pytest.raises(ValueError):
        m.infer(x[:, :2])


def _image_args(**kw):
    base = dict(method="forward_fill", mapper="div_6", convergence=0.5, divergence=2.0, synthetic_view="both", tta=False,
                low_vram=False, disable_amp=False, edge_dilation=2, depth_aa=False, state={"convergence_model": None},
                anaglyph=None, half_sbs=False, warp_steps=None, preserve_screen_border=False, stereo_width=None)
    base.update(kw)
    return argparse.Namespace(**base)


def test_process_image_forward_fill_sbs():
    """process_image with the NULL model, forward_fill SBS, checked as tests/test_gpu_depth_api.py checks it with a depth
    network: the engine's depth, normalised, warped by the oracle."""
    from nunif_b200 import synth
    from nunif_b200.iw3 import NullDepthModel, apply_divergence, process_image
    from oracle import iw3 as oiw
    dm = NullDepthModel("NULL").load(gpu=0)
    dm.disable_ema()
    x = synth.synth_image(5, 3, 96, 160).to(DEV)
    args = _image_args()
    sbs = process_image(x, args, dm, None)
    assert sbs.shape == (3, 96, 320)
    with torch.inference_mode():
        depth = dm.infer(x, edge_dilation=2)
        nd = dm.minmax_normalize_chw(depth)
    assert depth.shape == (1, 392, 392)
    dn = depth.cpu()
    want_nd = (dn - dn.min()) / (dn.max() - dn.min())
    assert float((nd.cpu() - want_nd).abs().max()) < 1e-6
    le, re = apply_divergence(nd, x, args, None)
    lo, ro = oiw.forward_warp(x.cpu().unsqueeze(0), oiw.mapper(want_nd.unsqueeze(0), "div_6"), 2.0, 0.5, fill=True, width_base=False)
    frac = max(float(((le.cpu() - lo[0]).abs() > 1e-3).float().mean()), float(((re.cpu() - ro[0]).abs() > 1e-3).float().mean()))
    log_metric("null_depth_process_image", frac_gt_1e3=frac)
    assert frac < 2e-3, frac
    assert torch.equal(sbs, torch.cat([le, re], dim=2).clamp(0, 1))


def test_batch_frame_callback_matches_reference_video():
    """bind_batch_frame_callback with the engine's NULL model on the reference's own video case (tests/golden/video_callbacks.npz,
    made with the reference's NullDepthModel): forward_fill SBS, EMA off, batch size 4.  The depths are within GOLDEN_ABS of
    the recorded ones, and the frames within the tolerance tests/test_gpu_video_callbacks.py holds the engine to."""
    from nunif_b200.iw3 import NullDepthModel, bind_batch_frame_callback, hwc_to_chw_float
    from tests import test_gpu_video_callbacks as tvc
    case = "ff_off"
    overrides, ema, use_16bit, _ = tvc.META["cases"][case]
    assert ema is None and not use_16bit and overrides == {"method": "forward_fill"}
    dm = NullDepthModel("NULL").load(gpu=0, resolution=tvc.META["res"])
    dm.disable_ema()
    clip = torch.from_numpy(tvc.G["clip/8"]).to(DEV)
    x = hwc_to_chw_float(clip)
    depth, want = dm.infer(x), torch.from_numpy(tvc.G["infer/8"]).to(DEV)
    err = float((depth.double() - want.double()).abs().max())
    d = ulp(depth, want)
    log_metric("null_depth_video_infer", max_abs=err, max_ulp=int(d.max()), n_diff=int((d > 0).sum()), n=d.numel())
    assert err <= GOLDEN_ABS, err
    args = tvc._args(**overrides, batch_size=4, state={"device": DEV, "convergence_model": None})
    cb = bind_batch_frame_callback(dm, None, tvc.SEGMENT_PTS, args)
    got = []
    for i in range(0, tvc.T, 4):
        y = cb(x[i:i + 4], [k * tvc.STEP for k in range(i, min(tvc.T, i + 4))], False)
        got += [] if y is None else list(y.cpu())
    assert cb(None, None, True) is None
    tvc._check_golden(case, got)
    assert np.isfinite(torch.stack(got).numpy()).all()
