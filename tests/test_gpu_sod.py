"""GPU parity of iw3's auto-convergence (--convergence-mode sod_v1, csrc/sod.cu): the sod_v1 saliency network against the real
reference's fp32 output (tests/golden/sod_v1.npz) within the autocast oracle's own error, the bit-exact resize, quantiles and
EMA, the per-frame convergence in the warps, and apply_divergence end to end."""
import types
import pytest
import torch
import torch.nn.functional as F

from tests.util import load_golden, t, log_metric, stats
from nunif_b200 import synth
from oracle import sod as osod, iw3 as oiw
from oracle.gen_golden_sod import NET_CASES, POS, EMA_FRAMES, EMA_RESET, E2E, E2E_ARGS, E2E_METHODS, frames

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def model():
    from nunif_b200.iw3 import SODV1
    return SODV1(synth.sod_v1_state_dict(0), DEV)


def _sd():
    return {k: v.to(DEV) for k, v in synth.sod_v1_state_dict(0).items()}


def _amp(rgb, d):
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        s, d192 = osod.sod_infer(_sd(), rgb.to(DEV), d.to(DEV))
    return s.float(), d192


@pytest.mark.parametrize("i", range(len(NET_CASES)))
def test_saliency_golden(model, i):
    """Engine error against fp32 within 2x the autocast oracle's own error (mean, p99.9, max) plus 1 fp16 ulp at 0.5."""
    g = load_golden("sod_v1")
    rgb, d = frames(*NET_CASES[i])
    ref = t(g[f"net{i}_sal"])
    sal, d192 = model.infer(rgb.to(DEV), d.to(DEV))
    amp, _ = _amp(rgb, d)
    se, sa = stats(sal, ref), stats(amp, ref)
    log_metric(f"sod_saliency_{i}", engine_max=se["max"], engine_mean=se["mean"], amp_max=sa["max"], amp_mean=sa["mean"])
    for k in ("mean", "p999", "max"):
        assert se[k] <= 2 * sa[k] + 5e-4, (k, se, sa)
    # depth_192 is ATen's CUDA bilinear resize bit for bit
    assert torch.equal(d192, F.interpolate(d.to(DEV), (192, 192), mode="bilinear", align_corners=False, antialias=False))
    # masks: equal to fp32's except where the fp32 saliency lies within the autocast error of 0.5
    band = max(sa["max"], se["max"])
    differ = (sal.cpu() > 0.5) != (ref > 0.5)
    assert bool(((ref - 0.5).abs()[differ] <= band).all()), int(differ.sum())
    # z_pos: the oracle's rule on the engine's own mask, bit for bit; the golden where the masks agree
    for k, pos in enumerate(POS):
        z = model_pos(sal, d192, pos)
        assert torch.equal(z, osod.depth_position(sal, d192, pos)), (pos, z, osod.depth_position(sal, d192, pos))
        for b in range(z.shape[0]):
            if not bool(differ[b].any()):
                assert float(z[b]) == float(g[f"net{i}_zpos"][k][b])


def model_pos(sal, d, pos):
    from nunif_b200.iw3.convergence_estimator import depth_position_from_ratio
    return depth_position_from_ratio(sal, d, pos)


@pytest.mark.parametrize("n", [0, 1, 2, 3, 7, 1000, 36864])
def test_quantiles_match_torch(n):
    g = torch.Generator().manual_seed(n)
    d = torch.rand(2, 1, 192, 192, generator=g).to(DEV)
    d[1] = torch.floor(d[1] * 8) / 8       # ties
    sal = torch.zeros(2, 1, 192, 192, device=DEV)
    idx = torch.randperm(192 * 192, generator=g)[:n].to(DEV)
    sal.view(2, -1)[:, idx] = 0.75
    for pos in (0.0, 0.3, 0.5, 0.8):
        assert torch.equal(model_pos(sal, d, pos), osod.depth_position(sal, d, pos))
    for b in range(2):
        m = d[b].flatten()[sal[b].flatten() > 0.5]
        if m.numel() and float(m.quantile(0.9) - m.quantile(0.1)) >= 1e-6:
            # the unclamped centre rule at pos 0.5 is the mean of the two quantiles
            want = ((m.quantile(0.1) + m.quantile(0.9)) / 2).clamp(0, 1)
            assert float(model_pos(sal[b:b + 1], d[b:b + 1], 0.5)) == float(want)


def test_position_constant_depth_and_empty():
    sal = torch.full((2, 1, 192, 192), 0.9, device=DEV)
    sal[1] = 0.2
    d = torch.full((2, 1, 192, 192), 0.37, device=DEV)
    z = model_pos(sal, d, 0.3).flatten()
    assert float(z[0]) == float(torch.tensor(0.37)) and float(z[1]) == 0.5


def test_ema_bitexact_and_no_host_sync():
    from nunif_b200.iw3 import ConvergenceEstimator
    g = load_golden("sod_v1")
    rgb, d = frames(*EMA_FRAMES)
    rgb, d = rgb.to(DEV), d.to(DEV)
    est = ConvergenceEstimator(0.3, 0, enable_ema=True, state_dict=synth.sod_v1_state_dict(0))
    raw = ConvergenceEstimator(0.3, 0, state_dict=synth.sod_v1_state_dict(0))
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        z = raw(rgb, d)
        a = est(rgb, d, reset_pts=EMA_RESET)
        b = est(rgb.flip(0), d.flip(0))
    finally:
        torch.cuda.set_sync_debug_mode("default")
    ema = osod.EMA(0.9)
    assert torch.equal(a, ema(z, EMA_RESET))
    assert torch.equal(b, ema(z.flip(0)))
    log_metric("sod_ema", zpos_vs_golden=float((z.cpu() - t(g["ema_raw"])).abs().max()))
    est.reset()
    assert torch.equal(est(rgb, d), osod.EMA(0.9)(z))


def test_saliency_batch_invariance(model):
    rgb, d = frames(*E2E)
    sal, _ = model.infer(rgb.to(DEV), d.to(DEV))
    for b in range(rgb.shape[0]):
        one, _ = model.infer(rgb[b:b + 1].to(DEV), d[b:b + 1].to(DEV))
        assert torch.equal(one, sal[b:b + 1])


CONV = torch.tensor([0.15, 0.5, 0.85]).reshape(3, 1, 1, 1)


def _frames3(H=54, W=96, h=24, w=42):
    c = torch.stack([synth.synth_image(50 + i, 3, H, W) for i in range(3)]).to(DEV)
    return c, synth.synth_depth(53, 3, h, w).to(DEV)


def test_per_frame_backward_warp():
    from nunif_b200.iw3 import apply_divergence_grid_sample
    c, d = _frames3()
    conv = CONV.to(DEV)
    for sv in ("both", "left", "right"):
        l, r = apply_divergence_grid_sample(c, d, 2.5, conv, sv)
        ol, orr = oiw.apply_divergence_grid_sample(c.cpu().double(), d.cpu().double(), 2.5, conv.cpu().float().double(), sv)
        assert stats(l, ol)["max"] < 1e-3 and stats(r, orr)["max"] < 1e-3, sv
        for b in range(3):
            lb, rb = apply_divergence_grid_sample(c[b:b + 1], d[b:b + 1], 2.5, conv[b:b + 1], sv)
            assert torch.equal(lb, l[b:b + 1]) and torch.equal(rb, r[b:b + 1])


def test_per_frame_forward_warp():
    from nunif_b200.iw3 import apply_divergence_forward_warp
    c, d = _frames3(48, 80, 48, 80)
    conv = CONV.to(DEV)
    for method in ("forward", "forward_fill"):
        l, r = apply_divergence_forward_warp(c, d, 3.0, conv, method=method, width_base=False)
        for b in range(3):
            lb, rb = apply_divergence_forward_warp(c[b:b + 1], d[b:b + 1], 3.0, conv[b:b + 1], method=method, width_base=False)
            assert torch.equal(lb, l[b:b + 1]) and torch.equal(rb, r[b:b + 1])
            # the tensor rounding: the scalar path with the fp32 product as its convergence term differs from it by at most
            # the last bit of shift_size * convergence
            ls, rs = apply_divergence_forward_warp(c[b:b + 1], d[b:b + 1], 3.0, float(conv[b]), method=method, width_base=False)
            assert stats(ls, lb)["frac_gt_1e3"] < 1e-2


def test_per_frame_learned_warp_input():
    from nunif_b200.iw3.row_flow import make_input
    d = synth.synth_depth(3, 3, 20, 40).to(DEV)
    conv = CONV.to(DEV)
    x = make_input(d, 2.0, conv, preserve_screen_border=True)
    for b in range(3):
        xb = make_input(d[b:b + 1], 2.0, conv[b:b + 1], preserve_screen_border=True)
        assert torch.equal(xb, x[b:b + 1])
    assert torch.equal(x[:, 2, 5, 20], osod.convergence_feature(2.0, conv, 40).flatten())


@pytest.mark.parametrize("method", E2E_METHODS)
def test_apply_divergence_with_estimator(method):
    from nunif_b200.iw3 import ConvergenceEstimator, apply_divergence, apply_divergence_grid_sample, apply_divergence_forward_warp
    g = load_golden("sod_v1")
    rgb, d = frames(*E2E)
    rgb, d = rgb.to(DEV), d.to(DEV)
    est = ConvergenceEstimator(E2E_ARGS["convergence"], 0, state_dict=synth.sod_v1_state_dict(0))
    args = types.SimpleNamespace(method=method, state={"convergence_model": est}, preserve_screen_border=False, stereo_width=None,
                                 disable_amp=False, warp_steps=None, **E2E_ARGS)
    left, right = apply_divergence(d, rgb, args, None)
    conv = est(rgb, d)
    dconv = stats(conv, t(g["e2e_conv"]))
    log_metric(f"sod_e2e_{method}", conv_diff=dconv["max"])
    if method == "backward":
        wl, wr = apply_divergence_grid_sample(rgb, d, E2E_ARGS["divergence"], conv, "both")
    else:
        wl, wr = apply_divergence_forward_warp(rgb, d, E2E_ARGS["divergence"], conv, method=method, width_base=False)
    assert torch.equal(left, wl) and torch.equal(right, wr)
    # the engine's fp16 saliency can move a pixel near 0.5 across the threshold, which moves the quantiles a little
    assert dconv["max"] < 2e-2, dconv
    # the warp driven by the reference's own convergences reproduces the reference's eyes under the scalar warp tests' bounds
    gconv = t(g["e2e_conv"], DEV)
    if method == "backward":
        gl, gr = apply_divergence_grid_sample(rgb, d, E2E_ARGS["divergence"], gconv, "both")
    else:
        gl, gr = apply_divergence_forward_warp(rgb, d, E2E_ARGS["divergence"], gconv, method=method, width_base=False)
    sl, sr = stats(gl, t(g[f"e2e_{method}_left"])), stats(gr, t(g[f"e2e_{method}_right"]))
    if method == "backward":
        assert sl["max"] < 1e-3 and sr["max"] < 1e-3, (sl, sr)
    else:
        assert sl["max"] == 0.0 and sr["max"] == 0.0, (sl, sr)   # full-resolution depth: the forward warp is exact
    if dconv["max"] == 0.0:
        assert torch.equal(left, gl) and torch.equal(right, gr)
