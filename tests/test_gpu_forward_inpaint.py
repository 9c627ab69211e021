"""GPU: iw3's forward_inpaint (image mode) on the engine against the reference's goldens (tests/golden/light_inpaint.npz) and
the oracle run under fp16 autocast (the reference's CUDA path), with the parity criterion of tests/test_gpu_models.check."""
import os
import sys
import types
import pytest
import torch

from tests.util import load_golden, t, log_metric, stats, true_fp32
from tests.test_gpu_models import check
from nunif_b200 import synth, _lib
from oracle import light_inpaint as oli

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import gen_golden_inpaint as gg  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"


@pytest.fixture(scope="module")
def g():
    return load_golden("light_inpaint")


@pytest.fixture(scope="module")
def sd():
    return synth.light_inpaint_v1_state_dict(0)


@pytest.fixture(scope="module")
def model(sd):
    from nunif_b200.iw3 import LightInpaintV1
    return LightInpaintV1(sd, DEV)


def sd_dev(sd):
    return {k: v.to(DEV) for k, v in sd.items()}


def amp_infer(sd, x, mask, mirror=False):
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        if mirror:
            return oli.infer(sd_dev(sd), x.flip(-1), mask.flip(-1)).float().flip(-1)
        return oli.infer(sd_dev(sd), x, mask).float()


def test_mask_stages_bit_exact(g):
    from nunif_b200.iw3 import mask_closing, dilate_outer, dilate_inner
    from nunif_b200.iw3.forward_inpaint import inpaint_mask
    seed, h, w, bw = (int(v) for v in g["mask_case"])
    src = oli.hole_mask(seed, 1, h, w, frac=0.05).to(DEV)
    c = mask_closing(src > 0)
    assert torch.equal(c.cpu().to(torch.uint8), t(g["mask_closing"]))
    o = dilate_outer(c, 3, bw)
    assert torch.equal(o.cpu().to(torch.uint8), t(g["mask_outer"]))
    i = dilate_inner(o, 2, bw)
    assert torch.equal(i.cpu().to(torch.uint8), t(g["mask_inner"]))
    # the fused chain, and its mirrored form (forward_left) against the oracle on the flipped mask
    assert torch.equal(inpaint_mask(src * 0.5, inner_dilation=2, outer_dilation=3, base_width=bw).cpu().to(torch.uint8),
                       t(g["mask_inner"]))
    want = oli.eye_mask(src.cpu().flip(-1), 2, 3, bw).flip(-1)
    assert torch.equal(inpaint_mask(src, inner_dilation=2, outer_dilation=3, base_width=bw, mirror=True).cpu(), want)


def test_blur(g):
    for i in range(3):
        h, w = (int(v) for v in g[f"net{i}_hw"])
        _, mask = oli.net_inputs(int(g[f"net{i}_seed"]), 1, h, w)
        m = mask.to(DEV)
        out = torch.empty_like(m)
        _lib.check(_lib.lib().nb200_inpaint_blur(_lib.ptr(m), 1, h, w, _lib.ptr(out), _lib.stream_ptr()))
        assert (out.cpu() - t(g[f"net{i}_blur"])).abs().max() <= 1e-6


@pytest.mark.parametrize("i", range(3))
def test_network_golden(g, sd, model, i):
    h, w = (int(v) for v in g[f"net{i}_hw"])
    x, mask = oli.net_inputs(int(g[f"net{i}_seed"]), 1, h, w)
    x, mask = x.to(DEV), mask.to(DEV)
    z = model.infer(x, mask)
    check(f"light_inpaint_net{i}", z, t(g[f"net{i}_z"]).to(DEV), amp_infer(sd, x, mask))


def test_network_mirror(sd, model):
    x, mask = oli.net_inputs(21, 2, 70, 150)
    x, mask = x.to(DEV), mask.to(DEV)
    z = model.infer(x, mask, mirror=True)
    with torch.no_grad(), true_fp32():
        want = oli.infer(sd_dev(sd), x.flip(-1), mask.flip(-1)).flip(-1)
    check("light_inpaint_mirror", z, want, amp_infer(sd, x, mask, mirror=True))


def test_unmasked_pixels_equal_input(model):
    """Where the blurred mask is 0 the output is the (clamped) input, bit for bit."""
    x, mask = oli.net_inputs(22, 1, 96, 200)
    x, mask = x.to(DEV), mask.to(DEV)
    z = model.infer(x, mask)
    _, blur = oli.prepare_mask(mask, x)
    keep = (blur == 0).expand_as(x)
    assert keep.float().mean() > 0.3
    assert torch.equal(z[keep], x[keep])


def test_batch_invariance(model):
    x, mask = oli.net_inputs(23, 3, 64, 130)
    x, mask = x.to(DEV), mask.to(DEV)
    z = model.infer(x, mask, mirror=True)
    for b in range(3):
        assert torch.equal(z[b:b + 1], model.infer(x[b:b + 1], mask[b:b + 1], mirror=True))


def test_tensor_core_and_simt_token_mixing_agree(model):
    x, mask = oli.net_inputs(24, 1, 80, 144)
    x, mask = x.to(DEV), mask.to(DEV)
    a = model.infer(x, mask)
    _lib.lib().nb200_tune_set(7, 1)
    try:
        b = model.infer(x, mask)
    finally:
        _lib.lib().nb200_tune_set(7, 0)
    s = stats(a, b)
    log_metric("light_inpaint_mma_vs_simt", **s)
    assert s["max"] < 2e-2 and s["mean"] < 1e-4, s


@pytest.mark.parametrize("i", range(len(gg.DRV_CASES)))
def test_driver_golden(g, sd, model, i):
    from nunif_b200.iw3 import ForwardInpaint
    seed, div, conv, view, inner, outer, mw = gg.DRV_CASES[i]
    x, depth = gg.drv_inputs(seed, mw)
    x, depth = x.to(DEV), depth.to(DEV)
    fi = ForwardInpaint(model, DEV)
    fi.set_mode("image")
    left, right = fi.infer(x, depth, div, conv, gg.VIEWS[view], inner_dilation=inner, outer_dilation=outer,
                           max_width=mw or None)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        la, ra = oli.forward_inpaint(sd_dev(sd), x, depth, div, conv, gg.VIEWS[view], inner, outer, mw or None)
    for tag, got, want, amp in (("left", left, t(g[f"drv{i}_left"]).to(DEV), la.float()),
                                ("right", right, t(g[f"drv{i}_right"]).to(DEV), ra.float())):
        # the check() criterion, except that on these 4096-pixel eyes p99.9 is the 5th-largest error of a plane and gets the
        # same 1.5 x allowance as the max
        ours, ref = stats(got, want), stats(amp, want)
        log_metric(f"forward_inpaint_drv{i}_{tag}", ours_max=ours["max"], refamp_max=ref["max"], ours_mean=ours["mean"],
                   refamp_mean=ref["mean"], ours_p999=ours["p999"], refamp_p999=ref["p999"])
        assert ours["mean"] <= max(5e-4, ref["mean"]), (tag, ours, ref)
        assert ours["p999"] <= max(1e-3, 1.5 * ref["p999"]), (tag, ours, ref)
        assert ours["max"] <= max(1e-3, 1.5 * ref["max"]), (tag, ours, ref)
    if gg.VIEWS[view] == "right" and not mw:
        assert torch.equal(left, x)
    if gg.VIEWS[view] == "left" and not mw:
        assert torch.equal(right, x)


def test_production_shape_1080p(sd, model):
    from nunif_b200.iw3 import ForwardInpaint
    x = synth.synth_image(31, 3, 1080, 1920).unsqueeze(0).to(DEV)
    depth = synth.synth_depth(31, 1, 392, 686).to(DEV)
    left, right = ForwardInpaint(model, DEV).infer(x, depth, 2.0, 0.5)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        la, ra = oli.forward_inpaint(sd_dev(sd), x, depth, 2.0, 0.5)
    for tag, got, amp in (("left", left, la.float()), ("right", right, ra.float())):
        s = stats(got, amp)
        log_metric(f"forward_inpaint_1080p_{tag}_vs_autocast", **s)
        assert s["mean"] < 1e-4 and s["p999"] < 2e-2, (tag, s)


def test_apply_divergence_forward_inpaint(model):
    from nunif_b200.iw3 import apply_divergence, ForwardInpaint
    x = synth.synth_image(32, 3, 32, 128).to(DEV)
    depth = synth.synth_depth(32, 1, 32, 64)[0].to(DEV)
    args = types.SimpleNamespace(method="forward_inpaint", mapper="none", convergence=0.5, divergence=10.0,
                                 synthetic_view="both", mask_inner_dilation=1, mask_outer_dilation=2, inpaint_max_width=None)
    fi = ForwardInpaint(model, DEV)
    left, right = apply_divergence(depth, x, args, fi)
    l2, r2 = fi.infer(x[None], depth[None], 10.0, 0.5, inner_dilation=1, outer_dilation=2)
    assert torch.equal(left, l2[0]) and torch.equal(right, r2[0])


def test_strict_keys(sd):
    from nunif_b200.iw3.row_flow import _create
    bad = dict(sd)
    bad.pop("enc2.3.norm2.weight")
    with pytest.raises(RuntimeError, match="missing key"):
        _create(15, bad, torch.device(DEV))
    bad = dict(sd)
    bad["extra"] = torch.zeros(1)
    with pytest.raises(RuntimeError, match="unexpected key"):
        _create(15, bad, torch.device(DEV))
