"""GPU: iw3's mask_mlbw_l2 and mlbw_l2_inpaint (image mode) on the engine against the reference's goldens
(tests/golden/mask_mlbw.npz) and the oracle run under fp16 autocast (the reference's CUDA path)."""
import math
import os
import sys
import types
import pytest
import torch

from tests.util import load_golden, t, log_metric, stats
from nunif_b200 import synth, _lib
from oracle import light_inpaint as oli
from oracle import mask_mlbw as omm

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, os.path.join(ROOT, "oracle"))
import gen_golden_mask_mlbw as gg  # noqa: E402

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
AMBIGUOUS = 1e-6          # |reference sigmoid - 0.15| below which fp32 rounding may decide the pixel


@pytest.fixture(scope="module")
def g():
    return load_golden("mask_mlbw")


@pytest.fixture(scope="module")
def sd():
    return synth.mask_mlbw_state_dict(0)


@pytest.fixture(scope="module")
def sd_inp():
    return synth.light_inpaint_v1_state_dict(0)


@pytest.fixture(scope="module")
def mm(sd):
    from nunif_b200.iw3 import MLBW
    return MLBW(sd, DEV)


@pytest.fixture(scope="module")
def side(sd_inp, mm):
    from nunif_b200.iw3 import MLBWInpaint, LightInpaintV1
    return MLBWInpaint(LightInpaintV1(sd_inp, DEV), mm, DEV)


def sd_dev(sd):
    return {k: v.to(DEV) for k, v in sd.items()}


def hole_mask(logits, H, W, threshold, mirror=False):
    logits = logits.to(DEV).contiguous()
    B, _, h, w = logits.shape
    out = torch.empty((B, 1, H, W), dtype=torch.float32, device=DEV)
    _lib.check(_lib.lib().nb200_hole_mask(_lib.ptr(logits), B, h, w, H, W, float(threshold), int(mirror), _lib.ptr(out),
                                          _lib.stream_ptr()))
    return out.cpu()


def test_hole_model_flags(mm):
    assert mm.hole_mask and mm.num_layers == 2


def test_extra_head_does_not_disturb_delta(g, sd, mm):
    """delta and layer_weight of the mask model are those of the same weights without lv1_out's fifth row, run as mlbw_l2."""
    from nunif_b200.iw3 import MLBW
    plain = dict(sd)
    plain["lv1_out.1.weight"], plain["lv1_out.1.bias"] = sd["lv1_out.1.weight"][:4], sd["lv1_out.1.bias"][:4]
    m2 = MLBW(plain, DEV)
    assert not m2.hole_mask
    for i in range(len(gg.NET_CASES)):
        x = t(g[f"net{i}_x"], DEV)
        d, lw, _ = mm(x)
        d2, lw2 = m2(x)
        assert torch.equal(d, d2) and torch.equal(lw, lw2)


@pytest.mark.parametrize("i", range(len(gg.NET_CASES)))
def test_network_golden(g, mm, i):
    delta, lw, logits = mm(t(g[f"net{i}_x"], DEV))
    for name, got, want in (("delta", delta, g[f"net{i}_delta"]), ("lw", lw, g[f"net{i}_lw"]), ("logits", logits, g[f"net{i}_logits"])):
        want = t(want)
        s = stats(got.cpu(), want)
        rng = max(float(want.abs().max()), 1.0)
        log_metric(f"mask_mlbw_net{i}_{name}", max=s["max"], mean=s["mean"], range=rng)
        # the test_gpu_mlbw.py bounds: fp16 network against the fp32 reference, relative to the range
        assert s["max"] < 2e-2 * rng and s["mean"] < 2e-3 * rng, (name, s)


def test_delta_entry_point_refuses_hole_model(mm):
    x = torch.zeros(1, 3, 8, 32, device=DEV)
    d = torch.empty(1, 2, 8, 32, device=DEV)
    lw = torch.empty_like(d)
    with pytest.raises(RuntimeError, match="nb200_mlbw_delta_hole"):
        _lib.check(_lib.lib().nb200_mlbw_delta(mm._h, _lib.ptr(x), 1, 8, 32, _lib.ptr(d), _lib.ptr(lw), _lib.stream_ptr()))


def test_lib_model_rejects_odd_lv1_out(sd):
    """Only the 5-output hole head (num_layers 2) exists upstream: a 7-element lv1_out bias is refused with a clear error."""
    bad = dict(sd)
    bad["lv1_out.1.weight"] = torch.cat([sd["lv1_out.1.weight"], sd["lv1_out.1.weight"][:2]])
    bad["lv1_out.1.bias"] = torch.cat([sd["lv1_out.1.bias"], sd["lv1_out.1.bias"][:2]])
    with pytest.raises(RuntimeError, match="lv1_out.1.bias"):
        _lib.Model("MLBW", bad, torch.device(DEV))


def _pp_case(g, i):
    flip, H, W, inner, outer = gg.PP_CASES[i]
    return bool(flip), H, W, inner, outer, t(g["net0_logits"])


def _unflip(a, flip):
    return a.flip(-1) if flip else a


@pytest.mark.parametrize("i", [i for i, c in enumerate(gg.PP_CASES) if c[3] == 0 and c[4] == 0])
def test_mask_kernel_golden(g, i):
    """The engine evaluates forward_left's flipped form with mirror=1 on the natural logits: its output is compared with the
    golden made on the flipped logits, flipped back."""
    flip, H, W, _, _, lg = _pp_case(g, i)
    closed = hole_mask(lg, lg.shape[2], lg.shape[3], float("nan"), mirror=flip)
    assert torch.equal(closed, _unflip(t(g[f"pp{i}_closed"]), flip))           # closing is bit-exact
    mask = hole_mask(lg, H, W, omm.THRESHOLD, mirror=flip)
    want = _unflip(t(g[f"pp{i}_mask"]), flip).float()
    sig = _unflip(t(g[f"pp{i}_sigmoid"]), flip)
    ambiguous = (sig - omm.THRESHOLD).abs() <= AMBIGUOUS
    diff = mask != want
    log_metric(f"mask_mlbw_pp{i}", differ=int(diff.sum()), ambiguous=int(ambiguous.sum()), pixels=mask.numel())
    assert not bool((diff & ~ambiguous).any())
    assert int(ambiguous.sum()) <= 1e-4 * mask.numel()


@pytest.mark.parametrize("i", [i for i, c in enumerate(gg.PP_CASES) if c[3] or c[4]])
def test_postprocess_hole_mask_dilated_golden(g, i):
    from nunif_b200.iw3 import postprocess_hole_mask
    flip, H, W, inner, outer, lg = _pp_case(g, i)
    got = postprocess_hole_mask(lg.to(DEV), (H, W), omm.THRESHOLD, inner, outer, mirror=flip).cpu()
    want = _unflip(t(g[f"pp{i}_mask"]), flip).float()
    # pixels whose reference sigmoid is within AMBIGUOUS of the threshold, spread by the dilation runs, may differ
    j = next(k for k, c in enumerate(gg.PP_CASES) if c[:3] == gg.PP_CASES[i][:3] and c[3] == 0 and c[4] == 0)
    amb = (_unflip(t(g[f"pp{j}_sigmoid"]), flip) - omm.THRESHOLD).abs() <= AMBIGUOUS
    n = max(inner, outer)
    amb = oli.dilate_outer(oli.dilate_inner(amb, n, lg.shape[-1]), n, lg.shape[-1])
    diff = got != want
    log_metric(f"mask_mlbw_pp{i}_dilated", differ=int(diff.sum()), excluded=int(amb.sum()), covered=float(want.mean()))
    assert not bool((diff & ~amb).any())


def test_network_driven_masks(g, sd, mm):
    """Masks from the engine's logits differ from the fp32 golden in at most 1.5x as many pixels as masks from the autocast
    oracle's logits (a floor of 1e-3): the hole head's fp16 error moves no more boundary pixels than the reference's own."""
    x = t(g["net0_x"], DEV)
    _, _, logits = mm(x)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        _, _, amp_logits = omm.mask_mlbw_delta(sd_dev(sd), x)
    for i in [i for i, c in enumerate(gg.PP_CASES) if c[0] == 0]:
        _, H, W, inner, outer, _ = _pp_case(g, i)
        from nunif_b200.iw3 import postprocess_hole_mask
        want = t(g[f"pp{i}_mask"]).bool()
        ours = postprocess_hole_mask(logits, (H, W), omm.THRESHOLD, inner, outer).cpu().bool()
        amp = omm.postprocess_hole_mask(amp_logits.float().cpu(), (H, W), omm.THRESHOLD, inner, outer)
        fo, fa = float((ours != want).float().mean()), float((amp != want).float().mean())
        log_metric(f"mask_mlbw_net_mask_pp{i}", ours_frac=fo, refamp_frac=fa)
        assert fo <= max(1e-3, 1.5 * fa), (i, fo, fa)


def _eye_check(tag, got, want, amp):
    # tests/test_gpu_forward_inpaint.py::test_driver_golden's criterion
    ours, ref = stats(got, want), stats(amp, want)
    log_metric(tag, ours_max=ours["max"], refamp_max=ref["max"], ours_mean=ours["mean"], refamp_mean=ref["mean"],
               ours_p999=ours["p999"], refamp_p999=ref["p999"])
    assert ours["mean"] <= max(5e-4, ref["mean"]), (tag, ours, ref)
    assert ours["p999"] <= max(1e-3, 1.5 * ref["p999"]), (tag, ours, ref)
    assert ours["max"] <= max(1e-3, 1.5 * ref["max"]), (tag, ours, ref)


def _footprint(H, W, h, w):
    """The output pixels one closed logit reaches through the align-corners resize from h x w to H x W: the source coordinate of
    an output pixel lies within one source pixel of that logit, so (2 H / h + 1) x (2 W / w + 1) pixels."""
    return math.ceil(2 * H / h + 1) * math.ceil(2 * W / w + 1)


def test_mask_mlbw_l2_golden(g, sd, mm):
    """`--method mask_mlbw_l2`: apply_divergence_nn_LR with the hole fill z * (1 - mask).  Where the engine's hole mask equals the
    fp32 reference's, the eyes meet test_driver_golden's criterion.  A logit at the threshold can land on either side in fp16, and
    then the fill blacks out (or keeps) a whole pixel; in that case the differing pixels are bounded by one logit's footprint,
    the eye is checked to be the engine's warp times (1 - its own mask) exactly, and the pixels where the masks agree meet
    tests/test_gpu_mlbw.py::test_mlbw_apply_divergence_golden's bounds for the warp."""
    from nunif_b200.iw3 import apply_divergence_nn_LR, apply_divergence_nn_delta_weight, postprocess_hole_mask
    d, c = gg.lr_inputs()
    left, right = apply_divergence_nn_LR(mm, c.to(DEV), d.to(DEV), 2.0, 0.5, steps=1)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        la, ra = omm.apply_divergence_nn_LR(sd_dev(sd), c.to(DEV), d.to(DEV), 2.0, 0.5)
    for tag, shift, got, amp in (("left", -1, left, la), ("right", 1, right, ra)):
        want = t(g[f"lr_{tag}"])
        z, lg = apply_divergence_nn_delta_weight(mm, c.to(DEV), d.to(DEV), 2.0, 0.5, 1, shift, return_mask=True)
        m = postprocess_hole_mask(lg, c.shape[-2:], omm.THRESHOLD)
        assert torch.equal(got, z * (1 - m))
        with torch.inference_mode():
            _, ref_lg = omm.apply_divergence_mask_mlbw(sd, c, d, 2.0, 0.5, shift, return_mask=True)
        agree = m.cpu().bool() == omm.postprocess_hole_mask(ref_lg, c.shape[-2:])
        differ = int((~agree).sum())
        log_metric(f"mask_mlbw_l2_{tag}_mask", differ=differ, pixels=agree.numel())
        if differ == 0:
            _eye_check(f"mask_mlbw_l2_{tag}", got.cpu(), want, amp.float().cpu())
            continue
        assert differ <= _footprint(*c.shape[-2:], *d.shape[-2:]), (tag, differ)
        keep = agree.expand_as(want)
        s = stats(got.cpu()[keep], want[keep])
        log_metric(f"mask_mlbw_l2_{tag}_where_masks_agree", **s)
        assert s["mean"] < 1e-3 and s["max"] < 3e-2, (tag, s)


def _engine_parts(side, x, depth, div, conv, shift, psb, inner, outer):
    """The warped eye and the hole mask MLBWInpaint hands to the inpainting network for one eye (mirror for the left eye)."""
    from nunif_b200.iw3 import apply_divergence_nn_delta_weight, postprocess_hole_mask
    z, lg = apply_divergence_nn_delta_weight(side.mask_mlbw, x, depth, div, conv, 1, shift, preserve_screen_border=psb,
                                             return_mask=True)
    return z, postprocess_hole_mask(lg, z.shape[-2:], omm.THRESHOLD, inner, outer, mirror=shift < 0)


def _amp_inpaint(sd_inp, z, m, mirror):
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        if mirror:
            return oli.infer(sd_dev(sd_inp), z.flip(-1), m.flip(-1)).flip(-1).float()
        return oli.infer(sd_dev(sd_inp), z, m).float()


@pytest.mark.parametrize("i", range(len(gg.DRV_CASES)))
def test_mlbw_inpaint_golden(g, sd, sd_inp, side, i):
    """Against the fp32 golden with test_gpu_forward_inpaint.py::test_driver_golden's criterion.  A hole-mask pixel whose logit
    sits at the threshold can land on either side in fp16; one such pixel changes the 4x4 mask tokens of light_inpaint_v1 and with
    them a whole window of the painted eye.  Where the engine's mask for an eye differs from the fp32 reference's, the eye is
    instead checked against the autocast oracle's inpainting of the engine's own warped eye and mask, and the mask difference is
    bounded."""
    seed, div, conv, view, inner, outer, mw, psb = gg.DRV_CASES[i]
    x, depth = gg.drv_inputs(seed, mw)
    x, depth = x.to(DEV), depth.to(DEV)
    side.set_mode("image")
    left, right = side.infer(x, depth, div, conv, preserve_screen_border=bool(psb), synthetic_view=gg.VIEWS[view],
                             inner_dilation=inner, outer_dilation=outer, max_width=mw or None)
    with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
        la, ra = omm.mlbw_inpaint(sd_dev(sd_inp), sd_dev(sd), x, depth, div, conv, gg.VIEWS[view], inner, outer, mw or None, bool(psb))
    xr = oli.resize_max_width(x.cpu(), mw or None)
    d2 = div if gg.VIEWS[view] == "both" else div * 2
    for tag, shift, got, amp in (("left", -1, left, la), ("right", 1, right, ra)):
        if gg.VIEWS[view] not in ("both", tag):
            assert torch.equal(got.cpu(), xr)           # the golden stores no eye the view does not synthesise: it is the frame
            continue
        want = g[f"drv{i}_{tag}"]
        z, m = _engine_parts(side, xr.to(DEV), depth, d2, conv, shift, bool(psb), inner, outer)
        _, lg = omm.apply_divergence_mask_mlbw(sd, xr, depth.cpu(), d2, conv, shift, bool(psb), return_mask=True)
        lg = lg.flip(-1) if shift < 0 else lg
        ref_m = omm.postprocess_hole_mask(lg, z.shape[-2:], omm.THRESHOLD, inner, outer)
        ref_m = ref_m.flip(-1) if shift < 0 else ref_m
        differ = int((m.cpu().bool() != ref_m).sum())
        log_metric(f"mlbw_inpaint_drv{i}_{tag}_mask", differ=differ, pixels=ref_m.numel())
        if differ == 0:
            _eye_check(f"mlbw_inpaint_drv{i}_{tag}", got.cpu(), t(want), amp.float().cpu())
        else:
            assert differ <= _footprint(*z.shape[-2:], *depth.shape[-2:]), (tag, differ)    # one straddling logit
            s = stats(got, _amp_inpaint(sd_inp, z, m, shift < 0))
            log_metric(f"mlbw_inpaint_drv{i}_{tag}_own_mask_vs_autocast", **s)
            # test_driver_golden's mean floor; the 1080p test's p99.9 bound
            assert s["mean"] <= 5e-4 and s["p999"] < 2e-2, (tag, s)
    if gg.VIEWS[view] == "right" and not mw:
        assert torch.equal(left, x)
    if gg.VIEWS[view] == "left" and not mw:
        assert torch.equal(right, x)


def test_production_shape_1080p(sd, sd_inp, side):
    """Each stage at 1080p with a 392 x 686 depth map: the hole masks agree with the autocast oracle's up to threshold-straddling
    pixels, and the painted eyes agree with the autocast oracle's inpainting of the same warped eyes and masks."""
    x = synth.synth_image(31, 3, 1080, 1920).unsqueeze(0).to(DEV)
    depth = synth.synth_depth(31, 1, 392, 686).to(DEV)
    left, right = side.infer(x, depth, 2.0, 0.5)
    for tag, shift, got in (("left", -1, left), ("right", 1, right)):
        z, m = _engine_parts(side, x, depth, 2.0, 0.5, shift, False, 0, 0)
        with torch.no_grad(), torch.autocast("cuda", dtype=torch.float16):
            _, lg = omm.apply_divergence_mask_mlbw(sd_dev(sd), x, depth, 2.0, 0.5, shift, return_mask=True)
        lg = lg.float().flip(-1) if shift < 0 else lg.float()
        am = omm.postprocess_hole_mask(lg, (1080, 1920))
        am = am.flip(-1) if shift < 0 else am
        frac = float((m.bool() != am).float().mean())
        s = stats(got, _amp_inpaint(sd_inp, z, m, shift < 0))
        log_metric(f"mlbw_inpaint_1080p_{tag}_vs_autocast", mask_differ_frac=frac, covered=float(m.mean()), **s)
        assert frac <= 1e-3, (tag, frac)
        assert s["mean"] < 1e-4 and s["p999"] < 2e-2, (tag, s)


def test_batch_invariance(side):
    x = torch.stack([synth.synth_image(40 + i, 3, 48, 150) for i in range(3)]).to(DEV)
    depth = synth.synth_depth(40, 3, 40, 96).to(DEV)
    left, right = side.infer(x, depth, 4.0, 0.5, inner_dilation=1, outer_dilation=2)
    for b in range(3):
        l1, r1 = side.infer(x[b:b + 1], depth[b:b + 1], 4.0, 0.5, inner_dilation=1, outer_dilation=2)
        assert torch.equal(left[b:b + 1], l1) and torch.equal(right[b:b + 1], r1)


def test_apply_divergence_mlbw_l2_inpaint(side):
    from nunif_b200.iw3 import apply_divergence
    x = synth.synth_image(32, 3, 32, 128).to(DEV)
    depth = synth.synth_depth(32, 1, 32, 64)[0].to(DEV)
    args = types.SimpleNamespace(method="mlbw_l2_inpaint", mapper="none", convergence=0.5, divergence=4.0, synthetic_view="both",
                                 preserve_screen_border=True, mask_inner_dilation=1, mask_outer_dilation=2, inpaint_max_width=None)
    left, right = apply_divergence(depth, x, args, side)
    l2, r2 = side.infer(x[None], depth[None], 4.0, 0.5, preserve_screen_border=True, inner_dilation=1, outer_dilation=2)
    assert torch.equal(left, l2[0]) and torch.equal(right, r2[0])
