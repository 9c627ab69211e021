"""GPU: iw3's frame steps around depth and warp on the engine: the autocrop detector (csrc/autocrop.cu) against the real
reference's masks and slices (tests/golden/autocrop.npz) and against the oracle evaluated by ATen on the same GPU at 1080p and
4K, the device-resident video detector, rot90, the align_corners bicubic resize, apply_rgbd / debug_depth_image, and
process_image end to end with every new option.

Exclusions (1080p / 4K): the engine sums a line in its own order, so its mean may differ from torch's in the last bits.  A
black-mode line whose oracle mean lies within DELTA of 32/255, or whose max deviation lies within DELTA of 16/255, may
differ; so may a flat-mode line whose within-fraction lies within one ulp of 0.99.  The test computes these lines and
asserts that the synthetic frames have none."""
import argparse

import numpy as np
import pytest
import torch
import torch.nn.functional as F

from tests.util import load_golden, t, log_metric
from nunif_b200 import synth
from oracle import autocrop as oac
from oracle.gen_golden_autocrop import CASES, MODES, case_frame, seq_frames, slice_ints

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
DELTA = 1e-4


@pytest.fixture(scope="module")
def g():
    return load_golden("autocrop")


def _masks(x, mode):
    from nunif_b200.nunif.autocrop import _run
    return _run(x, mode, masks=True, stats=True)


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_masks_and_slices_equal_reference(g, case):
    from nunif_b200.nunif import AutoCrop, AutoCropDetector
    name = case[0]
    x = case_frame(case).to(DEV)
    for mode in MODES:
        for m in (mode, mode.upper()):
            if mode in oac.TB:
                got = AutoCropDetector.detect_tb(x, m.startswith(("black", "BLACK")))
                assert got.shape == (1, x.shape[1], 1)
                assert np.array_equal(got.flatten().cpu().numpy(), g[f"case/{name}/{mode}/mask_tb"].astype(bool)), m
            if mode in oac.LR:
                got = AutoCropDetector.detect_lr(x, m.startswith(("black", "BLACK")))
                assert got.shape == (1, 1, x.shape[2])
                assert np.array_equal(got.flatten().cpu().numpy(), g[f"case/{name}/{mode}/mask_lr"].astype(bool)), m
            assert np.array_equal(slice_ints(*AutoCropDetector.detect(x, mode=m)), g[f"case/{name}/{mode}/slice"]), m
    ac = AutoCrop.from_image(x.unsqueeze(0))
    assert list(ac.get_pad()) == g[f"case/{name}/from_image/pad"].tolist()
    assert list(ac.get_crop() or (-1,) * 4) == g[f"case/{name}/from_image/crop"].tolist()


def _frames_large():
    out = []
    for i, (h, w) in enumerate(((1080, 1920), (2160, 3840))):
        out.append((f"{h}p_black", synth.letterbox_frame(30 + i, h, w, 140, 140, 0, 0, "black")))
        out.append((f"{h}p_tv_odd", synth.letterbox_frame(32 + i, h, w, 131, 77, 241, 99, "tv")))
        out.append((f"{h}p_grey", synth.letterbox_frame(34 + i, h, w, 0, 0, 240, 240, "grey")))
        out.append((f"{h}p_dark", synth.letterbox_frame(36 + i, h, w, 100, 100, 50, 50, "dark_texture")))
    return out


def _ambiguous(black, center, spread):
    """Lines whose decision may differ from torch's through summation order alone (module docstring)."""
    if black:
        return ((center - 32.0 / 255.0).abs() < DELTA) | ((spread - 16.0 / 255.0).abs() < DELTA)
    lim = torch.tensor(0.99, dtype=torch.float32, device=spread.device)
    ulp = torch.nextafter(lim, torch.tensor(1.0, device=spread.device)) - lim
    return (spread - lim).abs() <= ulp


def test_large_frames_equal_oracle_on_gpu():
    from nunif_b200.nunif import AutoCropDetector
    worst_mean = 0.0
    for name, x in _frames_large():
        x = x.to(DEV)
        H, W = x.shape[-2:]
        for mode in ("black", "flat"):
            black = mode == "black"
            m_tb, m_lr, s_tb, s_lr = _masks(x, mode)
            for dim, m, s, n in ((-1, m_tb, s_tb, H), (-2, m_lr, s_lr, W)):
                bar, center, spread = (v.flatten() for v in oac.line_stats(x, black, dim))
                amb = _ambiguous(black, center, spread)
                assert not bool(amb.any()), (name, mode, dim, int(amb.sum()))
                assert torch.equal(m[0].bool(), bar), (name, mode, dim)
                if black:
                    worst_mean = max(worst_mean, float((s[0] - center).abs().max()))
                else:
                    # the exact lower median: torch.median on the same GPU, bit for bit
                    assert torch.equal(s[0], center), (name, dim)
            want = oac.detect(x, mode)
            assert AutoCropDetector.detect(x, mode) == want, (name, mode)
    log_metric("autocrop_large_frames", worst_mean_vs_torch=worst_mean)
    assert worst_mean < 1e-6


def test_flat_median_equals_torch_median_on_ties_and_odd_lengths():
    g = torch.Generator().manual_seed(7)
    for h, w in ((37, 53), (64, 64), (2, 3), (1, 9), (300, 1)):
        x = torch.floor(torch.rand(3, h, w, generator=g) * 6) / 6        # many ties
        x[:, : h // 2] = torch.rand(3, h // 2, w, generator=g)
        x = x.to(DEV)
        _, _, s_tb, s_lr = _masks(x, "flat")
        y = oac.luma(x, False)
        assert torch.equal(s_tb[0], y.median(dim=-1).values.flatten()), (h, w)
        assert torch.equal(s_lr[0], y.median(dim=-2).values.flatten()), (h, w)


def test_video_detector_on_device_without_sync(g):
    from nunif_b200.nunif import AutoCropDetector
    frames = [f.to(DEV) for f in seq_frames()]
    batch = torch.stack(frames[8:])
    for mode in MODES:
        det = AutoCropDetector(mode=mode.upper() if mode.startswith("flat") else mode, mod=2)
        det.update(frames[0])                      # allocates the counts
        torch.cuda.synchronize()
        torch.cuda.set_sync_debug_mode("error")
        try:
            for f in frames[1:8]:
                det.update(f)
            det.update(batch)
        finally:
            torch.cuda.set_sync_debug_mode("default")
        assert det.frame_count == len(frames)
        got = det.get_crop()
        assert np.array_equal(slice_ints(*got), g[f"seq/{mode}/slice"]), mode
        want, ctb, clr = oac.get_crop(frames, mode)
        assert got == want
        if ctb is not None:
            assert torch.equal(det.border_count_tb, ctb.int()) and np.array_equal(det.border_count_tb.flatten().cpu().numpy(), g[f"seq/{mode}/count_tb"])
        if clr is not None:
            assert torch.equal(det.border_count_lr, clr.int()) and np.array_equal(det.border_count_lr.flatten().cpu().numpy(), g[f"seq/{mode}/count_lr"])
        # a stricter and a looser threshold give the oracle's answer too
        for thr in (0.9, 1.0):
            assert det.get_crop(thr) == oac.get_crop(frames, mode, threshold=thr)[0], (mode, thr)
        det.reset()
        assert det.get_crop() == (slice(None), slice(None))


@pytest.mark.parametrize("shape", [(3, 1080, 1920), (2, 3, 37, 65), (3, 1, 7), (3, 33, 1)])
def test_rot90_bit_exact(shape):
    from nunif_b200.iw3 import rot90
    x = torch.rand(shape, generator=torch.Generator().manual_seed(3)).to(DEV)
    for k in (1, 3):
        assert torch.equal(rot90(x, k), torch.rot90(x, k, (-2, -1))), k


@pytest.mark.parametrize("src,dst", [((2160, 3840), (1080, 1920)), ((1080, 1920), (720, 1280)), ((1081, 1921), (718, 1276)),
                                     ((61, 90), (1, 3))])
def test_resize_align_corners_matches_aten(src, dst):
    from nunif_b200.iw3 import resize_bicubic_aa
    x = synth.synth_image(9, 3, *src).to(DEV)
    got = resize_bicubic_aa(x, dst, align_corners=True)
    want = F.interpolate(x.unsqueeze(0), dst, mode="bicubic", antialias=True, align_corners=True)[0]
    err = float((got - want).abs().max())
    log_metric("resize_bicubic_aa_align_corners", src=src, dst=dst, max_err=err)
    assert err <= 1e-6, err
    clamped = resize_bicubic_aa(x, dst, clamp=True, align_corners=True)
    assert torch.equal(clamped, got.clamp(0, 1))


def test_preprocess_image_matches_oracle():
    from nunif_b200.iw3 import preprocess_image
    x = synth.synth_image(10, 3, 2160, 3840).to(DEV)
    for kw in (dict(max_output_height=1080), dict(rotate_left=True), dict(rotate_right=True, max_output_height=1081),
               dict(rotate_left=True, max_output_height=2000), dict()):
        got = preprocess_image(x, argparse.Namespace(**kw))
        want = oac.preprocess_image(x, **kw)
        assert got.shape == want.shape, kw
        assert float((got - want).abs().max()) <= 1e-6, kw
        if "max_output_height" not in kw:
            assert torch.equal(got, want)
    assert preprocess_image(x, argparse.Namespace()) is x
    b = torch.stack([x[:, :540, :960], x[:, 540:1080, :960]])
    got = preprocess_image(b, argparse.Namespace(rotate_right=True, max_output_height=480))
    assert float((got - oac.preprocess_image(b, rotate_right=True, max_output_height=480)).abs().max()) <= 1e-6


@pytest.mark.parametrize("mapper", ["div_6", "mul_1+mul_2=0.5", None])
def test_apply_rgbd_and_debug_depth_match_oracle(mapper):
    from nunif_b200.iw3 import apply_rgbd, debug_depth_image
    im = synth.synth_image(11, 3, 270, 480).to(DEV)
    depth = synth.synth_depth(12, 1, 140, 250)[0].to(DEV)
    left, right = apply_rgbd(im, depth, mapper)
    wl, wr = oac.apply_rgbd(im, depth, mapper)
    assert left is im and right.shape == im.shape
    # the align_corners=False resize rounds its centre like ATen's CPU kernel; ATen's CUDA kernel does not (2e-6 here)
    assert float((right - wr).abs().max()) <= 4e-6
    name = mapper or "none"
    got = debug_depth_image(depth, argparse.Namespace(mapper=name))
    want = oac.debug_depth_image(depth, name)
    assert got.shape == (3, 140, 500) and float((got - want).abs().max()) <= 2e-6


def _args(**kw):
    a = dict(method="forward_fill", mapper="div_6", convergence=0.5, divergence=2.0, synthetic_view="both", tta=False, low_vram=False,
             disable_amp=False, edge_dilation=2, depth_aa=False, state={"convergence_model": None}, warp_steps=None,
             preserve_screen_border=False, stereo_width=None, ipd_offset=0, autocrop=None, rotate_left=False, rotate_right=False,
             max_output_height=None, rgbd=False, half_rgbd=False, debug_depth=False)
    a.update(kw)
    return argparse.Namespace(**a)


@pytest.fixture(scope="module")
def depth_model():
    from nunif_b200.iw3 import DepthAnythingModel
    dm = DepthAnythingModel("Any_V2_S")
    dm.load_state_dict(synth.depth_anything_v2_state_dict(0, pos_grid=6), gpu=0, resolution=140)
    dm.disable_ema()
    return dm


def _composed(x, args, dm, uncrop):
    """process_image restated from the oracle's frame steps around the engine's depth, warp and postprocess."""
    from nunif_b200.iw3 import apply_divergence, postprocess_image
    s = oac.detect(x, args.autocrop) if args.autocrop else (slice(None), slice(None))
    pad = oac.calc_pad(*s, *x.shape[-2:])
    xp = oac.crop(oac.preprocess_image(x, args.rotate_left, args.rotate_right, args.max_output_height), s)
    with torch.inference_mode():
        depth = dm.minmax_normalize_chw(dm.infer(xp, tta=False, edge_dilation=2))
        if args.debug_depth:
            return oac.debug_depth_image(depth, args.mapper)
        if args.rgbd or args.half_rgbd:
            left, right = oac.apply_rgbd(xp, depth, args.mapper)
        else:
            left, right = apply_divergence(depth, xp, args, None)
        if args.autocrop and uncrop:
            left, right = oac.uncrop(left, pad), oac.uncrop(right, pad)
        return postprocess_image(left, right, args)


def test_process_image_every_option(depth_model):
    from nunif_b200.iw3 import process_image, apply_divergence, postprocess_image
    x = synth.letterbox_frame(40, 200, 320, 24, 24, 0, 0, "black")
    x[:, 24:176] = synth.synth_image(41, 3, 152, 320)
    x = x.to(DEV)
    # the default path: exactly what process_image computed before these options existed
    base = process_image(x, _args(), depth_model, None)
    with torch.inference_mode():
        d = depth_model.minmax_normalize_chw(depth_model.infer(x, tta=False, edge_dilation=2))
        want = postprocess_image(*apply_divergence(d, x, _args(), None), _args())
    assert torch.equal(base, want)
    shapes = {}
    for name, kw, uncrop, tol in (("autocrop_uncrop", dict(autocrop="black"), True, 0.0),
                                  ("autocrop_crop", dict(autocrop="black"), False, 0.0),
                                  ("rotate_left_autocrop", dict(autocrop="black", rotate_left=True), True, 0.0),
                                  ("rotate_right", dict(rotate_right=True), False, 0.0),
                                  ("rgbd", dict(rgbd=True), False, 1e-5),
                                  ("half_rgbd_autocrop", dict(half_rgbd=True, autocrop="black"), True, 1e-5),
                                  ("debug_depth", dict(debug_depth=True), False, 1e-5),
                                  ("max_output_height", dict(max_output_height=160), False, None)):
        args = _args(**kw)
        got = process_image(x, args, depth_model, None, autocrop_uncrop=uncrop)
        want = _composed(x, args, depth_model, uncrop)
        assert got.shape == want.shape, name
        shapes[name] = tuple(got.shape)
        if tol is None:
            # the resized frame differs from ATen's in the last bits, and the depth network sees that
            assert float((got - want).abs().mean()) < 1e-3, name
        else:
            err = float((got - want).abs().max())
            assert err <= tol, (name, err)
        assert got.shape != base.shape or not torch.equal(got, base), name
    # the crop is found on the frame as given and applied after the rotation: rows 24..176 of the 200 x 320 frame are cut
    # from the 320 x 200 rotated frame, and the uncrop pads 24 rows back on each side
    assert shapes["autocrop_crop"] == (3, 152, 640)
    assert shapes["rotate_left_autocrop"] == (3, 152 + 2 * 24, 400)
    assert shapes["debug_depth"] == (3, d.shape[-2], 2 * d.shape[-1])
    assert process_image(x, _args(autocrop="black"), depth_model, None, skip_autocrop=True).shape == base.shape
