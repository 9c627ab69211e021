"""CPU: the autocrop oracle (oracle/autocrop.py) and the host logic of nunif_b200.nunif.autocrop against
tests/golden/autocrop.npz, which the real nunif/utils/autocrop.py and iw3/utils.py generated (oracle/gen_golden_autocrop.py):
masks, slices, pads and crop ranges exactly, the frame steps of process_image bit for bit, and the error behaviour."""
import numpy as np
import pytest
import torch

from tests.util import load_golden, t
from nunif_b200 import synth
from oracle import autocrop as oac
from oracle.gen_golden_autocrop import (CASES, MODES, HOST_MOD, HOST_MASKS, HOST_PAD, PRE_CASES, PRE_FRAME, RGBD_IM, RGBD_DEPTH,
                                        RGBD_MAPPERS, case_frame, seq_frames, slice_ints)


@pytest.fixture(scope="module")
def g():
    return load_golden("autocrop")


@pytest.mark.parametrize("case", CASES, ids=[c[0] for c in CASES])
def test_oracle_masks_and_slices_match_reference(g, case):
    name = case[0]
    x = case_frame(case)
    assert float(x.double().sum()) == float(g[f"case/{name}/sum"])
    for mode in MODES:
        black = mode.startswith("black")
        if mode in oac.TB:
            assert np.array_equal(oac.detect_tb(x, black).flatten().numpy(), g[f"case/{name}/{mode}/mask_tb"].astype(bool)), mode
        if mode in oac.LR:
            assert np.array_equal(oac.detect_lr(x, black).flatten().numpy(), g[f"case/{name}/{mode}/mask_lr"].astype(bool)), mode
        assert np.array_equal(slice_ints(*oac.detect(x, mode)), g[f"case/{name}/{mode}/slice"]), mode
    s = oac.detect(x, "black")
    H, W = x.shape[-2:]
    assert list(oac.calc_pad(*s, H, W)) == g[f"case/{name}/from_image/pad"].tolist()
    assert list(oac.calc_crop(*s, H, W) or (-1,) * 4) == g[f"case/{name}/from_image/crop"].tolist()


def test_oracle_video_detector_matches_reference(g):
    frames = seq_frames()
    for mode in MODES:
        (s_tb, s_lr), ctb, clr = oac.get_crop(frames, mode)
        assert np.array_equal(slice_ints(s_tb, s_lr), g[f"seq/{mode}/slice"]), mode
        if ctb is not None:
            assert np.array_equal(ctb.flatten().numpy(), g[f"seq/{mode}/count_tb"])
        if clr is not None:
            assert np.array_equal(clr.flatten().numpy(), g[f"seq/{mode}/count_lr"])
    # the sequence keeps a bar seen in 90 % of the frames and crops one seen in exactly 95 %
    assert g["seq/black/slice"].tolist() == [12, -1, 10, 152]


def test_oracle_frame_steps_match_reference(g):
    x = synth.synth_image(*PRE_FRAME)
    for name, kw in PRE_CASES:
        assert torch.equal(oac.preprocess_image(x, **kw), t(g[f"pre/{name}"])), name
    batch = torch.stack([x, x.flip(0)])
    assert torch.equal(oac.preprocess_image(batch, rotate_right=True, max_output_height=30), t(g["pre/batch_rotate_right_max_h30"]))
    im, depth = synth.synth_image(*RGBD_IM), synth.synth_depth(*RGBD_DEPTH)[0]
    for m in RGBD_MAPPERS:
        left, right = oac.apply_rgbd(im, depth, m)
        assert left is im and right.shape == im.shape
        # the oracle's mappers restate iw3/mapper.py in fp32 (tests/test_mapper.py pins them): exact for "none"
        tol = 0 if m == "none" else 2e-6
        assert float((right[0] - t(g[f"rgbd/{m}"])).abs().max()) <= tol, m
        assert float((oac.debug_depth_image(depth, m)[0] - t(g[f"debug/{m}"])).abs().max()) <= tol, m


def test_host_logic_matches_reference(g):
    from nunif_b200.nunif import AutoCrop, AutoCropDetector
    got = [slice_ints(AutoCropDetector.apply_mod(slice(a, b), m), slice(None))[:2].tolist() for a, b, m in HOST_MOD]
    assert got == g["host/apply_mod"].tolist()
    got = [slice_ints(AutoCropDetector.mask_to_slice_tb(torch.tensor(m, dtype=torch.bool).view(1, -1, 1)),
                      AutoCropDetector.mask_to_slice_lr(torch.tensor(m, dtype=torch.bool).view(1, 1, -1))).tolist() for m in HOST_MASKS]
    assert got == g["host/mask_slice"].tolist()
    got = [list(AutoCrop.calc_pad(slice(a, b), slice(c, d), H, W)) + list(AutoCrop.calc_crop(slice(a, b), slice(c, d), H, W) or (-1,) * 4)
           for a, b, c, d, H, W in HOST_PAD]
    assert got == g["host/pad_crop"].tolist()
    assert slice_ints(*AutoCropDetector(mode="flat").get_crop()).tolist() == g["host/empty_get_crop"].tolist()
    # the oracle's host logic is the same
    assert [slice_ints(oac.apply_mod(slice(a, b), m), slice(None))[:2].tolist() for a, b, m in HOST_MOD] == g["host/apply_mod"].tolist()


def test_modes_and_unbuilt_entry_points():
    from nunif_b200.nunif import AutoCrop, AutoCropDetector
    from nunif_b200.nunif.autocrop import autocrop_analyze_video
    for mode in MODES:
        assert AutoCropDetector(mode=mode.upper()).mode == mode
    # the reference accepts any string here and fails later with UnboundLocalError
    for bad in ("blackk", "flat_tblr", ""):
        with pytest.raises(ValueError):
            AutoCropDetector(mode=bad)
        with pytest.raises(ValueError):
            AutoCropDetector.detect(torch.zeros(3, 8, 8), mode=bad)
    with pytest.raises(NotImplementedError, match="PyAV"):
        AutoCrop.from_video_file("video.mp4")
    with pytest.raises(NotImplementedError, match="PyAV"):
        autocrop_analyze_video("video.mp4")
    ac = AutoCrop(slice(2, 6), slice(None), (0, 0, 2, 4), 0, (0, 2, 8, 4), True)
    x = torch.arange(2 * 3 * 10 * 8, dtype=torch.float32).view(2, 3, 10, 8)
    assert torch.equal(ac.crop(x), x[:, :, 2:6]) and torch.equal(ac.crop(x[0]), x[0, :, 2:6])
    y = ac.uncrop(ac.crop(x))
    assert y.shape == x.shape and torch.equal(y[:, :, 2:6], x[:, :, 2:6]) and float(y[:, :, :2].abs().sum()) == 0
