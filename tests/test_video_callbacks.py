"""CPU: what tests/golden/video_callbacks.npz pins about the reference's video callbacks (oracle/gen_golden_video_callbacks.py):
how many frames each callback releases and which source pts each belongs to, and that the batch callback's frames equal
the single-frame callback's."""
import json

import numpy as np
import pytest

from tests.util import load_golden

G = load_golden("video_callbacks")
META = json.loads(str(G["meta"]))
T, STEP = META["T"], META["pts_step"]


def _runs(case):
    return ["single"] + ([f"batch{bs}" for bs in META["batch_sizes"]] if "batch" in META["cases"][case][3] else [])


@pytest.mark.parametrize("case", list(META["cases"]))
def test_every_frame_released_once_in_source_order(case):
    """Look-ahead or not, every source frame comes out exactly once and in pts order; the scene boundaries and the final
    flush release the frames the normaliser still holds."""
    for run in _runs(case):
        pts = G[f"{case}/{run}/pts"]
        np.testing.assert_array_equal(pts, np.arange(T) * STEP, err_msg=f"{case}/{run}")
        assert len(G[f"{case}/{run}/sha256"]) == T


@pytest.mark.parametrize("case", [c for c in META["cases"] if "batch" in META["cases"][c][3]])
def test_batch_frames_equal_single_frame_frames(case):
    for run in _runs(case)[1:]:
        np.testing.assert_array_equal(G[f"{case}/{run}/sha256"], G[f"{case}/single/sha256"], err_msg=f"{case}/{run}")


def test_debug_depth_red_line_only_on_scene_boundaries():
    rows = G["debug_b5/single/rows"]         # row 7 is the red line's last row, row 8 the first one below it
    boundary = np.isin(np.arange(T), META["scene_frames"])
    assert np.all(rows[boundary, 0, 0] == 1.0)
    assert not np.any(np.all(rows[~boundary, 0, 0] == 1.0, axis=-1))
    assert not np.any(np.all(rows[:, 0, 1] == 1.0, axis=-1))


def test_pix_fmt_requires_16bit():
    from nunif_b200.iw3.video import pix_fmt_requires_16bit
    assert pix_fmt_requires_16bit("yuv420p10le") and pix_fmt_requires_16bit("rgb48le")
    assert not pix_fmt_requires_16bit("yuv420p") and not pix_fmt_requires_16bit("yuv444p")
