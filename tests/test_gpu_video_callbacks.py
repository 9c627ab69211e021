"""GPU: the engine's video callbacks (nunif_b200/iw3/video.py) against tests/golden/video_callbacks.npz, the reference's
bind_single_frame_callback / bind_batch_frame_callback with its NullDepthModel (oracle/gen_golden_video_callbacks.py).

The depth model is a stand-in whose infer replays the recorded NullDepthModel.infer outputs in call order (the engine
does not build NULL); the normaliser is the engine's.  The recorded depths are uploaded once, so that the stand-in
allocates nothing per frame and memory_allocated sees only what the callbacks keep."""
import json
from argparse import Namespace

import pytest
import torch

from tests.util import load_golden, log_metric, stats

pytestmark = pytest.mark.gpu
DEV = torch.device("cuda:0")
G = load_golden("video_callbacks")
META = json.loads(str(G["meta"]))
T, STEP, ROWS = META["T"], META["pts_step"], META["rows"]
SEGMENT_PTS = {k * STEP for k in META["scene_frames"]}


class RecordedDepth:
    def __init__(self, outputs, ema):
        from nunif_b200.iw3.base_depth_model import BaseDepthModel
        self.base = BaseDepthModel("NULL")
        self.outputs = outputs.to(DEV)            # T,1,h,w
        self.i = 0
        if ema is None:
            self.base.disable_ema()
        else:
            self.base.enable_ema(decay=ema[0], buffer_size=ema[1])

    def __getattr__(self, name):
        return getattr(self.base, name)

    def infer(self, x, **kw):
        n = 1 if x.ndim == 3 else x.shape[0]
        y = self.outputs[self.i:self.i + n]
        self.i += n
        return y[0] if x.ndim == 3 else y


def _args(**kw):
    base = dict(method="forward_fill", divergence=2.0, convergence=0.5, synthetic_view="both", ipd_offset=0, mapper="none",
                edge_dilation=0, tta=False, low_vram=False, disable_amp=False, depth_aa=False, rotate_left=False,
                rotate_right=False, max_output_height=None, max_output_width=None, keep_aspect_ratio=False, pad=None,
                pad_mode=None, vr180=False, half_sbs=False, tb=False, half_tb=False, cross_eyed=False, anaglyph=None,
                rgbd=False, half_rgbd=False, debug_depth=False, preserve_screen_border=False, pix_fmt="yuv420p",
                batch_size=4, cuda_stream=False, stereo_width=None, warp_steps=None)
    base.update(kw)
    return Namespace(**base)


def _infer_name(overrides, use_16bit):
    return f"infer/{16 if use_16bit else 8}" + ("_pre" if overrides.get("rotate_left") or overrides.get("max_output_height") else "")


def _setup(case, batch_size=4):
    overrides, ema, use_16bit, _ = META["cases"][case]
    model = RecordedDepth(torch.from_numpy(G[_infer_name(overrides, use_16bit)]), ema)
    args = _args(**dict(overrides, batch_size=batch_size), state={"device": DEV, "convergence_model": None})
    clip = torch.from_numpy(G["clip/16" if use_16bit else "clip/8"]).to(DEV)
    return model, args, clip


def run_single(case):
    from nunif_b200.iw3 import bind_single_frame_callback
    model, args, clip = _setup(case)
    cb = bind_single_frame_callback(model, None, SEGMENT_PTS, args)
    out = []
    for k in range(T):
        out += [f.cpu() for f in cb(clip[k], k * STEP)]
    out += [f.cpu() for f in cb(None, None)]
    return out


def run_batch(case, bs):
    from nunif_b200.iw3 import bind_batch_frame_callback, hwc_to_chw_float
    model, args, clip = _setup(case, bs)
    cb = bind_batch_frame_callback(model, None, SEGMENT_PTS, args)
    out = []
    for i in range(0, T, bs):
        # code / 255 (65535) as the reference's to_tensor divides; torch's CUDA division by a scalar multiplies by the
        # reciprocal, which is one ulp off for some codes
        x = hwc_to_chw_float(clip[i:i + bs])
        y = cb(x, [k * STEP for k in range(i, min(T, i + bs))], False)
        out += [] if y is None else list(y.cpu())
    y = cb(None, None, True)
    return out + ([] if y is None else list(y.cpu()))


def _check_golden(case, got):
    """The image-mode tolerances of the same method (tests/test_gpu_iw3.py).  Measured on an H100 80GB HBM3 at 700 W:
    forward_fill, --rgbd and --debug-depth are exact, backward is within 1.4e-6, rotate + resize within 3e-7."""
    overrides = META["cases"][case][0]
    assert len(got) == T, (case, len(got))
    assert tuple(got[0].shape) == tuple(G[f"{case}/single/shape"]), case
    want = torch.from_numpy(G[f"{case}/single/rows"])
    s = stats(torch.stack([f[:, ROWS[0]:ROWS[1], :] for f in got]), want)
    log_metric(f"video_callbacks_{case}", **s)
    if overrides.get("method") == "forward_fill" and not overrides.get("rgbd") and not overrides.get("debug_depth"):
        assert s["frac_gt_1e3"] < 1e-3, (case, s)          # test_forward_warp_lowres_depth
    else:
        assert s["max"] < 1e-3, (case, s)                   # test_backward_warp_golden


@pytest.mark.parametrize("case", list(META["cases"]))
def test_callbacks_match_reference(case):
    """Count, order and pixels of the single-frame callback against the reference, and the batch callback's frames
    identical to it for every batch size."""
    single = run_single(case)
    _check_golden(case, single)
    if "batch" in META["cases"][case][3]:
        for bs in META["batch_sizes"]:
            got = run_batch(case, bs)
            assert len(got) == T
            for k in range(T):
                assert torch.equal(got[k], single[k]), (case, bs, k, float((got[k] - single[k]).abs().max()))


@pytest.mark.parametrize("bs", [1, 4])
def test_batch_debug_depth_is_single_without_red_line(bs):
    single = run_single("debug_b5")
    got = run_batch("debug_b5", bs)
    assert len(got) == T
    for k in range(T):
        if k in META["scene_frames"]:
            assert torch.all(single[k][0, :8] == 1.0)
            assert torch.equal(got[k][:, 8:], single[k][:, 8:]) and torch.equal(got[k][1:], single[k][1:])
            assert not torch.all(got[k][0, :8] == 1.0)
        else:
            assert torch.equal(got[k], single[k]), k


def test_look_ahead_warps_the_quantised_source(monkeypatch):
    """With buffer 5 the warp gets round(x * 255) / 255 of the preprocessed frames, not the frames themselves."""
    from nunif_b200.iw3 import video
    seen = []
    real = video.apply_divergence

    def spy(depth, im, *a, **kw):
        seen.append(im.clone())
        return real(depth, im, *a, **kw)
    monkeypatch.setattr(video, "apply_divergence", spy)
    model, args, _ = _setup("ff_b5")
    g = torch.Generator().manual_seed(3)
    x = torch.rand((T, 3, META["H"], META["W"]), generator=g).to(DEV)
    cb = video.bind_batch_frame_callback(model, None, SEGMENT_PTS, args)
    for i in range(0, T, 4):
        cb(x[i:i + 4], [k * STEP for k in range(i, i + 4)], False)
    cb(None, None, True)
    got = torch.cat(seen)
    assert got.shape == x.shape
    quantised = ((x * 255).round().clamp(0, 255).double() / 255).float()     # code / 255, correctly rounded
    assert torch.equal(got, quantised)
    assert not torch.equal(got, x)
    assert float((got - x).abs().max()) <= 0.5 / 255 + 1e-7


@pytest.mark.parametrize("kind", ["single", "batch"])
def test_source_ring_allocates_once(kind):
    """After the first frame of a shape, the look-ahead queue makes no device allocation: memory_allocated after frame
    2 equals memory_allocated after frame 24, although the normaliser holds a different number of frames."""
    from nunif_b200.iw3 import bind_batch_frame_callback, bind_single_frame_callback
    model, args, clip = _setup("ff_b5")
    x = clip.permute(0, 3, 1, 2).float() / 255
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated(DEV)
    marks = {}
    if kind == "single":
        cb = bind_single_frame_callback(model, None, SEGMENT_PTS, args)
        for k in range(T):
            released = [f.cpu() for f in cb(clip[k], k * STEP)]
            del released
            if k + 1 in (2, T):
                torch.cuda.synchronize()
                marks[k + 1] = torch.cuda.memory_allocated(DEV)
    else:
        cb = bind_batch_frame_callback(model, None, SEGMENT_PTS, args)
        for i in range(0, T, 4):
            y = cb(x[i:i + 4], [k * STEP for k in range(i, i + 4)], False)
            y = None if y is None else y.cpu()
            del y
            if i + 4 in (4, T):
                torch.cuda.synchronize()
                marks[i + 4] = torch.cuda.memory_allocated(DEV)
    first, last = marks[min(marks)], marks[T]
    log_metric(f"video_callbacks_ring_{kind}", base=base, first=first, last=last)
    assert first == last, marks
    assert first > base            # the ring itself
    cb(None, None) if kind == "single" else cb(None, None, True)


def test_real_network_1080p_matches_process_image():
    """Any_V2_S (seeded weights), forward_fill, EMA off, 12 frames at 1080p: each callback's frame equals process_image
    on the same frame."""
    from nunif_b200 import synth
    from nunif_b200.iw3 import (DepthAnythingModel, bind_batch_frame_callback, bind_single_frame_callback, hwc_to_chw_float,
                                process_image)
    dm = DepthAnythingModel("Any_V2_S").load_state_dict(synth.depth_anything_v2_state_dict(0), gpu=0)
    dm.disable_ema()
    args = _args(method="forward_fill", edge_dilation=2, state={"device": DEV, "convergence_model": None})
    frames = [(synth.synth_image(70 + i, 3, 1080, 1920).permute(1, 2, 0) * 255).round().to(torch.uint8).to(DEV)
              for i in range(12)]
    want = [process_image(hwc_to_chw_float(f), args, dm, None) for f in frames]
    segment = {5}
    single_cb = bind_single_frame_callback(dm, None, segment, args)
    single = []
    for k, f in enumerate(frames):
        single += single_cb(f, k)
    single += single_cb(None, None)
    batch_cb = bind_batch_frame_callback(dm, None, segment, args)
    batch = []
    for i in range(0, 12, 4):
        batch += list(batch_cb(torch.stack([hwc_to_chw_float(f) for f in frames[i:i + 4]]), list(range(i, i + 4)), False))
    assert batch_cb(None, None, True) is None
    assert len(single) == len(batch) == 12
    for k in range(12):
        assert torch.equal(single[k], want[k]), k
        assert torch.equal(batch[k], want[k]), (k, stats(batch[k], want[k]))
