"""Generate tests/golden/video_callbacks.npz from the reference's own bind_single_frame_callback and
bind_batch_frame_callback (iw3/utils.py:618-831), run on the CPU with its NullDepthModel.

iw3.utils imports nunif.utils.video, which imports PyAV; a minimal ``av`` stub goes into sys.modules first.  It has the
ColorRange / Colorspace enums and a VideoFrame that wraps an HWC ndarray (to_ndarray / from_ndarray) with a pts.

The clip is a seeded synthetic 24-frame clip with pts = 1001 * index and scene boundaries at frames 7 and 16.  Stored per
case and callback: the source pts each output frame belongs to (from the callback's own source queue) and the SHA-256 of
each float output frame VU.to_frame receives.  Per case, from the single-frame callback: rows ROWS of each output frame,
its shape.  Per source clip and preprocessing (``infer_name``): the NullDepthModel.infer output of each frame.
Run: python oracle/gen_golden_video_callbacks.py"""
import enum
import hashlib
import json
import sys
import types
from argparse import Namespace
from os import path

import numpy as np
import torch

ROOT = path.dirname(path.dirname(path.abspath(__file__)))
REF = "/root/reference"
T, H, W, RES = 24, 24, 40, 16
PTS_STEP = 1001
SCENE_FRAMES = (7, 16)
ROWS = (7, 9)            # the crop stored per frame: the last row of the debug red line and the row below it
BATCH_SIZES = (1, 4)
CASES = {
    # name: (args overrides, EMA (decay, buffer_size) or None for disable_ema, 16-bit source, callbacks)
    "ff_off": (dict(method="forward_fill"), None, False, ("single", "batch")),
    "ff_b1": (dict(method="forward_fill"), (0.75, 1), False, ("single", "batch")),
    "ff_b5": (dict(method="forward_fill"), (0.9, 5), False, ("single", "batch")),
    "ff_b5_16": (dict(method="forward_fill", pix_fmt="yuv420p10le"), (0.9, 5), True, ("single", "batch")),
    "bw_b5": (dict(method="backward"), (0.9, 5), False, ("single", "batch")),
    "bw_off": (dict(method="backward"), None, False, ("single", "batch")),
    "rgbd_b5": (dict(method="forward_fill", rgbd=True), (0.9, 5), False, ("single", "batch")),
    "debug_b5": (dict(method="forward_fill", debug_depth=True), (0.9, 5), False, ("single",)),
    "pre_b5": (dict(method="backward", rotate_left=True, max_output_height=32), (0.9, 5), False, ("single", "batch")),
}


def install_av_stub():
    av = types.ModuleType("av")
    av.__version__ = "14.0.0"
    av.codecs_available = set()

    class ColorRange(enum.IntEnum):
        UNSPECIFIED = 0
        MPEG = 1
        JPEG = 2

    class Colorspace(enum.IntEnum):
        ITU709 = 1
        FCC = 4
        ITU601 = 5
        SMPTE240M = 7

    class _Format:
        def __init__(self, bits):
            self.components = [types.SimpleNamespace(bits=bits)]

    class VideoFrame:
        def __init__(self, array, pts=None):
            self.array, self.pts = array, pts
            self.format = _Format(16 if array.dtype == np.uint16 else 8)

        def to_ndarray(self, format=None, **kw):
            return self.array

        @staticmethod
        def from_ndarray(array, format=None):
            return VideoFrame(array)

    mods = {name: types.ModuleType(name) for name in (
        "av.video", "av.video.reformatter", "av.video.frame", "av.codec", "av.sidedata", "av.sidedata.sidedata")}
    mods["av.video.reformatter"].ColorRange = ColorRange
    mods["av.video.reformatter"].Colorspace = Colorspace
    mods["av.video.frame"].VideoFrame = VideoFrame
    mods["av.codec"].codecs_available = set()
    mods["av.sidedata.sidedata"].Type = enum.IntEnum("Type", "DISPLAYMATRIX")
    av.video, av.codec, av.sidedata = mods["av.video"], mods["av.codec"], mods["av.sidedata"]
    av.video.reformatter, av.video.frame = mods["av.video.reformatter"], mods["av.video.frame"]
    av.sidedata.sidedata = mods["av.sidedata.sidedata"]
    av.VideoFrame = VideoFrame
    sys.modules["av"] = av
    sys.modules.update(mods)
    return VideoFrame


def make_args(**kw):
    base = dict(method="forward_fill", divergence=2.0, convergence=0.5, synthetic_view="both", ipd_offset=0, mapper="none",
                edge_dilation=0, tta=False, low_vram=False, disable_amp=False, depth_aa=False, rotate_left=False,
                rotate_right=False, max_output_height=None, max_output_width=None, keep_aspect_ratio=False, pad=None,
                pad_mode=None, vr180=False, half_sbs=False, tb=False, half_tb=False, cross_eyed=False, anaglyph=None,
                rgbd=False, half_rgbd=False, debug_depth=False, preserve_screen_border=False, pix_fmt="yuv420p",
                batch_size=4, cuda_stream=False, stereo_width=None, warp_steps=None)
    base.update(kw)
    return Namespace(**base)


def make_clip(use_16bit):
    """Smooth moving gradients with a seeded texture, the brightness changing per frame so that the EMA matters."""
    g = torch.Generator().manual_seed(20261019)
    yy, xx = torch.meshgrid(torch.linspace(0, 1, H), torch.linspace(0, 1, W), indexing="ij")
    texture = torch.rand((3, H, W), generator=g)
    frames = []
    for k in range(T):
        base = 0.5 + 0.4 * torch.sin(6.0 * xx + 0.4 * k + torch.arange(3).view(3, 1, 1)) * torch.cos(4.0 * yy - 0.3 * k)
        x = (0.7 * base + 0.3 * texture) * (0.6 + 0.4 * ((k * 5) % 7) / 6)
        scale = 65535 if use_16bit else 255
        x = (x.clamp(0, 1).permute(1, 2, 0) * scale).round()
        frames.append(x.to(torch.uint16 if use_16bit else torch.uint8).numpy())
    return frames


def infer_name(overrides, use_16bit):
    return f"infer/{16 if use_16bit else 8}" + ("_pre" if overrides.get("rotate_left") or overrides.get("max_output_height") else "")


def cell(fn, name):
    fn = getattr(fn, "__wrapped__", fn)       # torch.inference_mode() wraps the callbacks
    return fn.__closure__[fn.__code__.co_freevars.index(name)]


class PopRecorder(list):
    """The callback's source queue: records the pts of every entry it gives up, in order."""

    def __init__(self):
        super().__init__()
        self.popped = []

    def pop(self, i=-1):
        item = super().pop(i)
        pts = item[1]
        self.popped += list(pts) if isinstance(pts, list) else [pts]
        return item


def main():
    VideoFrame = install_av_stub()
    sys.path.insert(0, REF)
    import nunif.utils.video as VU
    from iw3 import utils as U
    from iw3.null_depth_model import NullDepthModel

    captured = []
    real_to_frame = VU.to_frame

    def capture_to_frame(x, use_16bit=False):
        captured.append(x.detach().float().clone())
        return real_to_frame(x, use_16bit=use_16bit)
    VU.to_frame = capture_to_frame

    segment_pts = {k * PTS_STEP for k in SCENE_FRAMES}
    out = {"meta": json.dumps({"T": T, "H": H, "W": W, "res": RES, "pts_step": PTS_STEP, "scene_frames": SCENE_FRAMES,
                               "rows": ROWS, "batch_sizes": BATCH_SIZES, "cases": CASES})}
    clips = {False: make_clip(False), True: make_clip(True)}
    out["clip/8"] = np.stack(clips[False])
    out["clip/16"] = np.stack(clips[True])
    for name, (overrides, ema, use_16bit, callbacks) in CASES.items():
        clip = clips[use_16bit]
        runs = [("single", None)] + [("batch", bs) for bs in BATCH_SIZES] if "batch" in callbacks else [("single", None)]
        for kind, bs in runs:
            model = NullDepthModel("NULL")
            model.load(gpu=-1, resolution=RES)
            if ema is None:
                model.disable_ema()
            else:
                model.enable_ema(decay=ema[0], buffer_size=ema[1])
            infer_outputs = []
            real_infer = model.infer

            def recording_infer(x, _infer=real_infer, _outs=infer_outputs, **kw):
                y = _infer(x, **kw)
                _outs.append(y.clone())
                return y
            model.infer = recording_infer
            args = make_args(**dict(overrides, batch_size=bs or 4),
                             state={"device": torch.device("cpu"), "convergence_model": None})
            captured.clear()
            with torch.inference_mode():
                if kind == "single":
                    cb = U.bind_single_frame_callback(model, None, segment_pts, args)
                    queue = PopRecorder()
                    cell(cb, "src_queue").cell_contents = queue
                    for k, frame in enumerate(clip):
                        cb(VideoFrame(frame, pts=k * PTS_STEP))
                    cb(None)
                else:
                    run, prep = U.bind_batch_frame_callback(model, None, segment_pts, args)
                    queue = PopRecorder()
                    cell(cell(run, "_postprocess").cell_contents, "src_queue").cell_contents = queue
                    scale = 65535.0 if use_16bit else 255.0
                    for i in range(0, T, bs):
                        x = torch.from_numpy(np.stack(clip[i:i + bs])).permute(0, 3, 1, 2).contiguous() / scale
                        run(prep(x, [k * PTS_STEP for k in range(i, min(T, i + bs))], False))
                    run(prep(None, None, True))
            key = f"{name}/{kind}" + (f"{bs}" if bs else "")
            assert len(queue.popped) == len(captured), (key, len(queue.popped), len(captured))
            out[f"{key}/pts"] = np.array(queue.popped, dtype=np.int64)
            out[f"{key}/sha256"] = np.array([hashlib.sha256(f.numpy().tobytes()).hexdigest() for f in captured])
            depths = np.concatenate([y.reshape(-1, *y.shape[-3:]).numpy() for y in infer_outputs])
            if kind == "single":
                out[f"{key}/rows"] = np.stack([f[:, ROWS[0]:ROWS[1], :].numpy() for f in captured])
                out[f"{key}/shape"] = np.array(captured[0].shape)
            # the depths depend only on the clip and its preprocessing (and the batched NullDepthModel gives each frame
            # the depth it gives it alone), so cases that share those share one record
            infer_key = infer_name(overrides, use_16bit)
            if infer_key in out:
                assert np.array_equal(depths, out[infer_key]), key
            else:
                out[infer_key] = depths
            print(key, len(captured), tuple(captured[0].shape), "frames; infer calls", len(infer_outputs))
    dst = path.join(ROOT, "tests", "golden", "video_callbacks.npz")
    np.savez_compressed(dst, **out)
    print(dst, path.getsize(dst), "bytes,", len(out), "arrays")


if __name__ == "__main__":
    main()
