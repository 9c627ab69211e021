"""The per-frame compute of iw3's video conversion on the engine: ``bind_single_frame_callback`` (iw3/utils.py:618-706)
and ``bind_batch_frame_callback`` (:709-831), with the reference's names and signatures.

Frames cross the boundary as tensors already on the device; decoding, encoding and ``VU.to_frame`` stay with the caller,
as for the video export (export.py).  Each released frame is paired with the depth the EMA look-ahead releases for it,
a scene boundary flushes and then resets the normaliser, and the end of the stream flushes it.

When the normaliser looks ahead (``get_ema_buffer_size() > 1``) the reference parks every source frame on the host as
``round(clamp(x * 255))`` uint8 (uint16 for a 16-bit ``--pix-fmt`` or source) and uploads it again on release.  The
engine keeps those frames on the device instead, in a ring of HWC uint8 / uint16 slots allocated once per frame shape
(``SourceRing``), with the same quantisation: the warp sees the same source pixels as in the reference.  With buffer
size 1 the queue holds the preprocessed float frames, as the reference's does.

With ``nunif_b200.nunif.video.FrameBatchPipeline`` the caller's loop can hand over the decoded planes and receive the
encoder's planes, so that neither colour conversion runs on the host:

    pix_fmt, source, target = configure_colorspace(input_stream, args.colorspace, args.pix_fmt)
    cb = bind_batch_frame_callback(depth_model, side_model, segment_pts, args)
    pipe = FrameBatchPipeline(lambda x: cb(x, next_pts(len(x))), args.batch_size,
                              use_16bit=pix_fmt_requires_16bit(pix_fmt), source=source, target=target)
    for frame in container.decode(input_stream):
        for planes in pipe(frame.to_ndarray()):
            output_container.mux(output_stream.encode(av.VideoFrame.from_ndarray(planes, format=pix_fmt)))
    for planes in pipe.finish():
        ...   # encode as above; then cb(None, None, True) flushes the EMA look-ahead as float frames, which the caller
              # quantises (chw_float_to_hwc) and converts (rgb_to_yuv(..., *target)) itself"""
from collections import deque

import torch

from .. import _lib
from .frames import hwc_to_chw_float
from .postprocess import postprocess_image
from .utils import apply_divergence, apply_rgbd, debug_depth_image, preprocess_image

_BITS = {torch.uint8: 8, torch.uint16: 16}
# the pixel formats for which iw3 writes 16-bit frames (nunif/utils/video.py pix_fmt_requires_16bit)
_PIX_FMT_16BIT = frozenset({"yuv420p10le", "p010le", "yuv422p10le", "yuv444p10le", "yuv420p12le", "yuv422p12le",
                            "yuv444p12le", "yuv444p16le", "gbrp16le", "gbrp12le", "gbrp10le", "rgb48le"})


def pix_fmt_requires_16bit(pix_fmt):
    return pix_fmt in _PIX_FMT_16BIT


def _arg(args, name, default=None):
    return getattr(args, name, default)


def _chunks(items, n):
    for i in range(0, len(items), n):
        yield items[i:i + n]


def _infer(depth_model, x, args):
    return depth_model.infer(x, tta=_arg(args, "tta", False), low_vram=_arg(args, "low_vram", False),
                             enable_amp=not _arg(args, "disable_amp", False), edge_dilation=_arg(args, "edge_dilation", 2),
                             depth_aa=_arg(args, "depth_aa", False))


class SourceRing:
    """FIFO of source frames waiting for their depth, as HWC uint8 / uint16 slots of one device buffer.

    ``capacity`` is the most frames that can wait at once: the normaliser holds ``buffer_size - 1`` frames between calls,
    and a call adds its own frames before any is released.  The buffer is allocated when the first frame of a shape or
    bit depth arrives; frames of an earlier shape keep their buffer alive until they are released.  Stores and loads are
    the bit-exact frame_ops conversions (csrc/frame_ops.cu), launched on the current stream with no host synchronisation.
    """

    def __init__(self, capacity):
        self.capacity = int(capacity)
        self.buf = None
        self.next_slot = 0
        self.entries = deque()          # (buffer, slot, pts), oldest first

    def _reserve(self, n, shape, dtype, device):
        """``n`` consecutive slots for frames of HWC ``shape``: a list of (first slot, count) runs (two when it wraps)."""
        if len(self.entries) + n > self.capacity:
            raise RuntimeError(f"the source ring holds {self.capacity} frames; {len(self.entries) + n} are waiting")
        if self.buf is None or tuple(self.buf.shape[1:]) != tuple(shape) or self.buf.dtype != dtype or self.buf.device != device:
            self.buf = torch.empty((self.capacity,) + tuple(shape), dtype=dtype, device=device)
            self.next_slot = 0
        s = self.next_slot
        self.next_slot = (s + n) % self.capacity
        first = min(n, self.capacity - s)
        return [(s, first)] + ([(0, n - first)] if n > first else [])

    def _append(self, runs, pts):
        for (s, k) in runs:
            for j in range(k):
                self.entries.append((self.buf, s + j, pts.pop(0)))

    def push_hwc(self, frame, pts):
        """Copy one HWC uint8 / uint16 frame (a decoded frame that needs no preprocessing) into a slot."""
        ((s, _),) = self._reserve(1, frame.shape, frame.dtype, frame.device)
        self.buf[s].copy_(frame)
        self._append([(s, 1)], [pts])

    def push_float(self, x, pts, bits):
        """Quantise CHW / BCHW float frames in [0, 1] into slots: ``round(x * (2**bits - 1))``, half to even, saturated
        (the reference's ``(x * scale).round().clamp(0, scale).to(dtype)``)."""
        x = x.unsqueeze(0) if x.ndim == 3 else x
        xf = x.float().contiguous()
        B, _, H, W = xf.shape
        pts = list(pts)
        runs = self._reserve(B, (H, W, 3), torch.uint16 if bits == 16 else torch.uint8, x.device)
        i = 0
        with torch.cuda.device(x.device):
            for s, k in runs:
                _lib.check(_lib.lib().nb200_chw_f32_to_hwc(_lib.ptr(xf[i]), bits, k, H, W, _lib.ptr(self.buf[s]),
                                                           _lib.stream_ptr(x.device)))
                i += k
        self._append(runs, pts)

    def pop(self, n):
        """The ``n`` oldest frames as float32 B,3,H,W in [0, 1] and their pts."""
        entries = [self.entries.popleft() for _ in range(n)]
        buf0 = entries[0][0]
        if any(b is not buf0 for b, _, _ in entries):
            raise ValueError("the frame size changed inside one batch of released frames")
        H, W = buf0.shape[1:3]
        out = torch.empty((n, 3, H, W), dtype=torch.float32, device=buf0.device)
        i = 0
        with torch.cuda.device(buf0.device):
            while i < n:
                s, k = entries[i][1], 1
                while i + k < n and entries[i + k][1] == s + k:
                    k += 1
                _lib.check(_lib.lib().nb200_hwc_to_chw_f32(_lib.ptr(buf0[s]), _BITS[buf0.dtype], k, H, W, _lib.ptr(out[i]),
                                                           _lib.stream_ptr(buf0.device)))
                i += k
        return out, [p for _, _, p in entries]


def bind_single_frame_callback(depth_model, side_model, segment_pts, args):
    """iw3/utils.py:618-706.  Returns ``callback(frame, pts)``: ``frame`` is one HWC uint8 / uint16 frame on the device,
    ``pts`` its presentation timestamp; ``callback(None, None)`` flushes at the end of the video.  Each call returns the
    list of output frames released so far, in order, as CHW float on the device (``VU.to_frame`` stays with the caller).

    ``--debug-depth`` frames get the reference's 8-row red line at the top when their pts is a scene boundary."""
    device = args.state["device"]
    look_ahead = depth_model.get_ema_buffer_size() > 1
    ring = SourceRing(depth_model.get_ema_buffer_size()) if look_ahead else None
    src_queue = deque()               # buffer size 1: (preprocessed CHW float frame, pts)
    preprocess = (_arg(args, "max_output_height", None) is not None or _arg(args, "rotate_right", False)
                  or _arg(args, "rotate_left", False))

    def _postprocess(depths, flush):
        frames = []
        for depth in depths:
            if look_ahead:
                x, (pts,) = ring.pop(1)
                x = x[0]
            else:
                x, pts = src_queue.popleft()
            reset_pts = [pts in segment_pts]
            if _arg(args, "debug_depth", False):
                out = [debug_depth_image(depth, args)]
            elif _arg(args, "rgbd", False) or _arg(args, "half_rgbd", False):
                left_eye, right_eye = apply_rgbd(x, depth, mapper=args.mapper)
                out = [postprocess_image(left_eye, right_eye, args)]
            else:
                left_eye, right_eye = apply_divergence(depth, x, args, side_model, reset_pts=reset_pts)
                if left_eye is None:
                    out = []
                elif left_eye.ndim == 3:
                    out = [postprocess_image(left_eye, right_eye, args)]
                else:
                    out = [postprocess_image(left, right, args) for left, right in zip(left_eye, right_eye)]
            if pts in segment_pts and _arg(args, "debug_depth", False):
                for o in out:
                    o[0, 0:8, :] = 1.0        # the debug red line
            frames += out
        if flush and hasattr(side_model, "flush"):
            # the video inpaint models' delayed frames; the engine does not build them (their set_mode("video") raises)
            left_eye, right_eye = side_model.flush(enable_amp=not _arg(args, "disable_amp", False))
            if left_eye is not None:
                frames += [postprocess_image(left, right, args) for left, right in zip(left_eye, right_eye)]
        return frames

    @torch.inference_mode()
    def callback(frame, pts):
        if frame is None:
            return _postprocess(depth_model.flush_minmax_normalize(), flush=True)
        if frame.dtype not in _BITS:
            raise ValueError(f"expected an HWC uint8 / uint16 frame, got {frame.dtype}")
        x = hwc_to_chw_float(frame, device)
        if look_ahead:
            if preprocess:
                x = preprocess_image(x, args)
                ring.push_float(x, [pts], _BITS[frame.dtype])
            else:
                ring.push_hwc(frame.to(device), pts)
        else:
            x = preprocess_image(x, args)
            src_queue.append((x, pts))
        depth = depth_model.minmax_normalize_chw(_infer(depth_model, x, args))
        depths = [depth] if depth is not None else []
        flush = pts in segment_pts
        if flush:
            depths += depth_model.flush_minmax_normalize()
            depth_model.reset_state()
        return _postprocess(depths, flush=flush)

    return callback


def bind_batch_frame_callback(depth_model, side_model, segment_pts, args):
    """iw3/utils.py:709-831.  Returns ``callback(x, pts, flush)``: ``x`` is B,3,H,W float in [0, 1] on the device and
    ``pts`` its B timestamps; ``callback(None, None, True)`` flushes at the end of the video.  Each call returns the frames
    released so far as one B',3,H',W' float tensor on the device, or None when none is released.  Released frames are
    warped in chunks of ``args.batch_size``, as in the reference.

    The reference returns a ``(_cuda_stream_wrapper, _preprocess)`` pair whose ticket locks and per-thread streams put
    its worker threads back in order.  The engine runs one process per GPU and issues that process's work on one stream
    (DESIGN.md section 6), so the callback is called in order and needs neither; ``--cuda-stream`` is accepted and
    changes nothing.  ``--debug-depth`` gives the depth images without the single-frame callback's red line (the
    reference sends ``--debug-depth`` to the single-frame callback)."""
    look_ahead = depth_model.get_ema_buffer_size() > 1
    use_16bit = pix_fmt_requires_16bit(_arg(args, "pix_fmt", None))
    batch_size = args.batch_size
    ring = None                       # sized from the first call's batch
    src_queue = deque()               # buffer size 1: (preprocessed B,3,H,W float frames, their pts)

    def _release(depth_list):
        frames = []
        for depths in _chunks(depth_list, batch_size):
            depths = torch.stack(depths)
            if look_ahead:
                x_srcs, pts = ring.pop(len(depths))
            else:
                x_srcs, pts = src_queue.popleft()
                if x_srcs.shape[0] != depths.shape[0]:
                    raise ValueError(f"a batch of {x_srcs.shape[0]} frames is larger than args.batch_size ({batch_size})")
            reset_pts = [t in segment_pts for t in pts]
            if _arg(args, "debug_depth", False):
                frames += [debug_depth_image(d, args) for d in depths]
                continue
            if _arg(args, "rgbd", False) or _arg(args, "half_rgbd", False):
                left_eyes, right_eyes = apply_rgbd(x_srcs, depths, mapper=args.mapper)
            else:
                left_eyes, right_eyes = apply_divergence(depths, x_srcs, args, side_model, reset_pts=reset_pts)
            frames += [postprocess_image(left_eyes[i], right_eyes[i], args) for i in range(left_eyes.shape[0])]
        return torch.stack(frames) if frames else None

    @torch.inference_mode()
    def callback(x, pts, flush=False):
        nonlocal ring
        if flush:
            return _release(depth_model.flush_minmax_normalize())
        _lib.require_cuda(x, "x")
        pts = list(pts)
        if x.ndim != 4 or x.shape[0] != len(pts):
            raise ValueError("expected B,3,H,W frames with B timestamps")
        x = preprocess_image(x, args)
        if look_ahead:
            if ring is None:
                ring = SourceRing(depth_model.get_ema_buffer_size() - 1 + max(batch_size, x.shape[0]))
            ring.push_float(x, pts, 16 if use_16bit else 8)
        else:
            src_queue.append((x, pts))
        depth_batch = _infer(depth_model, x, args)
        return _release(depth_model.minmax_normalize(depth_batch, reset_ema=[t in segment_pts for t in pts]))

    return callback
