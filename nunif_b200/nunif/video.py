"""Frame scheduling for video callbacks: the role of ``FrameCallbackPool`` (nunif/utils/video.py:1622-1757) and of the
per-thread CUDA streams iw3 wraps around it (iw3/utils.py:709-831), re-designed for one process per GPU.

The reference overlaps host<->device copies with compute by running the batch callback on a thread pool (one stream per
thread) and converting frames with blocking ``to_tensor`` / ``to_frame`` calls.  Here the overlap comes from the hardware
queues directly - no threads, no locks, deterministic ticket order:

    slot ring (depth R, default 3), each slot = pinned uint8 input batch + device uint8 batch + pinned uint8 output batch
    copy-in stream   H2D of slot k+1 ...........  |  under
    compute stream   uint8->float (csrc/frame_ops.cu), frame_callback(batch BCHW float) , float->uint8   of slot k
    copy-out stream  D2H of slot k-1 ...........  |  under

``pipeline(frame)`` queues one HWC uint8 (or uint16) frame and returns the list of finished frames that are next in
submission order (possibly empty) - the calling convention of ``FrameCallbackPool.__call__``; ``pipeline(None)`` /
``finish()`` drains.  ``frame_callback(batch)`` receives B,3,H,W float32 in [0,1] on the GPU and returns B',3,H',W' float
(B' may differ from B: models with look-ahead buffers emit later), exactly what the reference's batch callbacks do.

``hdr2sdr`` is the reference's HDR input stage (video.py:309-416, applied by input_reformatter :1025-1041 when
``use_hdr2sdr`` holds): PQ / HLG BT.2020 rgb48 frames tone-mapped to BT.709 / BT.601 SDR by csrc/hdr2sdr.cu.
``FrameBatchPipeline(..., hdr2sdr=(color_trc, output_colorspace))`` runs it as the uint16 -> float conversion of each batch.

``FrameBatchPipeline(..., grain=(strength, speed[, seed]))`` is waifu2x's video film grain (waifu2x/ui_utils.py:167-175):
the float -> uint8 / uint16 conversion of each callback output becomes the fused temporal grain + quantise kernel
(csrc/rgb_noise.cu), whose noise buffer stays on the device and advances over the emitted frames in ticket order.

``yuv_to_rgb`` / ``rgb_to_yuv`` (csrc/yuv.cu) are the conversions the reference leaves to libswscale at both ends of its video
path: ``frame.to_ndarray(format="rgb24" | "rgb48le", **rgb24_options)`` on decoded frames and the ``reformatter`` of
``configure_colorspace`` on encoder frames (nunif/utils/video.py:621-639, :763-850).  ``guess_color_range``,
``guess_colorspace``, ``guess_rgb24_options``, ``guess_target_colorspace`` and ``configure_colorspace`` mirror that colour
policy on duck-typed PyAV streams and give the ``(pix_fmt, colorspace, color_range)`` tuples the kernels take.
``FrameBatchPipeline(..., source=..., target=...)`` then takes the decoded frame's planes and returns the encoder's planes:

    pix_fmt, source, target = configure_colorspace(input_stream, args.colorspace, args.pix_fmt)
    pipeline = FrameBatchPipeline(callback, B, use_16bit=pix_fmt_requires_16bit(pix_fmt), source=source, target=target)
    for frame in container.decode(input_stream):     # frame.format.name == source[0]
        for planes in pipeline(frame.to_ndarray()):   # one contiguous Y, U, V buffer, see plane_shape()
            encode(av.VideoFrame.from_ndarray(planes, format=pix_fmt))

A frame's planes are ONE contiguous array of shape ``plane_shape(pix_fmt, H, W)`` = (rows, W): Y [H][W], then U and V (Cb,
Cr; for gbrp* the G, B, R planes) [ceil(H/sy)][ceil(W/sx)], each with a row pitch equal to its own width in elements, and
zero padding up to a whole row of W.  For even sizes that is exactly PyAV's ``to_ndarray()`` / ``from_ndarray()`` array of
yuv420p (H*3//2, W); for yuv422p it is (2H, W), for yuv444p / gbrp (3H, W).  8-bit formats are uint8, the 10- / 16-bit
*le formats uint16.
"""
import ctypes

import torch

from .. import _lib
from ..iw3.frames import hwc_to_chw_float, chw_float_to_hwc
from ..iw3.video import pix_fmt_requires_16bit  # noqa: F401  (re-exported next to the colour policy)
from .rgb_noise import TemporalGrain

COLORSPACE_BT2020 = 9
COLOR_TRC_SMPTE2084 = 16            # PQ (HDR10)
COLOR_TRC_ARIB_STD_B67 = 18         # HLG
_HDR2SDR_TARGETS = {"bt709", "bt709-tv", "bt709-pc", "bt601", "bt601-tv", "bt601-pc"}
_SDR_COLORSPACE = {"bt709": 0, "bt601": 1}   # NB200_SDR_BT709 / NB200_SDR_BT601


def use_hdr2sdr(frame_colorspace, color_trc, target_colorspace):
    """The condition of input_reformatter (video.py:1026-1029): a BT.2020 frame of a PQ or HLG stream, written out as
    BT.709 / BT.601 (``target_colorspace`` with or without its -tv / -pc suffix)."""
    return (frame_colorspace == COLORSPACE_BT2020 and color_trc in {COLOR_TRC_SMPTE2084, COLOR_TRC_ARIB_STD_B67}
            and target_colorspace in _HDR2SDR_TARGETS)


def _check_hdr2sdr_args(color_trc, output_colorspace, output="uint16"):
    if color_trc not in (COLOR_TRC_SMPTE2084, COLOR_TRC_ARIB_STD_B67):
        raise ValueError(f"color_trc must be {COLOR_TRC_SMPTE2084} (PQ) or {COLOR_TRC_ARIB_STD_B67} (HLG), got {color_trc!r}")
    if output_colorspace not in _SDR_COLORSPACE:
        raise ValueError(f"output_colorspace must be 'bt709' or 'bt601', got {output_colorspace!r}")
    if output not in ("uint16", "float"):
        raise ValueError(f"output must be 'uint16' or 'float', got {output!r}")


def hdr2sdr(x, color_trc, output_colorspace, pq_exposure=110.0, pq_white_point=5.0, hlg_exposure=1.2, hlg_white_point=0.8,
            hlg_saturation_gain=0.9, output="uint16", device=None):
    """nunif/utils/video.py:309-416 on rgb48 frames: x uint16 HWC or BHWC, full range, BT.2020 with the PQ (color_trc 16)
    or HLG (18) transfer, moved to ``device`` (default: x's device, which must be a GPU).

    output="uint16": the tone-mapped rgb48 frame(s) hdr2sdr returns, same shape as x.
    output="float":  that frame / 65535 as float32 CHW / BCHW - the frame ``to_tensor`` / ``hwc_to_chw_float`` would make of
                     it, without the intermediate uint16 frame."""
    _check_hdr2sdr_args(color_trc, output_colorspace, output)
    if not torch.is_tensor(x) or x.dtype != torch.uint16:
        raise ValueError("hdr2sdr expects a uint16 (rgb48) tensor")
    if x.ndim not in (3, 4) or x.shape[-1] != 3:
        raise ValueError(f"hdr2sdr expects HWC or BHWC frames with 3 channels, got shape {tuple(x.shape)}")
    dev = torch.device(device) if device is not None else x.device
    if dev.type != "cuda":
        raise ValueError("hdr2sdr runs on a CUDA (sm_90) device: pass device= a GPU or a CUDA tensor")
    xc = x.to(dev).contiguous()
    B = 1 if x.ndim == 3 else x.shape[0]
    H, W = x.shape[-3], x.shape[-2]
    if output == "float":
        out = torch.empty((B, 3, H, W), dtype=torch.float32, device=xc.device)
    else:
        out = torch.empty((B, H, W, 3), dtype=torch.uint16, device=xc.device)
    params = (ctypes.c_double * 5)(pq_exposure, pq_white_point, hlg_exposure, hlg_white_point, hlg_saturation_gain)
    with torch.cuda.device(xc.device):
        _lib.check(_lib.lib().nb200_hdr2sdr(_lib.ptr(xc), B, H, W, int(color_trc), _SDR_COLORSPACE[output_colorspace], params,
                                            int(output == "float"), _lib.ptr(out), _lib.stream_ptr(xc.device)))
    return out[0] if x.ndim == 3 else out


# ---- colour policy: nunif/utils/video.py:596-850 on duck-typed PyAV streams (pix_fmt, height, format.components[0].bits,
# codec_context.{colorspace, color_range, color_primaries, color_trc}), with PyAV's enums as their integer values
COLORSPACE_ITU709 = 1               # Colorspace.ITU709 / AVCOL_SPC_BT709
COLORSPACE_UNSPECIFIED = 2
COLORSPACE_ITU601 = 5               # Colorspace.ITU601 / AVCOL_SPC_BT470BG
COLORSPACE_SMPTE170M = 6
COLORSPACE_SMPTE240M = 7
COLOR_RANGE_UNSPECIFIED, COLOR_RANGE_MPEG, COLOR_RANGE_JPEG = 0, 1, 2
KNOWN_COLORSPACES = {COLORSPACE_ITU601, COLORSPACE_ITU709, COLORSPACE_SMPTE170M, COLORSPACE_SMPTE240M, COLORSPACE_BT2020}
COLORSPACE_ARGS = ("unspecified", "auto", "copy", "bt709", "bt709-tv", "bt709-pc", "bt601", "bt601-tv", "bt601-pc",
                   "bt2020", "bt2020-tv", "bt2020-pc", "bt2020-pq-tv")


def guess_color_range(input_stream):
    """video.py:596-607: the stream's MPEG / JPEG range, else one implied by its pix_fmt, else None."""
    if input_stream.codec_context.color_range in {COLOR_RANGE_MPEG, COLOR_RANGE_JPEG}:
        return input_stream.codec_context.color_range
    if input_stream.pix_fmt.startswith("yuv4"):
        return COLOR_RANGE_MPEG
    if input_stream.pix_fmt.startswith("yuvj4") or input_stream.pix_fmt.startswith(("rgb", "gbr")):
        return COLOR_RANGE_JPEG
    return None


def guess_colorspace(input_stream):
    """video.py:610-618: the stream's colorspace, else BT.709 from 720 lines up and BT.601 below."""
    if input_stream.codec_context.colorspace != COLORSPACE_UNSPECIFIED:
        return input_stream.codec_context.colorspace
    return COLORSPACE_ITU709 if input_stream.height >= 720 else COLORSPACE_ITU601


def guess_rgb24_options(input_stream, target_colorspace):
    """video.py:621-640: the to_ndarray / reformat options that turn a decoded frame into rgb24 / rgb48le, or {}."""
    src_color_range = guess_color_range(input_stream)
    src_colorspace = guess_colorspace(input_stream)
    if src_color_range is None or src_colorspace is None:
        return {}
    if int(target_colorspace) == COLORSPACE_UNSPECIFIED:
        target_colorspace = COLORSPACE_ITU601
    fmt = "rgb48le" if input_stream.format.components[0].bits > 8 else "rgb24"
    return dict(format=fmt, src_color_range=int(src_color_range), dst_color_range=COLOR_RANGE_JPEG,
                src_colorspace=int(src_colorspace), dst_colorspace=int(target_colorspace))


def _stream_range_or(input_stream, exported_source_color_range, default):
    color_range = guess_color_range(input_stream) if input_stream is not None else None
    if color_range is None:
        color_range = exported_source_color_range if exported_source_color_range in {COLOR_RANGE_MPEG, COLOR_RANGE_JPEG} \
            else default
    return color_range


def guess_target_colorspace(input_stream, colorspace_arg, pix_fmt, exported_output_colorspace=None,
                            exported_source_color_range=None):
    """video.py:643-760: the encoder's (color_primaries, color_trc, colorspace, color_range, pix_fmt) for ``--colorspace``
    and ``--pix-fmt``; a full-range yuv420p / yuv444p output becomes yuvj420p / yuvj444p."""
    if input_stream is not None and colorspace_arg == "auto":
        colorspace_arg = "copy"
    elif input_stream is None and colorspace_arg in {"auto", "copy"}:
        family = {COLORSPACE_ITU709: "bt709", COLORSPACE_ITU601: "bt601", COLORSPACE_BT2020: "bt2020"}
        if exported_output_colorspace in family:
            suffix = "-pc" if exported_source_color_range == COLOR_RANGE_JPEG else "-tv"
            colorspace_arg = family[exported_output_colorspace] + suffix
        else:
            colorspace_arg = "bt709-tv"

    if colorspace_arg in {"bt709", "bt709-pc", "bt709-tv"}:
        color_primaries = color_trc = colorspace = COLORSPACE_ITU709
        if colorspace_arg == "bt709":
            color_range = _stream_range_or(input_stream, exported_source_color_range, COLOR_RANGE_MPEG)
        else:
            color_range = COLOR_RANGE_MPEG if colorspace_arg == "bt709-tv" else COLOR_RANGE_JPEG
    elif colorspace_arg in {"bt2020", "bt2020-pc", "bt2020-tv", "bt2020-pq-tv"}:
        color_primaries = colorspace = COLORSPACE_BT2020
        color_trc = COLOR_TRC_SMPTE2084 if colorspace_arg == "bt2020-pq-tv" else COLOR_TRC_ARIB_STD_B67
        if colorspace_arg == "bt2020":
            color_range = _stream_range_or(input_stream, exported_source_color_range, COLOR_RANGE_MPEG)
        else:
            color_range = COLOR_RANGE_JPEG if colorspace_arg == "bt2020-pc" else COLOR_RANGE_MPEG
    elif colorspace_arg in {"bt601", "bt601-pc", "bt601-tv"}:
        color_primaries, color_trc, colorspace = COLORSPACE_ITU601, 6, COLORSPACE_ITU601
        if colorspace_arg == "bt601":
            color_range = _stream_range_or(input_stream, exported_source_color_range, COLOR_RANGE_MPEG)
        else:
            color_range = COLOR_RANGE_MPEG if colorspace_arg == "bt601-tv" else COLOR_RANGE_JPEG
    elif colorspace_arg == "copy":
        cc = input_stream.codec_context
        color_primaries, color_trc, colorspace, color_range = cc.color_primaries, cc.color_trc, cc.colorspace, cc.color_range
        if color_range == COLOR_RANGE_UNSPECIFIED:
            color_range = _stream_range_or(input_stream, exported_source_color_range, COLOR_RANGE_UNSPECIFIED)
    else:
        raise ValueError(f"colorspace {colorspace_arg!r} names no output colorspace")

    if color_range == COLOR_RANGE_JPEG:
        pix_fmt = {"yuv420p": "yuvj420p", "yuv444p": "yuvj444p"}.get(pix_fmt, pix_fmt)
    return color_primaries, color_trc, colorspace, color_range, pix_fmt


def configure_colorspace(input_stream, colorspace_arg, pix_fmt):
    """The conversions video.py:763-850 picks for an encoded output of a decoded input stream, as
    ``(pix_fmt, source, target)``:

    pix_fmt  the encoder's pix_fmt (``guess_target_colorspace`` may make it yuvj*);
    source   ``(input_stream.pix_fmt, src_colorspace, src_color_range)`` of ``rgb24_options``: how the decoded frame becomes
             RGB (FrameBatchPipeline(source=...)), or None when the reference converts with no options;
    target   ``(pix_fmt, dst_colorspace, dst_color_range)`` of the ``reformatter``: how the RGB output frame becomes the
             encoder's frame (FrameBatchPipeline(target=...)), or None when frames go to the encoder as RGB."""
    if colorspace_arg not in COLORSPACE_ARGS:
        raise ValueError(f"colorspace must be one of {', '.join(COLORSPACE_ARGS)}, got {colorspace_arg!r}")
    if pix_fmt in {"rgb24", "gbrp"} or colorspace_arg == "unspecified":
        return pix_fmt, None, None
    _, _, colorspace, color_range, pix_fmt = guess_target_colorspace(input_stream, colorspace_arg, pix_fmt)
    rgb24_options, target = {}, None
    if colorspace in KNOWN_COLORSPACES:
        rgb24_options = guess_rgb24_options(input_stream, target_colorspace=colorspace)
        target = (pix_fmt, colorspace, color_range)
    elif color_range in {COLOR_RANGE_MPEG, COLOR_RANGE_JPEG}:
        target_colorspace = guess_colorspace(input_stream)
        rgb24_options = guess_rgb24_options(input_stream, target_colorspace=target_colorspace)
        target = (pix_fmt, int(target_colorspace), color_range)
    source = None
    if rgb24_options:
        source = (input_stream.pix_fmt, rgb24_options["src_colorspace"], rgb24_options["src_color_range"])
    return pix_fmt, source, target


# ---- planar YUV <-> integer RGB (csrc/yuv.cu)
_LAYOUT = {"420": (0, 2, 2), "422": (1, 2, 1), "444": (2, 1, 1), "gbr": (3, 1, 1)}   # NB200_YUV420 ... NB200_GBR, sx, sy
YUV_SOURCE_FORMATS = {"yuv420p": ("420", 8), "yuvj420p": ("420", 8), "yuv422p": ("422", 8), "yuv444p": ("444", 8),
                      "yuv420p10le": ("420", 10), "yuv422p10le": ("422", 10), "yuv444p10le": ("444", 10)}
YUV_TARGET_FORMATS = {"yuv420p": ("420", 8), "yuvj420p": ("420", 8), "yuv444p": ("444", 8), "yuvj444p": ("444", 8),
                      "yuv420p10le": ("420", 10), "gbrp": ("gbr", 8), "gbrp10le": ("gbr", 10), "gbrp16le": ("gbr", 16)}
_MATRIX = {COLORSPACE_ITU601: 0, COLORSPACE_SMPTE170M: 0, COLORSPACE_ITU709: 1, COLORSPACE_BT2020: 2}  # NB200_MATRIX_*
_RANGE = {COLOR_RANGE_MPEG: 0, COLOR_RANGE_JPEG: 1}                                                    # NB200_RANGE_*


class _YuvFormat:
    """One validated (pix_fmt, colorspace, color_range) of YUV_SOURCE_FORMATS / YUV_TARGET_FORMATS."""
    __slots__ = ("pix_fmt", "layout", "sx", "sy", "bits", "matrix", "range", "dtype")

    def __init__(self, fmt, formats, what):
        if not isinstance(fmt, (tuple, list)) or len(fmt) != 3:
            raise ValueError(f"{what} must be a (pix_fmt, colorspace, color_range) tuple, got {fmt!r}")
        pix_fmt, colorspace, color_range = fmt
        if pix_fmt not in formats:
            raise ValueError(f"unsupported {what} pix_fmt {pix_fmt!r}; supported: {', '.join(formats)}")
        layout, self.bits = formats[pix_fmt]
        self.pix_fmt = pix_fmt
        self.layout, self.sx, self.sy = _LAYOUT[layout]
        self.dtype = torch.uint8 if self.bits == 8 else torch.uint16
        if layout == "gbr":                  # planar RGB: no matrix, full range
            self.matrix, self.range = 0, 1
            return
        if colorspace not in _MATRIX:
            raise ValueError(f"unsupported {what} colorspace {colorspace!r}; supported: {COLORSPACE_ITU709} (BT.709), "
                             f"{COLORSPACE_ITU601} / {COLORSPACE_SMPTE170M} (BT.601), {COLORSPACE_BT2020} (BT.2020-NCL)")
        if color_range not in _RANGE:
            raise ValueError(f"unsupported {what} color_range {color_range!r}; supported: {COLOR_RANGE_MPEG} (MPEG, limited), "
                             f"{COLOR_RANGE_JPEG} (JPEG, full)")
        self.matrix, self.range = _MATRIX[colorspace], _RANGE[color_range]

    def rows(self, H, W):
        n = H * W + 2 * -(-W // self.sx) * -(-H // self.sy)
        return -(-n // W)

    def size(self, shape):
        """(H, W) of a plane array's trailing (rows, W); rows(H) grows strictly with H, so at most one H fits."""
        rows, W = int(shape[-2]), int(shape[-1])
        lo, hi = 1, max(rows, 1)
        while lo < hi:
            mid = (lo + hi) // 2
            if self.rows(mid, W) < rows:
                lo = mid + 1
            else:
                hi = mid
        if W < 1 or self.rows(lo, W) != rows:
            raise ValueError(f"{tuple(shape)} is not the plane array of any {self.pix_fmt} frame (see plane_shape)")
        return lo, W


def plane_shape(pix_fmt, height, width):
    """The (rows, width) array that holds one frame's planes (module docstring)."""
    formats = YUV_SOURCE_FORMATS if pix_fmt in YUV_SOURCE_FORMATS else YUV_TARGET_FORMATS
    return (_YuvFormat((pix_fmt, COLORSPACE_ITU709, COLOR_RANGE_MPEG), formats, "pix_fmt").rows(height, width), width)


def _check_bits(fmt, use_16bit, what):
    if (fmt.bits > 8) != bool(use_16bit):
        raise ValueError(f"{what} {fmt.pix_fmt} is {fmt.bits}-bit, which needs use_16bit={fmt.bits > 8} "
                         f"(rgb48 frames for the >8-bit formats, rgb24 for the 8-bit ones)")


def _yuv_to_rgb_into(planes, fmt, out):
    B, H, W = out.shape[0], out.shape[1], out.shape[2]
    _lib.check(_lib.lib().nb200_yuv_to_rgb(_lib.ptr(planes), fmt.layout, fmt.bits, fmt.matrix, fmt.range,
                                           planes.shape[-2] * planes.shape[-1], B, H, W, 16 if out.dtype == torch.uint16 else 8,
                                           _lib.ptr(out), _lib.stream_ptr(out.device)))
    return out


def _rgb_to_yuv_into(rgb, fmt, out):
    B, H, W = rgb.shape[0], rgb.shape[1], rgb.shape[2]
    _lib.check(_lib.lib().nb200_rgb_to_yuv(_lib.ptr(rgb), 16 if rgb.dtype == torch.uint16 else 8, B, H, W, fmt.layout,
                                           fmt.bits, fmt.matrix, fmt.range, out.shape[-2] * out.shape[-1], _lib.ptr(out),
                                           _lib.stream_ptr(out.device)))
    return out


def yuv_to_rgb(planes, pix_fmt, colorspace, color_range, use_16bit=False, device=None):
    """A decoded frame's planes -> the full-range HWC frame ``frame.to_ndarray(format="rgb24" | "rgb48le",
    src_colorspace=colorspace, src_color_range=color_range, dst_color_range=JPEG)`` returns (video.py:621-639).

    planes: uint8 (8-bit formats) or uint16 (10-bit) array of shape plane_shape(pix_fmt, H, W), or a batch of them;
    pix_fmt in YUV_SOURCE_FORMATS; colorspace 1 (BT.709), 5 / 6 (BT.601) or 9 (BT.2020-NCL); color_range 1 (MPEG) or 2 (JPEG);
    use_16bit: rgb48 output, which the 10-bit formats need and the 8-bit ones refuse (to_ndarray's rule).
    Returns uint8 / uint16 (H, W, 3) or (B, H, W, 3) on ``device`` (default: planes' device, which must be a GPU).
    Chroma is replicated over the luma block it covers."""
    fmt = _YuvFormat((pix_fmt, colorspace, color_range), YUV_SOURCE_FORMATS, "source")
    _check_bits(fmt, use_16bit, "source")
    planes = torch.as_tensor(planes)
    if planes.dtype != fmt.dtype or planes.ndim not in (2, 3):
        raise ValueError(f"{pix_fmt} planes must be a {fmt.dtype} (rows, W) array or a batch of them, "
                         f"got {planes.dtype} {tuple(planes.shape)}")
    H, W = fmt.size(planes.shape)
    dev = torch.device(device) if device is not None else planes.device
    if dev.type != "cuda":
        raise ValueError("yuv_to_rgb runs on a CUDA (sm_90) device: pass device= a GPU or a CUDA tensor")
    pc = planes.to(dev).contiguous()
    B = 1 if planes.ndim == 2 else planes.shape[0]
    out = torch.empty((B, H, W, 3), dtype=torch.uint16 if use_16bit else torch.uint8, device=dev)
    with torch.cuda.device(dev):
        _yuv_to_rgb_into(pc, fmt, out)
    return out[0] if planes.ndim == 2 else out


def rgb_to_yuv(frames, pix_fmt, colorspace, color_range):
    """Full-range HWC rgb24 / rgb48 frame(s) on a GPU -> the planes of ``frame.reformat(format=pix_fmt,
    dst_colorspace=colorspace, dst_color_range=color_range)`` (the reformatter of video.py:763-850).

    frames: uint8 (8-bit pix_fmt) or uint16 (10- / 16-bit) CUDA tensor (H, W, 3) or (B, H, W, 3); pix_fmt in
    YUV_TARGET_FORMATS (the gbrp* ones ignore colorspace and color_range).  Returns the plane array(s) of shape
    plane_shape(pix_fmt, H, W) (batched like ``frames``) on the same device.  4:2:0 chroma is the mean of the unrounded
    full-resolution Cb / Cr over each 2x2 block."""
    fmt = _YuvFormat((pix_fmt, colorspace, color_range), YUV_TARGET_FORMATS, "target")
    if not torch.is_tensor(frames) or frames.dtype not in (torch.uint8, torch.uint16):
        raise ValueError("rgb_to_yuv expects a uint8 (rgb24) or uint16 (rgb48) tensor")
    _check_bits(fmt, frames.dtype == torch.uint16, "target")
    if frames.ndim not in (3, 4) or frames.shape[-1] != 3:
        raise ValueError(f"rgb_to_yuv expects HWC or BHWC frames with 3 channels, got shape {tuple(frames.shape)}")
    if frames.device.type != "cuda":
        raise ValueError("rgb_to_yuv runs on a CUDA (sm_90) device: pass a CUDA tensor")
    x = (frames if frames.ndim == 4 else frames[None]).contiguous()
    B, H, W = x.shape[:3]
    out = torch.empty((B,) + (fmt.rows(H, W), W), dtype=fmt.dtype, device=x.device)
    with torch.cuda.device(x.device):
        _rgb_to_yuv_into(x, fmt, out)
    return out if frames.ndim == 4 else out[0]


class _Slot:
    __slots__ = ("h_in", "d_in", "rgb", "h_out", "n", "n_out", "ready", "done", "out_shape", "direct")

    def __init__(self):
        self.h_in = self.d_in = self.rgb = self.h_out = None
        self.n = self.n_out = 0
        self.direct = 0          # bit i: frame i of the batch being filled was copied straight from the caller's pinned memory
        self.ready = torch.cuda.Event()
        self.done = torch.cuda.Event()
        self.out_shape = None


class FrameBatchPipeline:
    def __init__(self, frame_callback, batch_size, device="cuda:0", depth=3, use_16bit=False, copy_output=True, hdr2sdr=None,
                 grain=None, source=None, target=None):
        assert batch_size > 0 and depth >= 2
        # (pix_fmt, colorspace, color_range) of the decoded frames: __call__ takes their plane arrays (plane_shape) and each
        # batch is converted to rgb24 / rgb48 on the device (yuv_to_rgb) before everything else
        self.source = _YuvFormat(source, YUV_SOURCE_FORMATS, "source") if source is not None else None
        # (pix_fmt, colorspace, color_range) of the encoder: every emitted frame is converted to its planes (rgb_to_yuv)
        # after the uint8 / uint16 conversion or grain, and returned as a plane array
        self.target = _YuvFormat(target, YUV_TARGET_FORMATS, "target") if target is not None else None
        for fmt, what in ((self.source, "source"), (self.target, "target")):
            if fmt is not None:
                _check_bits(fmt, use_16bit, what)
        # (strength, speed[, seed]): add temporal film grain to every emitted frame as it is converted for the encoder
        if grain is not None:
            if len(grain) not in (2, 3):
                raise ValueError("grain must be (strength, speed) or (strength, speed, seed)")
            grain = TemporalGrain(*grain)
        self.grain = grain
        # (color_trc, output_colorspace): tone-map each uint16 batch to SDR (hdr2sdr(..., output="float")) in place of the
        # plain uint16 -> float conversion, so the callback receives SDR frames
        if hdr2sdr is not None:
            if not use_16bit:
                raise ValueError("hdr2sdr needs use_16bit=True (rgb48 frames)")
            color_trc, output_colorspace = hdr2sdr
            _check_hdr2sdr_args(color_trc, output_colorspace)
            hdr2sdr = (color_trc, output_colorspace)
        self.hdr2sdr = hdr2sdr
        self.frame_callback = frame_callback
        self.batch_size = int(batch_size)
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise RuntimeError("FrameBatchPipeline runs on a CUDA (sm_90) device")
        self.dtype = torch.uint16 if use_16bit else torch.uint8
        self.bits = 16 if use_16bit else 8
        self.slots = [_Slot() for _ in range(depth)]
        self.s_in = torch.cuda.Stream(self.device)
        self.s_out = torch.cuda.Stream(self.device)
        self.head = 0            # slot being filled
        self.inflight = []       # slot indices in submission (ticket) order
        self.fill = 0
        self.submitted = self.returned = 0
        # False: returned frames are VIEWS of the slot's pinned output batch, valid until `depth` more batches have been submitted
        # (an encoder that consumes each frame immediately saves one host memcpy per frame)
        self.copy_output = copy_output

    # ---- host side
    def _slot_buffers(self, slot, frame):
        shape = (self.batch_size,) + tuple(frame.shape)
        if slot.h_in is None or tuple(slot.h_in.shape) != shape:
            slot.h_in = torch.empty(shape, dtype=self.dtype).pin_memory()
            slot.d_in = torch.empty(shape, dtype=self.dtype, device=self.device)
            if self.source is not None:
                slot.rgb = torch.empty((self.batch_size,) + self.source.size(frame.shape) + (3,), dtype=self.dtype,
                                       device=self.device)

    def __call__(self, frame):
        if frame is None:
            return self.finish()
        frame = torch.as_tensor(frame)
        if self.source is None:
            assert frame.ndim == 3 and frame.shape[2] == 3 and frame.dtype == self.dtype, "HWC uint8/uint16 frame expected"
        elif frame.ndim != 2 or frame.dtype != self.dtype:
            raise ValueError(f"{self.source.pix_fmt} plane array (rows, W) of {self.dtype} expected, "
                             f"got {frame.dtype} {tuple(frame.shape)}")
        else:
            self.source.size(frame.shape)
        slot = self.slots[self.head]
        if self.fill > 0 and tuple(frame.shape) != tuple(slot.h_in.shape[1:]):
            # the frame size changed inside a batch: submit the frames of the old size as a partial batch
            self._launch(slot, self.fill)
            slot = self.slots[self.head]
        if self.fill == 0:
            if self.head in self.inflight:           # ring is full: the oldest ticket must be returned first
                out = self._collect(block=True)
            else:
                out = []
            self._slot_buffers(slot, frame)
        else:
            out = []
        if frame.is_pinned() and frame.is_contiguous():
            # zero-copy submit: the frame's own page-locked memory is the DMA source (a decoder writing into pinned buffers, the
            # bench); the caller must not overwrite it before the batch it belongs to has been launched
            with torch.cuda.stream(self.s_in):
                slot.d_in[self.fill].copy_(frame, non_blocking=True)
            slot.direct |= 1 << self.fill
        else:
            slot.h_in[self.fill].copy_(frame)        # host memcpy into the pinned batch (pageable source, e.g. a PyAV ndarray)
        self.fill += 1
        if self.fill == self.batch_size:
            self._launch(slot, self.fill)
        return out + self._collect(block=False)

    def _launch(self, slot, n):
        comp = torch.cuda.current_stream(self.device)
        with torch.cuda.stream(self.s_in):
            if slot.direct == 0:
                slot.d_in[:n].copy_(slot.h_in[:n], non_blocking=True)
            else:
                for i in range(n):                   # frames staged on the host go now; the pinned ones are already in flight
                    if not (slot.direct >> i) & 1:
                        slot.d_in[i].copy_(slot.h_in[i], non_blocking=True)
            slot.ready.record(self.s_in)
        slot.direct = 0
        comp.wait_event(slot.ready)
        with torch.inference_mode():
            rgb = slot.d_in[:n] if self.source is None else _yuv_to_rgb_into(slot.d_in[:n], self.source, slot.rgb[:n])
            if self.hdr2sdr is None:
                x = hwc_to_chw_float(rgb)
            else:
                x = hdr2sdr(rgb, *self.hdr2sdr, output="float")
            y = self.frame_callback(x)
            if y is not None and y.numel() > 0:
                if self.grain is None:
                    u = chw_float_to_hwc(y, use_16bit=self.bits == 16)
                else:
                    u = self.grain(y, dtype=self.dtype)
                if self.target is not None:
                    H, W = u.shape[1], u.shape[2]
                    u = _rgb_to_yuv_into(u, self.target, torch.empty((u.shape[0], self.target.rows(H, W), W),
                                                                     dtype=self.dtype, device=u.device))
                slot.n_out = u.shape[0]
                if slot.h_out is None or tuple(slot.h_out.shape[1:]) != tuple(u.shape[1:]) or slot.h_out.shape[0] < u.shape[0]:
                    slot.h_out = torch.empty((max(u.shape[0], self.batch_size),) + tuple(u.shape[1:]), dtype=self.dtype).pin_memory()
                ev = torch.cuda.Event()
                ev.record(comp)
                self.s_out.wait_event(ev)
                with torch.cuda.stream(self.s_out):
                    slot.h_out[:slot.n_out].copy_(u, non_blocking=True)
                    u.record_stream(self.s_out)
                    slot.done.record(self.s_out)
            else:
                slot.n_out = 0
                slot.done.record(comp)
        slot.n = n
        self.inflight.append(self.head)
        self.submitted += 1
        self.head = (self.head + 1) % len(self.slots)
        self.fill = 0

    def _collect(self, block):
        out = []
        while self.inflight:
            slot = self.slots[self.inflight[0]]
            if not block and not slot.done.query():
                break
            slot.done.synchronize()
            out += [slot.h_out[i].clone() if self.copy_output else slot.h_out[i] for i in range(slot.n_out)]
            self.inflight.pop(0)
            self.returned += 1
            block = False
        return out

    def finish(self):
        """Submit the partial batch and return every remaining frame in order (FrameCallbackPool.finish)."""
        if self.fill > 0:
            self._launch(self.slots[self.head], self.fill)
        out = []
        while self.inflight:
            out += self._collect(block=True)
        return out
