"""Black-bar / flat-border detection and cropping: nunif/utils/autocrop.py:6-207 on the engine (csrc/autocrop.cu).

``AutoCropDetector`` keeps its per-row and per-column bar counts on the device; ``update`` makes no host synchronisation,
``get_crop``, ``detect`` and ``AutoCrop.from_image`` make one each (4 ints).  Slices, pads and crop ranges are the
reference's, value for value.

Decoding stays with the caller (PyAV is not a dependency): ``AutoCrop.from_video_file`` and ``autocrop_analyze_video``
raise ``NotImplementedError``.  To analyse a video, feed its sampled frames (fp32 RGB CHW / BCHW in [0, 1]) to
``AutoCropDetector.update`` and build the ``AutoCrop`` from ``get_crop()`` with ``calc_pad`` / ``calc_crop``
(INTEGRATION.md)."""
import torch

from .. import _lib
from ..iw3._common import prep
from ..iw3.postprocess import _pad

MODES = ("black_tb", "black_lr", "black", "flat_tb", "flat_lr", "flat")
_TB = {"black_tb", "black", "flat_tb", "flat"}
_LR = {"black_lr", "black", "flat_lr", "flat"}


def _check_mode(mode):
    mode = mode.lower()
    if mode not in MODES:
        raise ValueError(f"autocrop mode {mode!r} is not one of {', '.join(MODES)}")
    return mode


def _run(frame, mode, count_tb=None, count_lr=None, masks=False, stats=False):
    """One nb200_autocrop_detect launch over a CHW / BCHW frame; returns (mask_tb, mask_lr, stat_tb, stat_lr) [B][H] / [B][W]
    (None where not requested or not in the mode)."""
    x = prep(frame, "frame")
    if x.ndim == 3:
        x = x.unsqueeze(0)
    if x.ndim != 4 or x.shape[1] != 3:
        raise ValueError(f"expected an RGB CHW / BCHW frame, got shape {tuple(frame.shape)}")
    B, _, H, W = x.shape
    tb, lr = mode in _TB, mode in _LR

    def buf(on, n, dtype):
        return torch.empty((B, n), dtype=dtype, device=x.device) if on else None
    m_tb, m_lr = buf(masks and tb, H, torch.uint8), buf(masks and lr, W, torch.uint8)
    s_tb, s_lr = buf(stats and tb, H, torch.float32), buf(stats and lr, W, torch.float32)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().nb200_autocrop_detect(
            _lib.ptr(x), B, H, W, 1 if mode.startswith("black") else 0, (1 if tb else 0) | (2 if lr else 0),
            _lib.ptr(m_tb), _lib.ptr(m_lr), _lib.ptr(count_tb if tb else None), _lib.ptr(count_lr if lr else None),
            _lib.ptr(s_tb), _lib.ptr(s_lr), _lib.stream_ptr(x.device)))
    return m_tb, m_lr, s_tb, s_lr


def _bounds(count_tb, count_lr, H, W, frame_count, threshold):
    """(first, last) non-bar row and column from the device counts, in one synchronisation."""
    dev = (count_tb if count_tb is not None else count_lr).device
    out = torch.empty(4, dtype=torch.int32, device=dev)
    with torch.cuda.device(dev):
        _lib.check(_lib.lib().nb200_autocrop_bounds(_lib.ptr(count_tb), H, _lib.ptr(count_lr), W, frame_count, float(threshold),
                                                    _lib.ptr(out), _lib.stream_ptr(dev)))
    return out.tolist()


def _slice_from_bounds(first, last, n):
    """mask_to_slice_*: no bar, or nothing but bars, is the full slice; an edge index becomes None."""
    if first < 0:
        return slice(None, None)
    start = first if first > 0 else None
    stop = last + 1 if last + 1 < n else None
    return slice(start, stop)


def _mask_slice(mask, n):
    keep = torch.nonzero(~mask.reshape(-1)).flatten()
    if keep.numel() == 0:
        return slice(None, None)
    return _slice_from_bounds(int(keep[0]), int(keep[-1]), n)


class AutoCropDetector():
    """nunif/utils/autocrop.py:6-203.  ``border_count_tb`` [1][H][1] and ``border_count_lr`` [1][1][W] are int32 device
    tensors, as in the reference."""

    def __init__(self, mode="black", mod=2, frame_variation_threshold=0.95):
        self.mode = _check_mode(mode)
        self.mod = mod
        self.frame_variation_threshold = frame_variation_threshold
        self.black_only = self.mode.startswith("black")
        self.reset()

    def reset(self):
        self.border_count_tb = None
        self.border_count_lr = None
        self.frame_count = 0

    def update(self, frame):
        """Add the bar masks of a CHW frame or of each frame of a BCHW batch to the device counts (no host synchronisation)."""
        if frame.ndim not in (3, 4):
            raise ValueError(f"unsupported ndim {frame.ndim}")
        H, W = frame.shape[-2:]
        for name, on, shape in (("border_count_tb", self.mode in _TB, (1, H, 1)), ("border_count_lr", self.mode in _LR, (1, 1, W))):
            if not on:
                continue
            cur = getattr(self, name)
            if cur is None:
                setattr(self, name, torch.zeros(shape, dtype=torch.int32, device=frame.device))
            elif tuple(cur.shape) != shape:
                raise ValueError(f"frame size {H}x{W} differs from the first frame's")
        _run(frame, self.mode, self.border_count_tb, self.border_count_lr)
        self.frame_count += 1 if frame.ndim == 3 else frame.shape[0]

    def get_crop(self, frame_variation_threshold=None):
        """(slice_tb, slice_lr): lines that are bars in at least ``frame_variation_threshold`` of the frames are cropped."""
        frame_variation_threshold = frame_variation_threshold or self.frame_variation_threshold
        if self.frame_count == 0:
            return slice(None), slice(None)
        ctb, clr = self.border_count_tb, self.border_count_lr
        H = ctb.shape[1] if ctb is not None else 1
        W = clr.shape[2] if clr is not None else 1
        b = _bounds(ctb, clr, H, W, self.frame_count, frame_variation_threshold)
        slice_tb = self.apply_mod(_slice_from_bounds(b[0], b[1], H), self.mod) if ctb is not None else slice(None)
        slice_lr = self.apply_mod(_slice_from_bounds(b[2], b[3], W), self.mod) if clr is not None else slice(None)
        return slice_tb, slice_lr

    @classmethod
    def detect(cls, frame, mode="black", mod=2):
        """The crop slices of one CHW frame (one synchronisation)."""
        mode = _check_mode(mode)
        if frame.ndim != 3:
            raise ValueError(f"detect takes one CHW frame, got ndim {frame.ndim}")
        H, W = frame.shape[-2:]
        ctb = torch.zeros(H, dtype=torch.int32, device=frame.device) if mode in _TB else None
        clr = torch.zeros(W, dtype=torch.int32, device=frame.device) if mode in _LR else None
        _run(frame, mode, ctb, clr)
        b = _bounds(ctb, clr, H, W, 1, 1.0)
        slice_tb = cls.apply_mod(_slice_from_bounds(b[0], b[1], H), mod) if ctb is not None else slice(None)
        slice_lr = cls.apply_mod(_slice_from_bounds(b[2], b[3], W), mod) if clr is not None else slice(None)
        return slice_tb, slice_lr

    @staticmethod
    def apply_mod(slice_value, mod):
        """Round a crop inwards to multiples of ``mod``: start up, stop down."""
        start, stop = slice_value.start, slice_value.stop
        if start is not None and start % mod != 0:
            start += mod - start % mod
        if stop is not None and stop % mod != 0:
            stop -= stop % mod
        return slice(start, stop)

    @classmethod
    def detect_tb(cls, x, black_only):
        """Per-row bar mask of a CHW / BCHW frame: bool [1][H][1] / [B][1][H][1]."""
        m = _run(x, "black_tb" if black_only else "flat_tb", masks=True)[0]
        return m.bool().view(*x.shape[:-3], 1, x.shape[-2], 1)

    @classmethod
    def detect_lr(cls, x, black_only):
        """Per-column bar mask of a CHW / BCHW frame: bool [1][1][W] / [B][1][1][W]."""
        m = _run(x, "black_lr" if black_only else "flat_lr", masks=True)[1]
        return m.bool().view(*x.shape[:-3], 1, 1, x.shape[-1])

    @classmethod
    def mask_to_slice_tb(cls, mask):
        assert mask.ndim == 3 and mask.shape[0] == 1 and mask.shape[2] == 1
        return _mask_slice(mask, mask.shape[1])

    @classmethod
    def mask_to_slice_lr(cls, mask):
        assert mask.ndim == 3 and mask.shape[0] == 1 and mask.shape[1] == 1
        return _mask_slice(mask, mask.shape[2])


def autocrop_analyze_video(video_file, *args, **kwargs):
    raise NotImplementedError("autocrop_analyze_video decodes with PyAV, which the engine does not use: feed the sampled "
                              "frames to AutoCropDetector.update and call get_crop()")


class AutoCrop():
    """nunif/utils/autocrop.py:206-343: crop a frame to the detected slices and pad it back."""

    def __init__(self, slice_h, slice_w, pad, pad_value, crop_range, uncrop_enabled):
        self.slice_h = slice_h
        self.slice_w = slice_w
        self.pad = pad
        self.crop_range = crop_range
        self.pad_value = pad_value
        self.uncrop_enabled = uncrop_enabled

    def get_slice(self):
        return self.slice_h, self.slice_w

    def get_pad(self):
        return self.pad

    def get_crop(self):
        return self.crop_range

    @staticmethod
    def calc_pad(slice_h, slice_w, H, W):
        """(left, right, top, bottom) that restores an H x W frame."""
        top, bottom, _ = slice_h.indices(H)
        left, right, _ = slice_w.indices(W)
        return (left, max(0, W - right), top, max(0, H - bottom))

    @staticmethod
    def calc_crop(slice_h, slice_w, H, W):
        """(x, y, width, height) of the kept region, None when it is the whole frame."""
        top, bottom, _ = slice_h.indices(H)
        left, right, _ = slice_w.indices(W)
        height = H - (top + max(0, H - bottom))
        width = W - (left + max(0, W - right))
        if top == 0 and left == 0 and height == H and width == W:
            return None
        return (left, top, width, height)

    @classmethod
    def from_image(cls, frame, mode="black", mod=2, pad_value=0, uncrop_enabled=True):
        if frame.ndim == 4:
            assert frame.shape[0] == 1, "batch size > 1 is not supported"
            frame = frame.squeeze(0)
        H, W = frame.shape[-2:]
        slice_h, slice_w = AutoCropDetector.detect(frame, mode=mode, mod=mod)
        return cls(slice_h=slice_h, slice_w=slice_w, pad=cls.calc_pad(slice_h, slice_w, H, W), pad_value=pad_value,
                   crop_range=cls.calc_crop(slice_h, slice_w, H, W), uncrop_enabled=uncrop_enabled)

    @classmethod
    def from_video_file(cls, video_file, *args, **kwargs):
        raise NotImplementedError("AutoCrop.from_video_file decodes with PyAV, which the engine does not use: feed the sampled "
                                  "frames to AutoCropDetector.update and build AutoCrop from get_crop() with calc_pad / calc_crop")

    def crop(self, frame):
        if frame.ndim == 3:
            return frame[:, self.slice_h, self.slice_w]
        if frame.ndim == 4:
            return frame[:, :, self.slice_h, self.slice_w]
        raise ValueError(f"ndim={frame.ndim} is not supported")

    def uncrop(self, frame):
        if not self.uncrop_enabled:
            return frame
        left, right, top, bottom = self.pad
        return _pad(frame, left, top, right, bottom, value=self.pad_value)


class AutoCropDummy():
    """No crop: what process_image uses without --autocrop."""

    def crop(self, frame):
        return frame

    def uncrop(self, frame):
        return frame
