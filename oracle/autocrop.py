"""Oracle: the autocrop detector (nunif/utils/autocrop.py:6-207) and the frame steps of iw3's process_image around it
(iw3/utils.py:74-88 apply_rgbd, :247-271 preprocess_image, :490-502 debug_depth_image) (TEST INFRASTRUCTURE).

A torch restatement that runs on whatever device its inputs are on: on the CPU it is pinned to the real reference by
oracle/gen_golden_autocrop.py (tests/golden/autocrop.npz); on the GPU it is what ATen's CUDA kernels compute, which the
engine's masks, medians and slices are compared with.
"""
import torch
import torch.nn.functional as F

from .mapper import mapper as _mapper

BLACK = {"black_tb", "black_lr", "black"}
TB = {"black_tb", "black", "flat_tb", "flat"}
LR = {"black_lr", "black", "flat_lr", "flat"}


def luma(x, tv_range):
    """Y of a CHW / BCHW frame, [.., 1, H, W]; clamped to the TV range in the black modes."""
    r, g, b = x[..., 0:1, :, :], x[..., 1:2, :, :], x[..., 2:3, :, :]
    y = r * 0.299 + g * 0.587 + b * 0.114
    return y.clamp(min=16.0 / 255.0, max=235.0 / 255.0) if tv_range else y


def line_stats(x, black_only, dim):
    """(is_bar, mean or median, max deviation or within-fraction) along ``dim`` (-1: rows, -2: columns)."""
    y = luma(x, black_only)
    if black_only:
        mean = y.mean(dim=dim, keepdim=True)
        dev = (y - mean).abs().amax(dim=dim, keepdim=True)
        return (mean <= 32.0 / 255.0) & (dev < 16 / 255.0), mean, dev
    median = y.median(dim=dim, keepdim=True).values
    within = ((y - median).abs() < 16.0 / 255.0).float().mean(dim=dim, keepdim=True)
    return within > 0.99, median, within


def detect_tb(x, black_only):
    return line_stats(x, black_only, -1)[0]


def detect_lr(x, black_only):
    return line_stats(x, black_only, -2)[0]


def mask_to_slice(mask):
    """A 1-D bar mask -> the slice of the non-bar lines (full when there are no bars or nothing else)."""
    keep = torch.nonzero(~mask.flatten()).flatten().tolist()
    n = mask.numel()
    if len(keep) in (0, n):
        return slice(None, None)
    start, stop = keep[0], keep[-1] + 1
    return slice(start if start > 0 else None, stop if stop < n else None)


def apply_mod(s, mod):
    start, stop = s.start, s.stop
    if start is not None and start % mod:
        start += mod - start % mod
    if stop is not None and stop % mod:
        stop -= stop % mod
    return slice(start, stop)


def _slices(mask_tb, mask_lr, mode, mod):
    s_tb = apply_mod(mask_to_slice(mask_tb), mod) if mode in TB else slice(None)
    s_lr = apply_mod(mask_to_slice(mask_lr), mod) if mode in LR else slice(None)
    return s_tb, s_lr


def detect(frame, mode="black", mod=2):
    """AutoCropDetector.detect for one CHW frame."""
    mode = mode.lower()
    black = mode in BLACK
    return _slices(detect_tb(frame, black) if mode in TB else None, detect_lr(frame, black) if mode in LR else None, mode, mod)


def get_crop(frames, mode="black", mod=2, threshold=0.95):
    """AutoCropDetector.update over ``frames`` (CHW each), then get_crop(); also returns the int32 counts."""
    mode = mode.lower()
    black = mode in BLACK
    ctb = sum(detect_tb(f, black).int() for f in frames) if mode in TB else None
    clr = sum(detect_lr(f, black).int() for f in frames) if mode in LR else None
    n = len(frames)
    if n == 0:
        return (slice(None), slice(None)), ctb, clr
    return _slices(ctb / n >= threshold if ctb is not None else None, clr / n >= threshold if clr is not None else None,
                   mode, mod), ctb, clr


def calc_pad(slice_h, slice_w, H, W):
    h0, h1, _ = slice_h.indices(H)
    w0, w1, _ = slice_w.indices(W)
    return (w0, max(0, W - w1), h0, max(0, H - h1))


def calc_crop(slice_h, slice_w, H, W):
    h0, h1, _ = slice_h.indices(H)
    w0, w1, _ = slice_w.indices(W)
    height, width = H - (h0 + max(0, H - h1)), W - (w0 + max(0, W - w1))
    return None if (h0, w0, height, width) == (0, 0, H, W) else (w0, h0, width, height)


def crop(x, slices):
    return x[..., slices[0], slices[1]]


def uncrop(x, pad, value=0):
    return F.pad(x, pad, mode="constant", value=value)


def preprocess_image(x, rotate_left=False, rotate_right=False, max_output_height=None):
    if rotate_left:
        x = torch.rot90(x, 1, (-2, -1))
    elif rotate_right:
        x = torch.rot90(x, 3, (-2, -1))
    h, w = x.shape[-2:]
    new_h, new_w = h, w
    if max_output_height is not None and h > max_output_height:
        new_w = int(max_output_height / h * w)
        new_h = max_output_height
    if (new_h, new_w) != (h, w):
        new_h -= new_h % 2
        new_w -= new_w % 2
        x4 = x if x.ndim == 4 else x.unsqueeze(0)
        x4 = F.interpolate(x4, (new_h, new_w), mode="bicubic", antialias=True, align_corners=True)
        x = (x4 if x.ndim == 4 else x4.squeeze(0)).clamp(0, 1)
    return x


def apply_rgbd(im, depth, mapper=None):
    if mapper is not None:
        depth = _mapper(depth, mapper)
    d4 = depth if depth.ndim == 4 else depth.unsqueeze(0)
    right = F.interpolate(d4, im.shape[-2:], mode="bicubic", antialias=True)
    right = right if depth.ndim == 4 else right.squeeze(0)
    return im, right.expand_as(im)


def debug_depth_image(depth, mapper):
    depth = depth.float()
    return torch.cat([depth, _mapper(depth, mapper)], dim=2).repeat((3, 1, 1))
