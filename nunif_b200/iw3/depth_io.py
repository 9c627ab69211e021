"""Depth maps to and from the 16-bit files of ``--export`` on the engine.

``export_depth_u16`` is the device side of an export (iw3/utils.py:1323-1328 images, :1378-1382 video, then
``BaseDepthModel.save_normalized_depth``, iw3/base_depth_model.py:203-204): mapper, fit resize, clamp and the 16-bit
quantisation in one kernel, so the host receives the uint16 map it encodes.  ``import_depth`` is ``load_depth``'s
arithmetic (:225-232) on a decoded map uploaded as is."""
import ctypes

import numpy as np
import torch

from .. import _lib
from ._common import prep
from .mapper import descriptor


def export_depth_u16(depth, mapper=None, size=None, align_corners=True):
    """depth: normalised CHW (1,h,w) or BCHW (B,1,h,w) on the GPU -> uint16 (h,w) or (B,h,w) (or ``size``).

    ``mapper``: a mapper name applied to the source pixels first (None or "none": identity).  ``size``: (H, W) of the
    antialiased bilinear fit, ``align_corners=True`` as ``F.interpolate`` in ``export_images``, False as ``TF.resize``
    in the video export."""
    d = prep(depth, "depth")
    batched = d.ndim == 4
    if not batched:
        d = d.unsqueeze(0)
    B, C, h, w = d.shape
    if C != 1:
        raise ValueError(f"depth must have one channel, got {C}")
    desc = descriptor(mapper) if mapper is not None else None
    H, W = (int(size[0]), int(size[1])) if size is not None else (h, w)
    out = torch.empty((B, H, W), dtype=torch.uint16, device=d.device)
    with torch.cuda.device(d.device):
        _lib.check(_lib.lib().nb200_depth_export_u16(_lib.ptr(d), B, h, w, ctypes.byref(desc) if desc is not None else None,
                                                     1 if size is not None else 0, H, W, 1 if align_corners else 0,
                                                     _lib.ptr(out), _lib.stream_ptr(d.device)))
    return out if batched else out.squeeze(0)


# element type of a decoded map -> NB200_DEPTH_* (include/nunif_b200.h)
_DTYPES = {np.dtype(np.uint8): 1, np.dtype(np.uint16): 2, np.dtype(np.int32): 3, np.dtype(np.float32): 4}


def import_depth(depth_map, device, depth_range=None):
    """One decoded depth map (``np.asarray`` of the image: uint16 / int32 / float32 (H,W), or uint8 (H,W) / (H,W,C) with
    C <= 4) -> fp32 (1,H,W) on ``device``.  ``depth_range``: (iw3_min_depth_value, iw3_max_depth_value) or None."""
    a = np.ascontiguousarray(depth_map)
    dtype = _DTYPES.get(a.dtype)
    if dtype is None:
        raise NotImplementedError(f"depth maps of dtype {a.dtype}: the engine imports 8-, 16- and 32-bit integer and "
                                  "32-bit float maps")
    if a.ndim not in (2, 3):
        raise ValueError(f"a depth map is (H, W) or (H, W, C), got shape {a.shape}")
    H, W = a.shape[:2]
    C = a.shape[2] if a.ndim == 3 else 1
    src = torch.from_numpy(a).to(device)
    out = torch.empty((1, H, W), dtype=torch.float32, device=src.device)
    lo, hi = depth_range if depth_range is not None else (0.0, 0.0)
    with torch.cuda.device(src.device):
        _lib.check(_lib.lib().nb200_depth_import(_lib.ptr(src), dtype, C, 1, H, W, float(lo), float(hi),
                                                 1 if depth_range is not None else 0, _lib.ptr(out),
                                                 _lib.stream_ptr(src.device)))
    return out
