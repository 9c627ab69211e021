"""CPU restatement of the per-frame steps of iw3's depth export and import (iw3/utils.py:1323-1328, :1378-1382,
:1400-1421, :1717-1720, :1907-1908; iw3/base_depth_model.py:203-204, :225-232) in plain torch ops."""
import numpy as np
import torch
import torch.nn.functional as F

from . import iw3 as oiw
from .depth_scaler import EMAMinMaxScaler


def export_frame(depth, mapper_fn=None, size=None, align_corners=True):
    """normalised depth (1,h,w) -> uint16 (h,w) or ``size``: mapper, antialiased bilinear fit, clamp, 0xffff * d."""
    if mapper_fn is not None:
        depth = mapper_fn(depth)
    if size is not None:
        depth = F.interpolate(depth.unsqueeze(0), size=tuple(size), mode="bilinear", antialias=True,
                              align_corners=align_corners).squeeze(0)
    return (0xffff * torch.clamp(depth, 0, 1)).to(torch.uint16).squeeze(0)


def import_frame(depth_map, depth_range=None):
    """A decoded map (uint16 (H,W), uint8 (H,W) or (H,W,C)) -> fp32 (1,H,W) as load_depth computes it."""
    d = torch.from_numpy(np.asarray(depth_map).astype(np.float32))
    d = d.unsqueeze(0) if d.ndim == 2 else d.permute(2, 0, 1)
    d = torch.clamp(d / 0xffff, 0, 1)
    if d.shape[0] != 1:
        d = torch.mean(d, dim=0, keepdim=True)
    if depth_range is not None:
        d = d * (depth_range[1] - depth_range[0]) + depth_range[0]
    return d


def export_video_frames(depths, scene_end, decay, buffer_size, mapper_fn=None, sizes=None):
    """The depth side of the video export callback over a sequence: raw depths (1,h,w) through the EMA min/max
    normaliser, flushed and reset after each scene_end frame and at the end, then export_frame with the TF.resize fit
    (align_corners=False) to sizes[i].  Returns (frame index, uint16 map) in emission order."""
    scaler = EMAMinMaxScaler(decay=decay, buffer_size=buffer_size)
    pending, out = [], []

    def emit(frames):
        for d in frames:
            d = torch.from_numpy(np.asarray(d))
            i = pending.pop(0)
            out.append((i, export_frame(d, mapper_fn, sizes[i] if sizes is not None else None, align_corners=False)))

    for i, (d, end) in enumerate(zip(depths, scene_end)):
        pending.append(i)
        y = scaler.update(d.numpy())
        emit([y] if y is not None else [])
        if end:
            emit(scaler.flush())
    emit(scaler.flush())
    return out


def config_video_batch(x, depths, edge_dilation, skip_edge_dilation, mapper_fn, divergence, convergence):
    """process_config_video's batch_callback (:1716-1738) for the forward_fill warp and the full-SBS layout: the inverted
    edge dilation of the imported depths (unless the export dilated them), the mapper, the warp, the SBS compose.
    x (B,3,H,W), depths (B,1,H,W) -> (B,3,H,2W)."""
    if not skip_edge_dilation and any(v != 0 for v in oiw.edge_dilation_parse(edge_dilation)):
        depths = -oiw.dilate_edge(-depths, edge_dilation)
    if mapper_fn is not None:
        depths = mapper_fn(depths)
    left, right = oiw.forward_warp(x, depths, divergence, convergence, fill=True, width_base=False)
    return oiw.sbs(left, right)
