"""CPU restatement of iw3's NULL depth model (iw3/null_depth_model.py): NullDepth.forward (:17-21) and
NullDepthModel.infer (:31-49), plus the seeded cases of tests/golden/null_depth.npz (oracle/gen_golden_null_depth.py).

The forward is the reference's two torch ops; on the CPU they are the reference's own evaluation, so the golden, made by
the real reference, is reproduced bit for bit.  On CUDA the same two ops are ATen's GPU kernels, the composition the
engine's nb200_null_depth is compared with on the same GPU.

On the CPU the last bits of ATen's bilinear resize depend on how many threads split the work, so the golden is made, and
restated here, with one intra-op thread."""
import contextlib
import hashlib

import numpy as np
import torch
import torch.nn.functional as F

from oracle import iw3 as oiw

DEFAULT_RESOLUTION = 392

# (name, B, H, W, resolution) of the golden cases; resolution None is the reference's default, 392
CASES = [
    ("land_1080p", 1, 1080, 1920, None),      # landscape, downscaled in both directions
    ("port_720p", 3, 1280, 720, 518),         # portrait
    ("odd", 3, 487, 731, 512),                # odd sizes
    ("small", 1, 120, 200, 392),              # smaller than R: the resize upscales
    ("mixed", 1, 270, 481, 518),              # upscaled vertically, downscaled horizontally
    ("square", 3, 392, 392, 392),             # already R x R: ATen copies
]
VARIANTS = [(tta, dil) for tta in (0, 1) for dil in (0, 2)]     # infer(tta=bool(tta), edge_dilation=dil)


def frames(case):
    """The seeded B,3,H,W fp32 frames in [0, 1) of a golden case."""
    seed = 1000 + [c[0] for c in CASES].index(case[0])
    _, B, H, W, _ = case
    return torch.rand((B, 3, H, W), generator=torch.Generator().manual_seed(seed))


def crops(y):
    """The parts of a B,1,R,R output the golden keeps: two 8 x 8 corners, the middle row and the middle column."""
    R = y.shape[-1]
    return [y[..., :8, :8], y[..., -8:, -8:], y[..., R // 2, :], y[..., :, R // 2]]


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


@contextlib.contextmanager
def one_thread():
    n = torch.get_num_threads()
    torch.set_num_threads(1)
    try:
        yield
    finally:
        torch.set_num_threads(n)


def null_depth(x, resolution=None):
    """NullDepth.forward: B,3,H,W -> B,1,R,R."""
    R = DEFAULT_RESOLUTION if resolution is None else resolution
    with one_thread():
        x = F.interpolate(x, size=(R, R), mode="bilinear")
        return x.mean(dim=1, keepdim=True)


def infer(x, resolution=None, tta=False, edge_dilation=0):
    """NullDepthModel.infer: 3,H,W or B,3,H,W; the TTA averages the model with itself (no flip); then dilate_edge."""
    batch = x.ndim != 3
    if not batch:
        x = x.unsqueeze(0)
    with one_thread():
        y = (null_depth(x, resolution) + null_depth(x, resolution)) * 0.5 if tta else null_depth(x, resolution)
        if oiw.edge_dilation_parse(edge_dilation) != (0, 0):
            y = oiw.dilate_edge(y, edge_dilation)
    return y if batch else y.squeeze(0)
