"""ORACLE (test infrastructure only - never imported by nunif_b200/): CPU/torch restatement of `iw3.depth_aa`
(iw3/models/depth_aa.py:11-87), the learned depth anti-aliasing filter applied after Depth-Anything when
`depth_aa=True` (iw3/depth_anything_model.py:153-154).  Its three window-attention blocks (the first and the last
shifted) are oracle/wa_block.py's.

SURVEY.md 8f rank 4 "next" row: the engine raises NotImplementedError for depth_aa today; this pins the algorithm
against the real reference model (tests/golden/depth_aa.npz, oracle/gen_golden.py depth_aa) for the round that ports it.
"""
import torch
import torch.nn.functional as F
from .wa_block import wa_block


def depth_aa_forward(sd, x, clamp=True):
    """DepthAA.forward: x B,1,H,W (normalised depth) -> B,1,H,W."""
    src = x
    H, W = x.shape[2:]
    pad_w, pad_h = 16 - W % 16, 16 - H % 16
    pw1, ph1 = pad_w // 2, pad_h // 2
    pw2, ph2 = pad_w - pw1, pad_h - ph1
    x = F.pad(x, (pw1, pw2, ph1, ph2), mode="replicate")
    x = F.pixel_unshuffle(x, 2)
    x = F.conv2d(x, sd["proj_in.weight"], sd["proj_in.bias"])
    for i, shift in enumerate((True, False, True)):
        x = wa_block(sd, f"blocks.{i}.", x, 8, 2, shift, act=True)
    x = F.conv2d(x, sd["proj_out.weight"], sd["proj_out.bias"])
    x = F.pixel_shuffle(x, 2)
    x = x[:, :, ph1:x.shape[2] - ph2, pw1:x.shape[3] - pw2]
    x = src + x
    return x.clamp(0, 1) if clamp else x


def depth_aa_infer(sd, x):
    """DepthAA.infer (depth_aa.py:46-55): min/max normalise, filter without clamp, de-normalise."""
    mn, mx = x.amin(), x.amax()
    scale = mx - mn
    y = torch.nan_to_num((x - mn) / scale)
    return depth_aa_forward(sd, y, clamp=False) * scale + mn
