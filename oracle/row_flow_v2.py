"""ORACLE (test infrastructure only - never imported by nunif_b200/): CPU/torch restatement of `sbs.row_flow_v2`
(iw3/models/row_flow_v2.py:10-86) in delta_output mode, of backward_warp with the reference's operand types, and of the drivers
apply_divergence_nn_LR for a non-symmetric delta network (iw3/backward_warp.py:124-232) and apply_divergence_nn_symmetric
(:344-379, row_flow_v3_sym).

Pinned against the real reference modules (oracle/gen_golden_row_flow_v2.py -> tests/golden/row_flow_v2.npz).
Functional style (state_dict in); the networks are passed to the drivers as ``delta_fn(x) -> B,1,h,w``.
"""
import torch
import torch.nn.functional as F
from .row_flow import make_input

def row_flow_v2_delta(sd, x):
    """RowFlowV2._forward_delta_only (iw3/models/row_flow_v2.py:43-47,80-86): x B,3,H,W -> delta B,1,H,W (the x component),
    with the reference's pre_pad, inner replicate pads and crop.  Under CUDA autocast the result is fp16, as in the reference."""
    def conv(t, key, pad=None):
        if pad is not None:
            t = F.pad(t, pad, mode="replicate")
        return F.conv2d(t, sd[key + ".weight"], sd[key + ".bias"])
    x = F.pad(x, (28,) * 4, mode="replicate")
    f = F.relu(conv(x, "feature.0", (1, 1, 0, 0)))
    non_overlap = conv(f, "non_overlap")
    r = F.relu(conv(f, "overlap_residual.0", (4, 4, 0, 0)))
    r = F.relu(conv(r, "overlap_residual.2", (4, 4, 0, 0)))
    r = F.relu(conv(r, "overlap_residual.4", (4, 4, 0, 0)))
    r = conv(r, "overlap_residual.6", (1, 1, 1, 1))
    return (non_overlap + r)[:, :, 28:-28, 28:-28]


def backward_warp(c, delta, delta_scale):
    """backward_warp(c, grid, delta, delta_scale) (backward_warp.py:67-83) with the reference's types: an fp16 delta makes
    `delta * delta_scale` an fp16 op; delta_scale is a 0-dim fp32 tensor or a Python float."""
    B, _, h, w = delta.shape
    my, mx = torch.meshgrid(torch.linspace(-1, 1, h, device=c.device), torch.linspace(-1, 1, w, device=c.device), indexing="ij")
    grid = torch.stack([mx, my], 0).unsqueeze(0).expand(B, 2, h, w)
    grid = grid + torch.cat([delta, torch.zeros_like(delta)], dim=1) * delta_scale
    if c.shape[2:] != grid.shape[2:]:
        grid = F.interpolate(grid, size=c.shape[-2:], mode="bilinear", align_corners=True)
    z = F.grid_sample(c, grid.permute(0, 2, 3, 1), mode="bilinear", padding_mode="border", align_corners=True)
    return z.clamp(0, 1)


def apply_divergence_nn_delta_LR(delta_fn, c, depth, divergence, convergence, synthetic_view="both", steps=1,
                                 preserve_screen_border=False):
    """apply_divergence_nn_LR for a non-symmetric delta network ``delta_fn(x) -> B,1,h,w`` (backward_warp.py:124-232), with
    delta_scale a 0-dim fp32 tensor on c's device as in :201."""
    def one(shift, div):
        cc, dd = (torch.flip(c, (3,)), torch.flip(depth, (3,))) if shift > 0 else (c, depth)
        Wd = dd.shape[3]
        scale = torch.tensor(1.0 / (Wd // 2 - 1), dtype=c.dtype, device=c.device)
        dw, deltas = dd, []
        for j in range(steps):
            deltas.append(delta_fn(make_input(dw, div / steps, convergence, preserve_screen_border).to(c.device)))
            if j + 1 < steps:
                dw = backward_warp(dw, deltas[-1], scale)
        z = cc
        for delta in deltas:
            z = backward_warp(z, delta, scale)
        return torch.flip(z, (3,)) if shift > 0 else z
    if synthetic_view == "both":
        return one(-1, divergence), one(1, divergence)
    if synthetic_view == "right":
        return c, one(1, divergence * 2)
    return one(-1, divergence * 2), c


def apply_divergence_nn_symmetric(delta_fn, c, depth, divergence, convergence, synthetic_view="both"):
    """backward_warp.py:344-379: one delta with the feature values at base width W (the depth width), no flip, delta_scale a
    Python float, the left eye warped by +delta and the right eye by -delta."""
    B, _, H, W = depth.shape
    if synthetic_view != "both":
        divergence = divergence * 2
    div_pix = divergence * 0.5 * 0.01 * W
    x = torch.cat([depth, torch.full_like(depth, div_pix / 32.0), torch.full_like(depth, (-div_pix * convergence) / 32.0)], dim=1)
    delta = delta_fn(x)
    scale = 1.0 / (W // 2 - 1)
    left = backward_warp(c, delta, scale) if synthetic_view != "right" else c
    right = backward_warp(c, -delta, scale) if synthetic_view != "left" else c
    return left, right
