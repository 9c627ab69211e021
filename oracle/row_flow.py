"""ORACLE (test infrastructure only - never imported by nunif_b200/): CPU/torch restatement of the learned stereo
warp `sbs.row_flow_v3` (iw3/models/row_flow_v3.py:14-128) and of its driver apply_divergence_nn_LR /
apply_divergence_nn_delta (iw3/backward_warp.py:124-232) incl. steps > 1 and preserve_screen_border
(tests/golden/row_flow_steps.npz).

Pinned against the real reference model (create_model("sbs.row_flow_v3") with a seeded state_dict, run from
/root/reference): tests/golden/row_flow.npz (oracle/gen_golden.py row_flow).  Functional style (state_dict in).
"""
import torch
import torch.nn.functional as F
from .wa_block import wa_block

OFFSET = 32
MOD = 12
PACK = 8


def row_flow_delta(sd, x):
    """RowFlowV3._forward (row_flow_v3.py:57-68): x B,3,H,W (depth, divergence feature, convergence feature) -> delta B,1,H,W."""
    H, W = x.shape[2:]
    pad1 = MOD * PACK - W % (MOD * PACK)
    pad2 = MOD - H % MOD
    x = F.pad(x, (0, pad1, 0, pad2), mode="replicate")
    B, C, Hp, Wp = x.shape
    x = x.reshape(B, C, Hp, 1, Wp // PACK, PACK).permute(0, 1, 3, 5, 2, 4).reshape(B, C * PACK, Hp, Wp // PACK)   # pixel_unshuffle (1, 8)
    x = F.conv2d(x, sd["blocks.0.weight"], sd["blocks.0.bias"])
    x = wa_block(sd, "blocks.1.", x, 4, 2, False, act=True)
    x = wa_block(sd, "blocks.2.", x, 3, 2, False, act=True)
    C = x.shape[1]
    x = x.reshape(B, C // PACK, 1, PACK, Hp, Wp // PACK).permute(0, 1, 4, 2, 5, 3).reshape(B, C // PACK, Hp, Wp)  # pixel_shuffle (1, 8)
    x = x[:, :, :H, :W]
    x = F.pad(x, (1, 1, 1, 1), mode="replicate")
    return F.conv2d(x, sd["last_layer.1.weight"], sd["last_layer.1.bias"])


def make_input(depth, divergence, convergence, preserve_screen_border=False):
    """make_input_tensor(None, depth, ...) for a batch (backward_warp.py:8-63), image_width = max(H, W)."""
    B, _, H, W = depth.shape
    base = max(H, W)
    div_pix = divergence * 0.5 * 0.01 * base
    df, cf = torch.full_like(depth, div_pix / 32.0), torch.full_like(depth, (-div_pix * convergence) / 32.0)
    if preserve_screen_border:                               # :33-47: the parallax fades to zero towards the left / right edges
        bp = round(divergence * 0.75 * 0.01 * base * (W / base))
        if bp > 0:
            wl, wr = torch.linspace(0.0, 1.0, bp), torch.linspace(1.0, 0.0, bp)
            for f in (df, cf):
                f[..., :bp] = wl * f[..., :bp]
                f[..., -bp:] = wr * f[..., -bp:]
    return torch.cat([depth, df, cf], dim=1)


def warp_delta(c, delta, W_depth):
    """backward_warp(c, grid, delta, delta_scale) (backward_warp.py:67-83) with grid = make_grid at the depth size."""
    B, _, h, w = delta.shape
    my, mx = torch.meshgrid(torch.linspace(-1, 1, h), torch.linspace(-1, 1, w), indexing="ij")
    grid = torch.stack([mx, my], 0).unsqueeze(0).expand(B, 2, h, w).to(c.dtype)
    d2 = torch.cat([delta.float(), torch.zeros_like(delta.float())], dim=1)
    grid = grid + d2 * torch.tensor(1.0 / (W_depth // 2 - 1), dtype=c.dtype)
    if c.shape[2:] != grid.shape[2:]:
        grid = F.interpolate(grid, size=c.shape[-2:], mode="bilinear", align_corners=True)
    z = F.grid_sample(c, grid.permute(0, 2, 3, 1), mode="bilinear", padding_mode="border", align_corners=True)
    return z.clamp(0, 1)


def apply_divergence_nn_LR(sd, c, depth, divergence, convergence, synthetic_view="both", steps=1, preserve_screen_border=False):
    """backward_warp.py:124-232: the right eye is the left-eye procedure on the mirrored frame; with steps > 1 the divergence is
    applied in `steps` equal parts, the DEPTH being re-warped by each part's delta before the next (:205-221), and the image is
    warped by the deltas one after the other (:223-226)."""
    def one(shift, div):
        cc, dd = (torch.flip(c, (3,)), torch.flip(depth, (3,))) if shift > 0 else (c, depth)
        Wd = dd.shape[3]
        dw, deltas = dd, []
        for j in range(steps):
            deltas.append(row_flow_delta(sd, make_input(dw, div / steps, convergence, preserve_screen_border)))
            if j + 1 < steps:
                dw = warp_delta(dw, deltas[-1], Wd)
        z = cc
        for delta in deltas:
            z = warp_delta(z, delta, Wd)
        return torch.flip(z, (3,)) if shift > 0 else z
    if synthetic_view == "both":
        return one(-1, divergence), one(1, divergence)
    if synthetic_view == "right":
        return c, one(1, divergence * 2)
    return one(-1, divergence * 2), c
