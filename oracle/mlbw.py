"""ORACLE (test infrastructure only - never imported by nunif_b200/): CPU/torch restatement of the multi-layer learned
stereo warp `sbs.mlbw` (iw3/models/mlbw.py:17-127,237-245; MLBW(num_layers=L, base_dim=32, small=False, hole_mask=False))
in delta_output mode and of its driver apply_divergence_nn_delta_weight (iw3/backward_warp.py:262-329, steps ignored by the
reference for this model).

SURVEY.md 8f rank 2 (second learned warp): the engine implements sbs.row_flow_v3 and raises NotImplementedError for
sbs.mlbw today; this pins the algorithm against the real reference model (tests/golden/mlbw.npz) for the round that ports it.
"""
import torch
import torch.nn.functional as F
from .row_flow import make_input
from .wa_block import wa_block

PACK = 8
MOD = 4


def mlbw_delta(sd, x, num_layers=2, small=False):
    """MLBW._forward in eval mode: x B,3,H,W -> (delta B,L,H,W ; layer_weight B,L,H,W softmax over L)."""
    H, W = x.shape[2:]
    pad_w, pad_h = MOD * PACK - W % (MOD * PACK), MOD - H % MOD
    pw1, ph1 = pad_w // 2, pad_h // 2
    pw2, ph2 = pad_w - pw1, pad_h - ph1
    x = F.pad(x, (pw1, pw2, ph1, ph2), mode="replicate")
    x1 = F.leaky_relu(F.conv2d(F.pad(x, (4, 4, 0, 0), mode="replicate"), sd["lv1_in.1.weight"], sd["lv1_in.1.bias"]), 0.2)
    B, C1, Hp, Wp = x1.shape
    t = x1.reshape(B, C1, Hp, 1, Wp // PACK, PACK).permute(0, 1, 3, 5, 2, 4).reshape(B, C1 * PACK, Hp, Wp // PACK)
    for i, shift in enumerate(((False, True), False) if small else (True, False, True, False)):       # mlbw.py:53-64
        t = wa_block(sd, f"lv2.{i}.", t, 4, num_layers, shift, act=False)
    C = t.shape[1]
    t = t.reshape(B, C // PACK, 1, PACK, Hp, Wp // PACK).permute(0, 1, 4, 2, 5, 3).reshape(B, C // PACK, Hp, Wp)
    y = F.conv2d(F.pad(t + x1, (4, 4, 0, 0), mode="replicate"), sd["lv1_out.1.weight"], sd["lv1_out.1.bias"])
    y = y[:, :, ph1:Hp - ph2, pw1:Wp - pw2]
    delta, lw = y.chunk(2, dim=1)
    return delta.float(), F.softmax(lw.float(), dim=1)


def _warp(c, delta, W_depth):
    B, _, h, w = delta.shape
    my, mx = torch.meshgrid(torch.linspace(-1, 1, h), torch.linspace(-1, 1, w), indexing="ij")
    grid = torch.stack([mx, my], 0).unsqueeze(0).expand(B, 2, h, w).to(c.dtype)
    grid = grid + torch.cat([delta, torch.zeros_like(delta)], 1) * torch.tensor(1.0 / (W_depth // 2 - 1), dtype=c.dtype)
    if c.shape[2:] != grid.shape[2:]:
        grid = F.interpolate(grid, size=c.shape[-2:], mode="bilinear", align_corners=True)
    z = F.grid_sample(c, grid.permute(0, 2, 3, 1), mode="bilinear", padding_mode="border", align_corners=True)
    return z.clamp(0, 1)   # backward_warp() clamps every layer (iw3/backward_warp.py:81-82)


def apply_divergence_mlbw(sd, c, depth, divergence, convergence, shift, num_layers=2):
    """apply_divergence_nn_delta_weight (backward_warp.py:262-329) without hole mask."""
    if shift > 0:
        c, depth = torch.flip(c, (3,)), torch.flip(depth, (3,))
    delta, lw = mlbw_delta(sd, make_input(depth, divergence, convergence), num_layers)
    if c.shape[2:] != lw.shape[2:]:
        lw = F.interpolate(lw, size=c.shape[-2:], mode="bilinear", align_corners=True, antialias=True)
    z = torch.zeros_like(c)
    for i in range(num_layers):
        z = z + _warp(c, delta[:, i:i + 1], depth.shape[3]) * lw[:, i:i + 1]
    z = z.clamp(0, 1)
    return torch.flip(z, (3,)) if shift > 0 else z
