"""ORACLE (test infrastructure only - never imported by nunif_b200/): CPU/torch restatement of iw3's `mlbw_l2_inpaint` in image mode
and of `--method mask_mlbw_l2`:
  - the hole_mask head of `sbs.mlbw` (iw3/models/mlbw.py:70-74,104-109,232-240; MLBW(num_layers=2, base_dim=32, hole_mask=True)),
  - postprocess_hole_mask (iw3/backward_warp.py:382-393) with closing (iw3/dilation.py:41-64),
  - apply_divergence_nn_delta_weight with return_mask and the hole fill (backward_warp.py:262-341),
  - MLBWInpaintImage.forward (iw3/mlbw_inpaint.py:18-151) on oracle.light_inpaint's network.
Pinned to the real reference by tests/golden/mask_mlbw.npz (oracle/gen_golden_mask_mlbw.py).  Under ``torch.autocast`` on a GPU
the networks follow the reference's CUDA path; the backward warp runs on the CPU in fp32 (oracle.mlbw's warp is CPU code and has
no autocast-dependent arithmetic).
"""
import torch
import torch.nn.functional as F

from . import light_inpaint as oli
from .mlbw import MOD, PACK, _warp
from .row_flow import make_input
from .wa_block import wa_block

THRESHOLD = 0.15          # MASK_MLBW_THRESHOLD (mlbw_inpaint.py:18) and the hole fill (backward_warp.py:337)
NUM_LAYERS = 2


def mask_mlbw_delta(sd, x):
    """MLBW(hole_mask=True)._forward_delta_only in eval mode: x B,3,H,W -> (delta B,2,H,W ; layer_weight B,2,H,W softmax over the
    layers ; hole logits B,1,H,W), lv1_out's outputs in the order [delta x L | layer-weight logits x L | hole logit]."""
    H, W = x.shape[2:]
    pad_w, pad_h = MOD * PACK - W % (MOD * PACK), MOD - H % MOD
    pw1, ph1 = pad_w // 2, pad_h // 2
    pw2, ph2 = pad_w - pw1, pad_h - ph1
    x = F.pad(x, (pw1, pw2, ph1, ph2), mode="replicate")
    x1 = F.leaky_relu(F.conv2d(F.pad(x, (4, 4, 0, 0), mode="replicate"), sd["lv1_in.1.weight"], sd["lv1_in.1.bias"]), 0.2)
    B, C1, Hp, Wp = x1.shape
    t = x1.reshape(B, C1, Hp, 1, Wp // PACK, PACK).permute(0, 1, 3, 5, 2, 4).reshape(B, C1 * PACK, Hp, Wp // PACK)
    for i, shift in enumerate((True, False, True, False)):
        t = wa_block(sd, f"lv2.{i}.", t, 4, NUM_LAYERS, shift, act=False)
    C = t.shape[1]
    t = t.reshape(B, C // PACK, 1, PACK, Hp, Wp // PACK).permute(0, 1, 4, 2, 5, 3).reshape(B, C // PACK, Hp, Wp)
    y = F.conv2d(F.pad(t + x1, (4, 4, 0, 0), mode="replicate"), sd["lv1_out.1.weight"], sd["lv1_out.1.bias"])
    y = y[:, :, ph1:Hp - ph2, pw1:Wp - pw2]
    delta, lw = y[:, :2 * NUM_LAYERS].chunk(2, dim=1)
    return delta.float(), F.softmax(lw.float(), dim=1), y[:, 2 * NUM_LAYERS:].float()


def closing(logits):
    """closing(mask, n_iter=1) (dilation.py:57-64): 3x3 max pool, then 3x3 min pool, both with -inf padding."""
    m = F.max_pool2d(logits.float(), 3, stride=1, padding=1)
    return -F.max_pool2d(-m, 3, stride=1, padding=1)


def hole_mask_stages(logits, target_size, threshold=THRESHOLD):
    """The first three steps of postprocess_hole_mask: (closed logits, sigmoid at target_size, sigmoid > threshold)."""
    c = closing(logits)
    z = c
    if tuple(target_size) != tuple(c.shape[-2:]):
        z = F.interpolate(c, size=tuple(target_size), mode="bilinear", align_corners=True, antialias=False)
    s = torch.sigmoid(z)
    return c, s, s > threshold


def postprocess_hole_mask(logits, target_size, threshold=THRESHOLD, inner_dilation=0, outer_dilation=0):
    """backward_warp.py:382-393 -> bool B,1,H,W."""
    bw = logits.shape[-1]
    m = hole_mask_stages(logits, target_size, threshold)[2]
    m = oli.dilate_inner(m, n_iter=inner_dilation, base_width=bw)
    return oli.dilate_outer(m, n_iter=outer_dilation, base_width=bw)


def apply_divergence_mask_mlbw(sd, c, depth, divergence, convergence, shift, preserve_screen_border=False, return_mask=False):
    """apply_divergence_nn_delta_weight (backward_warp.py:262-341) for the hole_mask model."""
    dev = c.device
    if shift > 0:
        c, depth = torch.flip(c, (3,)), torch.flip(depth, (3,))
    x = make_input(depth.float().cpu(), divergence, convergence, preserve_screen_border).to(dev)
    delta, lw, logits = mask_mlbw_delta(sd, x)
    if c.shape[2:] != lw.shape[2:]:
        lw = F.interpolate(lw, size=c.shape[-2:], mode="bilinear", align_corners=True, antialias=True)
    z = torch.zeros_like(c, dtype=torch.float32)
    for i in range(NUM_LAYERS):
        z = z + _warp(c.float().cpu(), delta[:, i:i + 1].float().cpu(), depth.shape[3]).to(dev) * lw[:, i:i + 1].float()
    z = z.clamp(0, 1)
    if shift > 0:
        z, logits = z.flip((3,)), logits.flip((3,))
    if return_mask:
        return z, logits
    return z * (1 - postprocess_hole_mask(logits, c.shape[-2:], THRESHOLD).float())


def apply_divergence_nn_LR(sd, c, depth, divergence, convergence, synthetic_view="both", preserve_screen_border=False):
    """apply_divergence_nn_LR (backward_warp.py:124-160) with the mask_mlbw_l2 model: `--method mask_mlbw_l2`."""
    kw = dict(preserve_screen_border=preserve_screen_border)
    if synthetic_view == "both":
        return (apply_divergence_mask_mlbw(sd, c, depth, divergence, convergence, -1, **kw),
                apply_divergence_mask_mlbw(sd, c, depth, divergence, convergence, 1, **kw))
    if synthetic_view == "right":
        return c, apply_divergence_mask_mlbw(sd, c, depth, divergence * 2, convergence, 1, **kw)
    return apply_divergence_mask_mlbw(sd, c, depth, divergence * 2, convergence, -1, **kw), c


def mlbw_inpaint(sd_inpaint, sd_mask, x, depth, divergence, convergence, synthetic_view="both", inner_dilation=0, outer_dilation=0,
                 max_width=None, preserve_screen_border=False):
    """MLBWInpaintImage.forward (mlbw_inpaint.py:112-151) with forward_left / forward_right (:21-34)."""
    x = oli.resize_max_width(x, max_width)
    kw = dict(preserve_screen_border=preserve_screen_border, return_mask=True)
    div = divergence if synthetic_view == "both" else divergence * 2
    left = right = x
    if synthetic_view in ("both", "left"):
        left, lm = apply_divergence_mask_mlbw(sd_mask, x, depth, div, convergence, -1, **kw)
        m = postprocess_hole_mask(lm.flip(-1), left.shape[-2:], THRESHOLD, inner_dilation, outer_dilation)
        left = oli.infer(sd_inpaint, left.flip(-1), m).flip(-1)
    if synthetic_view in ("both", "right"):
        right, rm = apply_divergence_mask_mlbw(sd_mask, x, depth, div, convergence, 1, **kw)
        m = postprocess_hole_mask(rm, right.shape[-2:], THRESHOLD, inner_dilation, outer_dilation)
        right = oli.infer(sd_inpaint, right, m)
    return left, right
