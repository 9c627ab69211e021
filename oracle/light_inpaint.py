"""Oracle: iw3's image-mode `forward_inpaint` (TEST INFRASTRUCTURE).

Functional fp32 restatement of
  - iw3/models/light_inpaint_v1.py:88-154 (LightInpaintV1.infer / forward, eval mode),
  - the GMLPBlock it is built from (light_inpaint_v1.py:15-49, nunif/modules/attention.py:621-693, window order
    nunif/modules/permute.py:85-127),
  - the mask operations (iw3/dilation.py:41-98,145-152) and the separable 15-tap Gaussian (nunif/modules/gaussian_filter.py),
  - the image-mode driver ForwardInpaintImage.forward (iw3/forward_inpaint.py:18-40,69-103).
Run under ``torch.autocast`` on a GPU it mimics the reference's CUDA path (the layer norms then run in fp16, as
FastLayerNorm does, nunif/modules/norm.py:78-101).
"""
import torch
import torch.nn.functional as F

from . import iw3 as oiw3


# ---------------------------------------------------------------------------------------------------------------------------
# masks
# ---------------------------------------------------------------------------------------------------------------------------
def mask_closing(mask):
    """dilation.py:41-64,145-152: 2x dilate 3x3 + 2x erode 3x3 (max_pool2d, implicit -inf padding), OR the input."""
    m0 = m = mask.float()
    for _ in range(2):
        m = F.max_pool2d(m, 3, stride=1, padding=1)
    for _ in range(2):
        m = -F.max_pool2d(-m, 3, stride=1, padding=1)
    return (m + m0).clamp(0, 1)


def _run_count(W, n_iter, base_width):
    return max(round(W / base_width * n_iter), 1) if base_width is not None else n_iter


def dilate_outer(mask, n_iter, base_width=None):
    """dilation.py:67-82: grow runs to the right by n pixels (right-view base)."""
    if n_iter <= 0:
        return mask
    dtype, m = mask.dtype, mask.bool()
    for _ in range(_run_count(m.shape[-1], n_iter, base_width)):
        m = m | F.pad(m, (1, 0, 0, 0))[:, :, :, :-1]
    return m.to(dtype)


def dilate_inner(mask, n_iter, base_width=None):
    """dilation.py:85-98: grow runs to the left by n pixels."""
    if n_iter <= 0:
        return mask
    dtype, m = mask.dtype, mask.bool()
    for _ in range(_run_count(m.shape[-1], n_iter, base_width)):
        m = m | F.pad(m, (0, 1, 0, 0))[:, :, :, 1:]
    return m.to(dtype)


def gaussian_kernel15():
    """get_gaussian_kernel1d(15) (gaussian_filter.py:8-19): sigma = 15 * 0.15 + 0.35."""
    x = torch.linspace(-7.0, 7.0, steps=15, dtype=torch.float32)
    k = torch.exp(-0.5 * (x / (15 * 0.15 + 0.35)).pow(2))
    return k / k.sum()


def blur15(mask):
    """SeparableGaussianFilter2d(1, 15, padding=7) (gaussian_filter.py:51-74): replicate pad, horizontal then vertical pass."""
    k = gaussian_kernel15().to(mask.device, mask.dtype)
    x = F.pad(mask, (7, 7, 7, 7), mode="replicate")
    x = F.conv2d(x, k.view(1, 1, 1, 15))
    return F.conv2d(x, k.view(1, 1, 15, 1))


def prepare_mask(mask, x):
    """LightInpaintV1.preprocess with closing=False and no dilation (light_inpaint_v1.py:88-100): the hole-zeroed frame and
    the blurred mask clamp(blur15(mask) + mask, 0, 1)."""
    mask = mask.float()
    return x * (1 - mask), torch.clamp(blur15(mask) + mask, 0, 1)


# ---------------------------------------------------------------------------------------------------------------------------
# network
# ---------------------------------------------------------------------------------------------------------------------------
def _ln(x, w):
    """FastLayerNorm without bias, eps 1e-5, over the last dim (under autocast: in the autocast dtype)."""
    if torch.is_autocast_enabled(x.device.type):
        dt = torch.get_autocast_dtype(x.device.type)
        with torch.autocast(x.device.type, enabled=False):
            return F.layer_norm(x.to(dt), (x.shape[-1],), w.to(dt), None, 1e-5)
    return F.layer_norm(x, (x.shape[-1],), w, None, 1e-5)


def _to_windows(x, ws):
    B, C, H, W = x.shape
    x = x.reshape(B, C, H // ws, ws, W // ws, ws).permute(0, 2, 4, 3, 5, 1)
    return x.reshape(B * (H // ws) * (W // ws), ws * ws, C)


def _from_windows(x, shape, ws):
    B, C, H, W = shape
    x = x.reshape(B, H // ws, W // ws, ws, ws, C).permute(0, 5, 1, 3, 2, 4)
    return x.reshape(B, C, H, W)


def _replicate_pad(x, pad):
    """replication_pad2d_naive (left, right, top, bottom)."""
    return F.pad(x, pad, mode="replicate")


def gmlp_block(sd, p, x, ws, shift):
    """GMLPBlock.forward: x + WindowGMLP2d(x) (whose GMLP adds its own shortcut), then x + GLUConvMLP(x)."""
    g = p + ".gmlp.gmlp"
    h = F.pad(x, (ws // 2,) * 4) if shift else x
    shape = h.shape
    t = _to_windows(h, ws)
    y = F.gelu(F.linear(_ln(t, sd[p + ".norm1.weight"]), sd[g + ".proj_in.weight"], sd[g + ".proj_in.bias"]))
    u, v = y.chunk(2, dim=-1)
    v = _ln(v, sd[p + ".norm2.weight"])
    v = F.conv1d(v, sd[g + ".proj_spatial.weight"], sd[g + ".proj_spatial.bias"])
    y = F.linear(u * v, sd[g + ".proj_out.weight"], sd[g + ".proj_out.bias"]) + t
    y = _from_windows(y, shape, ws)
    if shift:
        y = y[:, :, ws // 2:-(ws // 2), ws // 2:-(ws // 2)]
    x = x + y
    h = F.glu(F.conv2d(x, sd[p + ".glu_conv.w1.weight"], sd[p + ".glu_conv.w1.bias"]), dim=1)
    h = F.conv2d(_replicate_pad(h, (1, 1, 1, 1)), sd[p + ".glu_conv.w2.weight"], sd[p + ".glu_conv.w2.bias"])
    return x + h


def network(sd, x, mask):
    """LightInpaintV1.forward(x, mask, skip_i2i_offset=True) (light_inpaint_v1.py:107-154) in eval mode.
    x: the hole-zeroed frame, mask: the blurred mask (both B,C,H,W fp32)."""
    src = x
    x = (x - 0.5) / 0.5
    H, W = x.shape[2:]
    pad = (0, 64 - W % 64, 0, 64 - H % 64)        # 64, not 0, when the size is already a multiple of 64
    x, m = _replicate_pad(x, pad), _replicate_pad(mask, pad)
    x = F.leaky_relu(F.conv2d(F.pixel_unshuffle(x, 4), sd["patch.0.weight"], sd["patch.0.bias"]), 0.2)
    tok = F.pixel_unshuffle(m, 4).amax(dim=1, keepdim=True) > 0.99
    x = torch.where(tok, sd["mask_bias"].to(x.dtype), x)
    x1 = gmlp_block(sd, "enc1", x, 16, True)
    x2 = F.conv2d(x1, sd["down.weight"], sd["down.bias"], stride=2)
    for i in range(4):
        x2 = gmlp_block(sd, f"enc2.{i}", x2, 8, i % 2 == 1)
    x2 = F.pixel_shuffle(F.conv2d(x2, sd["up.weight"], sd["up.bias"]), 2)
    x = gmlp_block(sd, "dec1", x1 + x2, 16, False)
    x = F.conv2d(_replicate_pad(x, (1, 1, 1, 1)), sd["to_image.1.weight"], sd["to_image.1.bias"])
    x = F.pixel_shuffle(x, 4)[:, :, :H, :W]
    mask = mask.expand_as(src)
    return (src * (1 - mask) + x * mask).clamp(0, 1)


def infer(sd, x, mask):
    """LightInpaintV1.infer(x, mask) with the defaults forward_left / forward_right use (light_inpaint_v1.py:102-105)."""
    x, m = prepare_mask(mask, x)
    return network(sd, x, m)


# ---------------------------------------------------------------------------------------------------------------------------
# image-mode driver
# ---------------------------------------------------------------------------------------------------------------------------
def eye_mask(mask, inner_dilation, outer_dilation, base_width):
    """forward_right's mask chain (forward_inpaint.py:18-25): > 0, closing, dilate_outer, dilate_inner."""
    m = mask_closing(mask > 0)
    m = dilate_outer(m, n_iter=outer_dilation, base_width=base_width)
    return dilate_inner(m, n_iter=inner_dilation, base_width=base_width)


def forward_right(sd, eye, mask, inner_dilation, outer_dilation, base_width):
    return infer(sd, eye, eye_mask(mask, inner_dilation, outer_dilation, base_width))


def forward_left(sd, eye, mask, inner_dilation, outer_dilation, base_width):
    """forward_inpaint.py:28-40: the same chain on the mirrored eye and mask, mirrored back."""
    m = eye_mask(mask.flip(-1), inner_dilation, outer_dilation, base_width)
    return infer(sd, eye.flip(-1), m).flip(-1)


def resize_max_width(x, max_width):
    """forward_inpaint.py:74-81."""
    if max_width is None or x.shape[-1] <= max_width:
        return x
    if max_width % 2 != 0:
        max_width += 1
    new_h = int((max_width / x.shape[-1]) * x.shape[-2])
    if new_h % 2 != 0:
        new_h += 1
    return F.interpolate(x, size=(new_h, max_width), mode="bilinear", antialias=True, align_corners=False)


def forward_inpaint(sd, x, depth, divergence, convergence, synthetic_view="both", inner_dilation=0, outer_dilation=0,
                    max_width=None):
    """ForwardInpaintImage.forward (forward_inpaint.py:69-103)."""
    x = resize_max_width(x, max_width)
    # the warp runs on the CPU in fp32 (oracle.iw3 is CPU code; the reference's warp has no autocast-dependent arithmetic)
    dev = x.device
    left, right, lm, rm = oiw3.forward_warp(x.float().cpu(), depth.float().cpu(), divergence, convergence, fill=False,
                                            synthetic_view=synthetic_view, return_mask=True, width_base=False)
    left, right = left.to(dev), right.to(dev)
    lm, rm = (m.to(dev) if m is not None else None for m in (lm, rm))
    kw = dict(inner_dilation=inner_dilation, outer_dilation=outer_dilation, base_width=depth.shape[-1])
    if synthetic_view in ("both", "left"):
        left = forward_left(sd, left, lm, **kw)
    if synthetic_view in ("both", "right"):
        right = forward_right(sd, right, rm, **kw)
    return left, right


def flops(H, W):
    """Multiply-add FLOPs (2 per MAC) of one network forward at an H x W frame, counted from the layer shapes."""
    Hp, Wp = H + 64 - H % 64, W + 64 - W % 64
    t4, t8 = (Hp // 4) * (Wp // 4), (Hp // 8) * (Wp // 8)

    def block(C, tokens, ws, shift, h, w):
        tp = (h + ws) * (w + ws) if shift else tokens
        N = ws * ws
        return 2 * (tp * C * 4 * C + tp * N * 2 * C + tp * 2 * C * C + tokens * C * C + tokens * 9 * (C // 2) * C)

    f = 2 * t4 * 48 * 96
    f += block(96, t4, 16, True, Hp // 4, Wp // 4)
    f += 2 * t8 * 4 * 96 * 192
    for i in range(4):
        f += block(192, t8, 8, i % 2 == 1, Hp // 8, Wp // 8)
    f += 2 * t8 * 192 * 384
    f += block(96, t4, 16, False, Hp // 4, Wp // 4)
    f += 2 * t4 * 9 * 96 * 48
    return f


# ---------------------------------------------------------------------------------------------------------------------------
# seeded inputs of tests/golden/light_inpaint.npz (oracle/gen_golden_inpaint.py)
# ---------------------------------------------------------------------------------------------------------------------------
def hole_mask(seed, b, h, w, frac=0.015):
    """A binary B,1,H,W mask of short horizontal runs (what the forward warp leaves behind foreground edges), about `frac`
    of the pixels, plus a few isolated pixels and 2-pixel gaps for the closing to act on."""
    g = torch.Generator().manual_seed(int(seed))
    m = torch.zeros((b, 1, h, w))
    n = max(1, int(frac * h * w / 3))
    ys = torch.randint(0, h, (b, n), generator=g)
    xs = torch.randint(0, w, (b, n), generator=g)
    ls = torch.randint(1, 6, (b, n), generator=g)
    for i in range(b):
        for y, x, ln in zip(ys[i].tolist(), xs[i].tolist(), ls[i].tolist()):
            m[i, 0, y, x:x + ln] = 1
    return m


def net_inputs(seed, b, h, w):
    from nunif_b200 import synth
    x = torch.stack([synth.synth_image(seed * 16 + i, 3, h, w) for i in range(b)])
    return x, hole_mask(seed, b, h, w)
