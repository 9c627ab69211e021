"""Seeded synthetic weights with the reference's exact state_dict key names.

There are no pretrained checkpoints offline (SURVEY.md section 8c), so parity
and bench runs use random-init weights.  The generators here emit tensors
under the *reference's* key names and shapes (waifu2x/models/cunet.py:10-163,
waifu2x/models/swin_unet.py:119-199, torchvision swin_transformer.py:234-312)
so the same dict loads into the real reference modules with
``load_state_dict(strict=True)`` (done in oracle/gen_golden.py) and into the
H100 engine's weight packer.

Gains are chosen so activations stay O(1) through the stack and the final
output spans [0, 1] (the clamps and the seam blend are then exercised).
"""
import math
import torch


def _gen(seed):
    g = torch.Generator(device="cpu")
    g.manual_seed(int(seed))
    return g


def _normal(g, shape, std):
    return torch.randn(shape, generator=g, dtype=torch.float32) * std


def _conv(sd, g, name, cout, cin, kh, kw, gain=1.0, bias_std=0.02, transpose=False):
    fan_in = cin * kh * kw
    std = gain * math.sqrt(2.0 / fan_in)
    shape = (cin, cout, kh, kw) if transpose else (cout, cin, kh, kw)
    sd[name + ".weight"] = _normal(g, shape, std)
    sd[name + ".bias"] = _normal(g, (cout,), bias_std)


def _linear(sd, g, name, cout, cin, gain=1.0, bias_std=0.02):
    std = gain * math.sqrt(1.0 / cin)
    sd[name + ".weight"] = _normal(g, (cout, cin), std)
    sd[name + ".bias"] = _normal(g, (cout,), bias_std)


# ----------------------------------------------------------------------------
# CUNet family (waifu2x/models/cunet.py)
# ----------------------------------------------------------------------------

def _unet_conv(sd, g, prefix, cin, cmid, cout, se):
    _conv(sd, g, prefix + ".conv.0", cmid, cin, 3, 3)
    _conv(sd, g, prefix + ".conv.2", cout, cmid, 3, 3)
    if se:
        _conv(sd, g, prefix + ".seblock.conv1", cout // 8, cout, 1, 1, gain=0.7, bias_std=0.1)
        _conv(sd, g, prefix + ".seblock.conv2", cout, cout // 8, 1, 1, gain=0.7, bias_std=0.1)


def _unet1(sd, g, prefix, cin, cout, deconv):
    _unet_conv(sd, g, prefix + ".conv1", cin, 32, 64, se=False)
    _conv(sd, g, prefix + ".conv1_down", 64, 64, 2, 2)
    _unet_conv(sd, g, prefix + ".conv2", 64, 128, 64, se=True)
    # ConvTranspose2d(64, 64, 2, 2): weight is (in, out, 2, 2); fan-in per output = 64
    sd[prefix + ".conv2_up.weight"] = _normal(g, (64, 64, 2, 2), math.sqrt(2.0 / 64))
    sd[prefix + ".conv2_up.bias"] = _normal(g, (64,), 0.02)
    _conv(sd, g, prefix + ".conv3", 64, 64, 3, 3, gain=0.7)
    if deconv:
        # ConvTranspose2d(64, cout, 4, 2, 3): each output sees 2x2 taps x 64 ch
        sd[prefix + ".conv_bottom.weight"] = _normal(g, (64, cout, 4, 4), 0.6 * math.sqrt(1.0 / 256))
        sd[prefix + ".conv_bottom.bias"] = torch.full((cout,), 0.5) + _normal(g, (cout,), 0.02)
    else:
        _conv(sd, g, prefix + ".conv_bottom", cout, 64, 3, 3, gain=0.6)
        sd[prefix + ".conv_bottom.bias"] = torch.full((cout,), 0.5) + _normal(g, (cout,), 0.02)


def _unet2(sd, g, prefix, cin, cout):
    _unet_conv(sd, g, prefix + ".conv1", cin, 32, 64, se=False)
    _conv(sd, g, prefix + ".conv1_down", 64, 64, 2, 2)
    _unet_conv(sd, g, prefix + ".conv2", 64, 64, 128, se=True)
    _conv(sd, g, prefix + ".conv2_down", 128, 128, 2, 2)
    _unet_conv(sd, g, prefix + ".conv3", 128, 256, 128, se=True)
    sd[prefix + ".conv3_up.weight"] = _normal(g, (128, 128, 2, 2), math.sqrt(2.0 / 128))
    sd[prefix + ".conv3_up.bias"] = _normal(g, (128,), 0.02)
    _unet_conv(sd, g, prefix + ".conv4", 128, 64, 64, se=True)
    sd[prefix + ".conv4_up.weight"] = _normal(g, (64, 64, 2, 2), math.sqrt(2.0 / 64))
    sd[prefix + ".conv4_up.bias"] = _normal(g, (64,), 0.02)
    _conv(sd, g, prefix + ".conv5", 64, 64, 3, 3, gain=0.7)
    _conv(sd, g, prefix + ".conv_bottom", cout, 64, 3, 3, gain=0.3)
    sd[prefix + ".conv_bottom.bias"] = _normal(g, (cout,), 0.02)


def upcunet_state_dict(seed=0, in_channels=3, out_channels=3):
    """Keys of ``waifu2x.upcunet`` (cunet.py:139-147)."""
    g = _gen(seed)
    sd = {}
    _unet1(sd, g, "unet1", in_channels, out_channels, deconv=True)
    _unet2(sd, g, "unet2", in_channels, out_channels)
    return sd


def cunet_state_dict(seed=0, in_channels=3, out_channels=3):
    """Keys of ``waifu2x.cunet`` (cunet.py:173-181)."""
    g = _gen(seed)
    sd = {}
    _unet1(sd, g, "unet1", in_channels, out_channels, deconv=False)
    _unet2(sd, g, "unet2", in_channels, out_channels)
    return sd


# ----------------------------------------------------------------------------
# UpConv7 / VGG7 (waifu2x/models/upconv_7.py, vgg_7.py): nn.Sequential `net.{0,2,...,12}`
# ----------------------------------------------------------------------------

def _plain_stack(sd, g, widths):
    for i in range(len(widths) - 1):
        _conv(sd, g, f"net.{2 * i}", widths[i + 1], widths[i], 3, 3)


def upconv7_state_dict(seed=0):
    """Keys of ``waifu2x.upconv_7`` (upconv_7.py:12-26); the output ConvTranspose2d(256, 3, 4, 2, 3) is scaled so the tile
    spans [0, 1] with both clamps hit."""
    g = torch.Generator().manual_seed(50_000 + int(seed))
    sd = {}
    _plain_stack(sd, g, [3, 16, 32, 64, 128, 128, 256])
    # weight (in, out, 4, 4); each output sees 2x2 taps x 256 channels
    sd["net.12.weight"] = _normal(g, (256, 3, 4, 4), 1.2 * math.sqrt(1.0 / 1024))
    sd["net.12.bias"] = torch.full((3,), 0.5) + _normal(g, (3,), 0.02)
    return sd


def vgg7_state_dict(seed=0):
    """Keys of ``waifu2x.vgg_7`` (vgg_7.py:12-25); the output Conv2d(128, 3, 3) is scaled so the tile spans [0, 1] with both
    clamps hit."""
    g = torch.Generator().manual_seed(60_000 + int(seed))
    sd = {}
    _plain_stack(sd, g, [3, 32, 32, 64, 64, 128, 128])
    sd["net.12.weight"] = _normal(g, (3, 128, 3, 3), 0.9 * math.sqrt(1.0 / 1152))
    sd["net.12.bias"] = torch.full((3,), 0.35) + _normal(g, (3,), 0.02)   # the hidden activations' mean lifts the output by ~0.1
    return sd


# ----------------------------------------------------------------------------
# SwinUNet family (waifu2x/models/swin_unet.py)
# ----------------------------------------------------------------------------

def relative_position_index(ws=6):
    """torchvision swin_transformer.py:267-279 (define_relative_position_index)."""
    coords = torch.stack(torch.meshgrid(torch.arange(ws), torch.arange(ws), indexing="ij"))
    cf = torch.flatten(coords, 1)
    rel = (cf[:, :, None] - cf[:, None, :]).permute(1, 2, 0).contiguous()
    rel[:, :, 0] += ws - 1
    rel[:, :, 1] += ws - 1
    rel[:, :, 0] *= 2 * ws - 1
    return rel.sum(-1).flatten()


def _swin_blocks(sd, g, prefix, dim, heads, layers, ws=6):
    for i in range(layers):
        p = f"{prefix}.block.{i}"
        sd[p + ".attn.relative_position_bias_table"] = _normal(g, ((2 * ws - 1) ** 2, heads), 0.5)
        sd[p + ".attn.relative_position_index"] = relative_position_index(ws)
        _linear(sd, g, p + ".attn.qkv", dim * 3, dim, gain=1.0)
        _linear(sd, g, p + ".attn.proj", dim, dim, gain=0.5)
        _linear(sd, g, p + ".mlp.0", dim * 2, dim, gain=1.0)
        _linear(sd, g, p + ".mlp.3", dim, dim * 2, gain=0.5)


def swin_unet_state_dict(seed=0, scale_factor=4, in_channels=3, out_channels=3, base_dim=96):
    """Keys of ``SwinUNetBase`` under the ``unet.`` prefix (swin_unet.py:119-199)."""
    assert scale_factor in (1, 2, 4)
    g = _gen(seed)
    sd = {}
    C = base_dim
    H = C // 16
    _conv(sd, g, "unet.patch.0", C // 2, in_channels, 3, 3)
    _conv(sd, g, "unet.patch.2", C, C // 2, 3, 3)
    _swin_blocks(sd, g, "unet.swin1", C, H, 2)
    _conv(sd, g, "unet.down1.conv", C * 2, C, 2, 2, gain=0.7)
    _swin_blocks(sd, g, "unet.swin2", C * 2, H, 2)
    _conv(sd, g, "unet.down2.conv", C * 2, C * 2, 2, 2, gain=0.7)
    _swin_blocks(sd, g, "unet.swin3", C * 2, H, 6)
    _linear(sd, g, "unet.up2.proj", C * 2 * 4, C * 2, gain=0.7)
    if scale_factor in (1, 2):
        _swin_blocks(sd, g, "unet.swin4", C * 2, H, 2)
        _linear(sd, g, "unet.up1.proj", C * 4, C * 2, gain=0.7)
        _swin_blocks(sd, g, "unet.swin5", C, H, 2)
        _linear(sd, g, "unet.to_image.proj", out_channels * scale_factor ** 2, C, gain=0.08)
    else:
        _linear(sd, g, "unet.proj2", C * 2, C, gain=0.7)
        _swin_blocks(sd, g, "unet.swin4", C * 2, H, 2)
        _linear(sd, g, "unet.up1.proj", C * 2 * 4, C * 2, gain=0.7)
        _swin_blocks(sd, g, "unet.swin5", C * 2, H, 2)
        _linear(sd, g, "unet.to_image.proj", out_channels * scale_factor ** 2, C * 2, gain=0.08)
    sd["unet.to_image.proj.bias"] = torch.full_like(sd["unet.to_image.proj.bias"], 0.5) \
        + _normal(g, sd["unet.to_image.proj.bias"].shape, 0.05)
    return sd


# ----------------------------------------------------------------------------
# Synthetic images / depth (SURVEY.md section 8d "Value distributions / seeds")
# ----------------------------------------------------------------------------

def synth_image(seed, c, h, w, smooth=True):
    """Uniform noise image in [0,1]; ``smooth`` mixes in low-frequency content."""
    g = _gen(seed)
    x = torch.rand((c, h, w), generator=g, dtype=torch.float32)
    if smooth:
        import torch.nn.functional as F
        lo = torch.rand((1, c, max(h // 16, 2), max(w // 16, 2)), generator=g, dtype=torch.float32)
        lo = F.interpolate(lo, size=(h, w), mode="bilinear", align_corners=False)[0]
        x = (0.25 * x + 0.75 * lo).clamp(0, 1)
    return x


def synth_depth(seed, b, h, w, boxes=True):
    """Smooth depth in [0,1] plus the reference _bench box pattern
    (iw3/forward_warp.py:311-316) so holes/layered holes occur."""
    import torch.nn.functional as F
    g = _gen(seed)
    d = torch.rand((b, 1, max(h // 24, 2), max(w // 24, 2)), generator=g, dtype=torch.float32)
    d = F.interpolate(d, size=(h, w), mode="bicubic", align_corners=False)
    d = d + torch.rand((b, 1, h, w), generator=g, dtype=torch.float32) * 1e-3  # break exact ties
    if boxes:
        y0, y1 = h // 4, h // 4 + h // 3
        x0, x1 = w // 4, w // 4 + w // 4
        d[:, :, y0:y1, x0:x1] += 1.0
        y0, y1 = h // 2, h // 2 + h // 4
        x0, x1 = w // 2 + w // 8, w // 2 + w // 8 + w // 5
        d[:, :, y0:y1, x0:x1] += 0.5
    mn = d.amin(dim=(1, 2, 3), keepdim=True)
    mx = d.amax(dim=(1, 2, 3), keepdim=True)
    return ((d - mn) / (mx - mn)).contiguous()


def depth_anything_v2_state_dict(seed=0, encoder="vits", pos_grid=37):
    """Seeded Depth-Anything-V2 weights with the upstream key names (`pretrained.*` = DINOv2 ViT, `depth_head.*` = DPT head).
    No checkpoint can be downloaded here; gains are chosen so that activations stay O(1) through the 12 blocks and the
    predicted depth is a non-trivial positive map.  pos_grid=37 is the 518/14 training grid of the released models."""
    dim, depth, heads, feat, oc = {"vits": (384, 12, 6, 64, (48, 96, 192, 384)),
                                   "vitb": (768, 12, 12, 128, (96, 192, 384, 768)),
                                   "vitl": (1024, 24, 16, 256, (256, 512, 1024, 1024))}[encoder]
    g = torch.Generator().manual_seed(10_000 + seed)

    def rn(*shape, std=1.0):
        return torch.randn(*shape, generator=g) * std

    sd = {}
    sd["pretrained.cls_token"] = rn(1, 1, dim, std=0.02)
    sd["pretrained.pos_embed"] = rn(1, 1 + pos_grid * pos_grid, dim, std=0.2)
    sd["pretrained.mask_token"] = torch.zeros(1, dim)
    sd["pretrained.patch_embed.proj.weight"] = rn(dim, 3, 14, 14, std=1.0 / (3 * 14 * 14) ** 0.5)
    sd["pretrained.patch_embed.proj.bias"] = rn(dim, std=0.02)
    for i in range(depth):
        p = f"pretrained.blocks.{i}."
        sd[p + "norm1.weight"] = 1.0 + rn(dim, std=0.1)
        sd[p + "norm1.bias"] = rn(dim, std=0.05)
        sd[p + "attn.qkv.weight"] = rn(3 * dim, dim, std=1.2 / dim ** 0.5)
        sd[p + "attn.qkv.bias"] = rn(3 * dim, std=0.02)
        sd[p + "attn.proj.weight"] = rn(dim, dim, std=1.0 / dim ** 0.5)
        sd[p + "attn.proj.bias"] = rn(dim, std=0.02)
        sd[p + "ls1.gamma"] = 0.3 + rn(dim, std=0.05)
        sd[p + "norm2.weight"] = 1.0 + rn(dim, std=0.1)
        sd[p + "norm2.bias"] = rn(dim, std=0.05)
        sd[p + "mlp.fc1.weight"] = rn(4 * dim, dim, std=1.0 / dim ** 0.5)
        sd[p + "mlp.fc1.bias"] = rn(4 * dim, std=0.02)
        sd[p + "mlp.fc2.weight"] = rn(dim, 4 * dim, std=1.0 / (4 * dim) ** 0.5)
        sd[p + "mlp.fc2.bias"] = rn(dim, std=0.02)
        sd[p + "ls2.gamma"] = 0.3 + rn(dim, std=0.05)
    sd["pretrained.norm.weight"] = 1.0 + rn(dim, std=0.1)
    sd["pretrained.norm.bias"] = rn(dim, std=0.05)
    for i, c in enumerate(oc):
        sd[f"depth_head.projects.{i}.weight"] = rn(c, dim, 1, 1, std=1.0 / dim ** 0.5)
        sd[f"depth_head.projects.{i}.bias"] = rn(c, std=0.02)
        sd[f"depth_head.scratch.layer{i + 1}_rn.weight"] = rn(feat, c, 3, 3, std=1.0 / (9 * c) ** 0.5)
    sd["depth_head.resize_layers.0.weight"] = rn(oc[0], oc[0], 4, 4, std=1.0 / oc[0] ** 0.5)
    sd["depth_head.resize_layers.0.bias"] = rn(oc[0], std=0.02)
    sd["depth_head.resize_layers.1.weight"] = rn(oc[1], oc[1], 2, 2, std=1.0 / oc[1] ** 0.5)
    sd["depth_head.resize_layers.1.bias"] = rn(oc[1], std=0.02)
    sd["depth_head.resize_layers.3.weight"] = rn(oc[3], oc[3], 3, 3, std=1.0 / (9 * oc[3]) ** 0.5)
    sd["depth_head.resize_layers.3.bias"] = rn(oc[3], std=0.02)
    for r in (1, 2, 3, 4):
        p = f"depth_head.scratch.refinenet{r}."
        sd[p + "out_conv.weight"] = rn(feat, feat, 1, 1, std=1.0 / feat ** 0.5)
        sd[p + "out_conv.bias"] = rn(feat, std=0.02)
        for u in (1, 2):
            for cv in (1, 2):
                sd[p + f"resConfUnit{u}.conv{cv}.weight"] = rn(feat, feat, 3, 3, std=0.7 / (9 * feat) ** 0.5)
                sd[p + f"resConfUnit{u}.conv{cv}.bias"] = rn(feat, std=0.02)
    sd["depth_head.scratch.output_conv1.weight"] = rn(feat // 2, feat, 3, 3, std=1.0 / (9 * feat) ** 0.5)
    sd["depth_head.scratch.output_conv1.bias"] = rn(feat // 2, std=0.02)
    sd["depth_head.scratch.output_conv2.0.weight"] = rn(32, feat // 2, 3, 3, std=1.4 / (9 * feat // 2) ** 0.5)
    sd["depth_head.scratch.output_conv2.0.bias"] = 0.2 + rn(32, std=0.05)
    sd["depth_head.scratch.output_conv2.2.weight"] = rn(1, 32, 1, 1, std=1.0 / 32 ** 0.5).abs()
    sd["depth_head.scratch.output_conv2.2.bias"] = torch.full((1,), 0.3)
    return sd


def row_flow_v3_state_dict(seed=0):
    """Seeded weights with the key names of `sbs.row_flow_v3` (iw3/models/row_flow_v3.py); buffers (`index`, `delta`,
    `delta_scale`) are the constants the reference constructs.  Gains give deltas of a few pixels for unit-range depth."""
    g = torch.Generator().manual_seed(20_000 + seed)

    def rn(*shape, std=1.0):
        return torch.randn(*shape, generator=g) * std

    sd = {"blocks.0.weight": rn(64, 24, 1, 1, std=1.0 / 24 ** 0.5), "blocks.0.bias": rn(64, std=0.05)}
    for bi, ws in ((1, 4), (2, 3)):
        p = f"blocks.{bi}."
        N = ws * ws
        hid = int(N ** 0.5) * 2
        sd[p + "mha.mha.qkv_proj.weight"] = rn(192, 64, std=1.2 / 8)
        sd[p + "mha.mha.qkv_proj.bias"] = rn(192, std=0.05)
        sd[p + "mha.mha.head_proj.weight"] = rn(64, 64, std=0.6 / 8)
        sd[p + "mha.mha.head_proj.bias"] = rn(64, std=0.02)
        sd[p + "conv_mlp.0.weight"] = rn(64, 64, 1, 1, std=1.0 / 8)
        sd[p + "conv_mlp.0.bias"] = rn(64, std=0.05)
        sd[p + "conv_mlp.3.weight"] = rn(64, 64, 3, 3, std=0.6 / 24)
        sd[p + "conv_mlp.3.bias"] = rn(64, std=0.02)
        pos = torch.stack(torch.meshgrid(torch.arange(ws), torch.arange(ws), indexing="ij"), dim=2).reshape(N, 2)
        delta = [tuple(d) for d in (pos[:, None, :] - pos[None, :, :]).reshape(N * N, 2).tolist()]
        uniq = sorted(set(delta))
        sd[p + "bias.index"] = torch.tensor([uniq.index(d) for d in delta], dtype=torch.int64)
        ud = torch.tensor(uniq, dtype=torch.float32)
        sd[p + "bias.delta"] = ud / ud.abs().max()
        sd[p + "bias.to_bias.0.weight"] = rn(hid, 2, std=1.0)
        sd[p + "bias.to_bias.0.bias"] = rn(hid, std=0.3)
        sd[p + "bias.to_bias.2.weight"] = rn(1, hid, std=1.0)
        sd[p + "bias.to_bias.2.bias"] = rn(1, std=0.1)
    sd["last_layer.1.weight"] = rn(1, 8, 3, 3, std=1.5 / 72 ** 0.5)
    sd["last_layer.1.bias"] = rn(1, std=0.1)
    sd["delta_scale"] = torch.tensor(1.0 / 127.0)
    return sd


def row_flow_v2_state_dict(seed=0):
    """Seeded weights with the key names of `sbs.row_flow_v2` (iw3/models/row_flow_v2.py:13-37).  He-style gains with small
    positive biases keep the ReLUs alive; the two heads give deltas of a few pixels for unit-range depth."""
    g = torch.Generator().manual_seed(21_000 + seed)

    def rn(*shape, std=1.0):
        return torch.randn(*shape, generator=g) * std

    return {
        "feature.0.weight": rn(16, 3, 1, 3, std=(2.0 / 9) ** 0.5), "feature.0.bias": 0.05 + rn(16, std=0.05),
        "non_overlap.weight": rn(1, 16, 1, 1, std=0.5), "non_overlap.bias": rn(1, std=0.1),
        "overlap_residual.0.weight": rn(16, 16, 1, 9, std=(2.0 / 144) ** 0.5), "overlap_residual.0.bias": 0.05 + rn(16, std=0.05),
        "overlap_residual.2.weight": rn(32, 16, 1, 9, std=(2.0 / 144) ** 0.5), "overlap_residual.2.bias": 0.05 + rn(32, std=0.05),
        "overlap_residual.4.weight": rn(32, 32, 1, 9, std=(2.0 / 288) ** 0.5), "overlap_residual.4.bias": 0.05 + rn(32, std=0.05),
        "overlap_residual.6.weight": rn(1, 32, 3, 3, std=1.0 / 288 ** 0.5), "overlap_residual.6.bias": rn(1, std=0.1),
        "delta_scale": torch.tensor(1.0 / 127.0),
    }


def _window_bias_buffers(ws):
    """`index` / `delta` buffers of WindowScoreBias (nunif/modules/attention.py:347-372) for a square window."""
    N = ws * ws
    pos = torch.stack(torch.meshgrid(torch.arange(ws), torch.arange(ws), indexing="ij"), dim=2).reshape(N, 2)
    delta = [tuple(d) for d in (pos[:, None, :] - pos[None, :, :]).reshape(N * N, 2).tolist()]
    uniq = sorted(set(delta))
    index = torch.tensor([uniq.index(d) for d in delta], dtype=torch.int64)
    ud = torch.tensor(uniq, dtype=torch.float32)
    return index, ud / ud.abs().max()


def depth_aa_state_dict(seed=0):
    """Seeded weights with the key names of `iw3.depth_aa` (iw3/models/depth_aa.py); the released model zero-initialises
    proj_out, here every tensor is random so that the filter is non-trivial."""
    g = torch.Generator().manual_seed(30_000 + seed)

    def rn(*shape, std=1.0):
        return torch.randn(*shape, generator=g) * std

    C = 32
    sd = {"proj_in.weight": rn(C, 4, 1, 1, std=0.5), "proj_in.bias": rn(C, std=0.05)}
    for i in range(3):
        p = f"blocks.{i}."
        sd[p + "mha.mha.qkv_proj.weight"] = rn(3 * C, C, std=1.0 / C ** 0.5)
        sd[p + "mha.mha.qkv_proj.bias"] = rn(3 * C, std=0.05)
        sd[p + "mha.mha.head_proj.weight"] = rn(C, C, std=0.6 / C ** 0.5)
        sd[p + "mha.mha.head_proj.bias"] = rn(C, std=0.02)
        sd[p + "conv_mlp.0.weight"] = rn(C, C, 1, 1, std=1.0 / C ** 0.5)
        sd[p + "conv_mlp.0.bias"] = rn(C, std=0.05)
        sd[p + "conv_mlp.3.weight"] = rn(C, C, 3, 3, std=0.6 / (9 * C) ** 0.5)
        sd[p + "conv_mlp.3.bias"] = rn(C, std=0.02)
        sd[p + "bias.index"], sd[p + "bias.delta"] = _window_bias_buffers(8)
        sd[p + "bias.to_bias.0.weight"] = rn(16, 2, std=1.0)
        sd[p + "bias.to_bias.0.bias"] = rn(16, std=0.3)
        sd[p + "bias.to_bias.2.weight"] = rn(1, 16, std=0.7)
        sd[p + "bias.to_bias.2.bias"] = rn(1, std=0.1)
    sd["proj_out.weight"] = rn(4, C, 1, 1, std=0.05)
    sd["proj_out.bias"] = rn(4, std=0.01)
    return sd


def mlbw_state_dict(seed=0, num_layers=2):
    """Seeded weights with the key names of `sbs.mlbw` (iw3/models/mlbw.py, MLBW(num_layers, base_dim=32))."""
    g = torch.Generator().manual_seed(40_000 + seed)

    def rn(*shape, std=1.0):
        return torch.randn(*shape, generator=g) * std

    C = 32 * num_layers
    c1 = C // 8
    sd = {"lv1_in.1.weight": rn(c1, 3, 1, 9, std=1.0 / 27 ** 0.5), "lv1_in.1.bias": rn(c1, std=0.05)}
    for i in range(4):
        p = f"lv2.{i}."
        sd[p + "mha.mha.qkv_proj.weight"] = rn(3 * C, C, std=1.0 / C ** 0.5)
        sd[p + "mha.mha.qkv_proj.bias"] = rn(3 * C, std=0.05)
        sd[p + "mha.mha.head_proj.weight"] = rn(C, C, std=0.6 / C ** 0.5)
        sd[p + "mha.mha.head_proj.bias"] = rn(C, std=0.02)
        sd[p + "conv_mlp.0.weight"] = rn(C, C, 1, 1, std=1.0 / C ** 0.5)
        sd[p + "conv_mlp.0.bias"] = rn(C, std=0.05)
        sd[p + "conv_mlp.3.weight"] = rn(C, C, 3, 3, std=0.6 / (9 * C) ** 0.5)
        sd[p + "conv_mlp.3.bias"] = rn(C, std=0.02)
        sd[p + "bias.index"], sd[p + "bias.delta"] = _window_bias_buffers(4)
        sd[p + "bias.to_bias.0.weight"] = rn(8, 2, std=1.0)
        sd[p + "bias.to_bias.0.bias"] = rn(8, std=0.3)
        sd[p + "bias.to_bias.2.weight"] = rn(1, 8, std=0.7)
        sd[p + "bias.to_bias.2.bias"] = rn(1, std=0.1)
    sd["lv1_out.1.weight"] = rn(2 * num_layers, c1, 1, 9, std=1.5 / (9 * c1) ** 0.5)
    sd["lv1_out.1.bias"] = rn(2 * num_layers, std=0.1)
    return sd


MASK_MLBW_HOLE_BIAS = -2.1


def mask_mlbw_state_dict(seed=0):
    """Seeded weights of `sbs.mask_mlbw_l2` (MLBW(num_layers=2, base_dim=32, hole_mask=True), iw3/models/mlbw.py:70-74): the
    weights of mlbw_state_dict(seed, 2) plus a fifth lv1_out output, the hole logit, drawn from a generator of its own so that
    mlbw_state_dict's streams stay as they are.  Its bias puts a few percent of the pixels of a typical frame over the 0.15
    threshold of iw3/mlbw_inpaint.py:18 (oracle/gen_golden_mask_mlbw.py checks 3-30 % on the golden inputs)."""
    sd = mlbw_state_dict(seed, 2)
    g = torch.Generator().manual_seed(41_000 + seed)
    c1 = 8
    w = torch.randn(1, c1, 1, 9, generator=g) * (1.5 / (9 * c1) ** 0.5)
    sd["lv1_out.1.weight"] = torch.cat([sd["lv1_out.1.weight"], w])
    sd["lv1_out.1.bias"] = torch.cat([sd["lv1_out.1.bias"], torch.tensor([MASK_MLBW_HOLE_BIAS])])
    return sd


ZOED_N = dict(dim=1024, depth=24, heads=16, hooks=(5, 11, 17, 23), oc=(256, 512, 1024, 1024), feat=256, old_grid=24)
ZOED_MINI = dict(dim=256, depth=4, heads=4, hooks=(0, 1, 2, 3), oc=(64, 128, 256, 256), feat=128, old_grid=6)


def zoedepth_state_dict(seed=0, cfg=None):
    """Seeded ZoeD_N weights with the upstream checkpoint key names (ZoeD_M12_N.pt: `core.core.pretrained.model.*` = timm
    BEiT-L/16, `core.core.pretrained.act_postprocess*` / `core.core.scratch.*` = MiDaS DPT head, the rest = ZoeDepth bins
    head).  No checkpoint can be downloaded here; gains keep activations O(1) through the blocks and give a metric depth
    map that varies over the image.  `cfg`: ZOED_N (default) or ZOED_MINI (fast tests, same code path)."""
    cfg = cfg or ZOED_N
    dim, depth, heads, oc, feat, grid = cfg["dim"], cfg["depth"], cfg["heads"], cfg["oc"], cfg["feat"], cfg["old_grid"]
    g = torch.Generator().manual_seed(30_000 + seed)

    def rn(*shape, std=1.0):
        return torch.randn(*shape, generator=g) * std

    def conv(name, cout, cin, k, gain=1.0, bias=0.02, bias_mean=0.0):
        sd[name + ".weight"] = rn(cout, cin, k, k, std=gain / (cin * k * k) ** 0.5)
        sd[name + ".bias"] = bias_mean + rn(cout, std=bias)

    sd = {}
    bb, pp, sc = "core.core.pretrained.model.", "core.core.pretrained.", "core.core.scratch."
    sd[bb + "cls_token"] = rn(1, 1, dim, std=0.5)
    sd[bb + "patch_embed.proj.weight"] = rn(dim, 3, 16, 16, std=2.0 / (3 * 16 * 16) ** 0.5)
    sd[bb + "patch_embed.proj.bias"] = rn(dim, std=0.2)
    nrd = (2 * grid - 1) ** 2 + 3
    for i in range(depth):
        p = f"{bb}blocks.{i}."
        sd[p + "gamma_1"] = 0.5 + rn(dim, std=0.1)
        sd[p + "gamma_2"] = 0.5 + rn(dim, std=0.1)
        sd[p + "norm1.weight"] = 1.0 + rn(dim, std=0.1)
        sd[p + "norm1.bias"] = rn(dim, std=0.05)
        sd[p + "attn.q_bias"] = rn(dim, std=0.05)
        sd[p + "attn.v_bias"] = rn(dim, std=0.05)
        sd[p + "attn.relative_position_bias_table"] = rn(nrd, heads, std=0.8)
        sd[p + "attn.qkv.weight"] = rn(3 * dim, dim, std=1.2 / dim ** 0.5)
        sd[p + "attn.proj.weight"] = rn(dim, dim, std=1.0 / dim ** 0.5)
        sd[p + "attn.proj.bias"] = rn(dim, std=0.02)
        sd[p + "norm2.weight"] = 1.0 + rn(dim, std=0.1)
        sd[p + "norm2.bias"] = rn(dim, std=0.05)
        sd[p + "mlp.fc1.weight"] = rn(4 * dim, dim, std=1.0 / dim ** 0.5)
        sd[p + "mlp.fc1.bias"] = rn(4 * dim, std=0.02)
        sd[p + "mlp.fc2.weight"] = rn(dim, 4 * dim, std=1.0 / (4 * dim) ** 0.5)
        sd[p + "mlp.fc2.bias"] = rn(dim, std=0.02)
    for i, c in enumerate(oc):
        p = f"{pp}act_postprocess{i + 1}."
        sd[p + "0.project.0.weight"] = rn(dim, 2 * dim, std=1.0 / (2 * dim) ** 0.5)
        sd[p + "0.project.0.bias"] = rn(dim, std=0.02)
        conv(p + "3", c, dim, 1, gain=1.5)
        sd[f"{sc}layer{i + 1}_rn.weight"] = rn(feat, c, 3, 3, std=1.0 / (9 * c) ** 0.5)
    p = pp + "act_postprocess1.4"
    sd[p + ".weight"], sd[p + ".bias"] = rn(oc[0], oc[0], 4, 4, std=1.0 / oc[0] ** 0.5), rn(oc[0], std=0.02)
    p = pp + "act_postprocess2.4"
    sd[p + ".weight"], sd[p + ".bias"] = rn(oc[1], oc[1], 2, 2, std=1.0 / oc[1] ** 0.5), rn(oc[1], std=0.02)
    conv(pp + "act_postprocess4.4", oc[3], oc[3], 3)
    for r in (1, 2, 3, 4):
        p = f"{sc}refinenet{r}."
        conv(p + "out_conv", feat, feat, 1)
        for u in (1, 2):
            for cv in (1, 2):
                conv(p + f"resConfUnit{u}.conv{cv}", feat, feat, 3, gain=0.7)
    conv(sc + "output_conv.0", feat // 2, feat, 3)
    conv(sc + "output_conv.2", 32, feat // 2, 3, gain=1.4, bias=0.05, bias_mean=0.2)
    sd[sc + "output_conv.4.weight"] = rn(1, 32, 1, 1, std=1.0 / 32 ** 0.5).abs()
    sd[sc + "output_conv.4.bias"] = torch.full((1,), 0.3)
    # bins head (zoedepth_v1.py): conv2, SeedBinRegressorUnnormed (mlp_dim 256), Projector (mlp_dim 128), AttractorLayerUnnormed
    conv("conv2", feat, feat, 1)
    conv("seed_bin_regressor._net.0", 256, feat, 1, gain=1.4)
    conv("seed_bin_regressor._net.2", 64, 256, 1, gain=2.0, bias=1.0, bias_mean=1.0)
    conv("seed_projector._net.0", 128, feat, 1, gain=1.4)
    conv("seed_projector._net.2", 128, 128, 1, gain=1.4)
    for i, na in enumerate((16, 8, 4, 1)):
        conv(f"projectors.{i}._net.0", 128, feat, 1, gain=1.4)
        conv(f"projectors.{i}._net.2", 128, 128, 1, gain=1.4)
        conv(f"attractors.{i}._net.0", 128, 128, 1, gain=1.4)
        conv(f"attractors.{i}._net.2", na, 128, 1, gain=2.0, bias=1.0, bias_mean=1.0)
    conv("conditional_log_binomial.mlp.0", (33 + 128) // 2, 33 + 128, 1, gain=1.4)
    conv("conditional_log_binomial.mlp.2", 4, (33 + 128) // 2, 1, gain=2.0, bias=0.5)
    return sd


# ----------------------------------------------------------------------------
# iw3 inpainting (iw3/models/light_inpaint_v1.py)
# ----------------------------------------------------------------------------

def _gmlp_block(sd, g, prefix, C, N):
    """One GMLPBlock (light_inpaint_v1.py:37-49, nunif/modules/attention.py:621-660).  proj_spatial gets about +-1/sqrt(N) and a
    varied bias instead of the reference's init (+-1e-3/C, bias 1), which would make the token mixing invisible in the output."""
    p = prefix + ".gmlp.gmlp"
    _linear(sd, g, p + ".proj_in", 4 * C, C, gain=1.0, bias_std=0.2)
    sd[p + ".proj_spatial.weight"] = (torch.rand((N, N, 1), generator=g) * 2 - 1) * (1.0 / math.sqrt(N))
    sd[p + ".proj_spatial.bias"] = 0.5 + torch.rand((N,), generator=g)
    _linear(sd, g, p + ".proj_out", C, 2 * C, gain=0.5, bias_std=0.05)
    sd[prefix + ".norm1.weight"] = 1.0 + _normal(g, (C,), 0.1)
    sd[prefix + ".norm2.weight"] = 1.0 + _normal(g, (2 * C,), 0.1)
    _conv(sd, g, prefix + ".glu_conv.w1", C, C, 1, 1, gain=1.0, bias_std=0.1)
    _conv(sd, g, prefix + ".glu_conv.w2", C, C // 2, 3, 3, gain=0.3, bias_std=0.02)


def light_inpaint_v1_state_dict(seed=0):
    """`inpaint.light_inpaint_v1` (81 tensors).  The output head is scaled so that the network's output spans [0, 1] around
    0.5 and the hole pixels, which take the network output, show every stage; `mask_bias` is far from zero."""
    g = _gen(seed)
    sd = {}
    C = 96
    sd["mask_bias"] = _normal(g, (1, C, 1, 1), 0.5)
    _conv(sd, g, "patch.0", C, 48, 1, 1, gain=1.0, bias_std=0.05)
    _gmlp_block(sd, g, "enc1", C, 256)
    _conv(sd, g, "down", 2 * C, C, 2, 2, gain=0.5, bias_std=0.02)
    for i in range(4):
        _gmlp_block(sd, g, f"enc2.{i}", 2 * C, 64)
    _conv(sd, g, "up", 4 * C, 2 * C, 1, 1, gain=0.5, bias_std=0.02)
    _gmlp_block(sd, g, "dec1", C, 256)
    _conv(sd, g, "to_image.1", 48, C, 3, 3, gain=0.05, bias_std=0.0)
    sd["to_image.1.bias"] = 0.5 + _normal(g, (48,), 0.05)
    return sd


# ----------------------------------------------------------------------------
# iw3.sod_v1 (iw3/models/sod_v1.py: U2NETP(in_ch=6), nunif/utils/u2netp.py)
# ----------------------------------------------------------------------------

# the outconv bias of sod_v1_state_dict: with it the saliency > 0.5 mask covers part of each golden frame, neither none nor
# all of it (oracle/gen_golden_sod.py prints and checks the fraction)
SOD_OUT_BIAS = 0.76

SOD_STAGES = (("stage1", 7, 6), ("stage2", 6, 64), ("stage3", 5, 64), ("stage4", 4, 64), ("stage5", 0, 64), ("stage6", 0, 64),
              ("stage5d", 0, 128), ("stage4d", 4, 128), ("stage3d", 5, 128), ("stage2d", 6, 128), ("stage1d", 7, 128))


def sod_rebnconvs():
    """(name, cin, cout, dilation) of every REBNCONV of U2NETP(in_ch=6) in forward order; RSU4F is n = 0."""
    out = []
    for stage, n, cin in SOD_STAGES:
        p = f"u2netp.{stage}.rebnconv"
        out += [(p + "in", cin, 64, 1), (p + "1", 64, 16, 1)]
        if n == 0:
            out += [(p + "2", 16, 16, 2), (p + "3", 16, 16, 4), (p + "4", 16, 16, 8), (p + "3d", 32, 16, 4), (p + "2d", 32, 16, 2)]
        else:
            out += [(p + str(k), 16, 16, 1) for k in range(2, n)] + [(p + str(n), 16, 16, 2)]
            out += [(p + f"{k}d", 32, 16, 1) for k in range(n - 1, 1, -1)]
        out.append((p + "1d", 32, 64, 1))
    return out


def sod_v1_state_dict(seed=0):
    """Seeded weights with the key names of `iw3.sod_v1` (SODV1.u2netp).  Every BatchNorm has non-trivial statistics
    (running_var != 1, gamma, beta, mean) so that the folding of U2NETP.fuse() matters; the gains keep the activations of
    the residual stages in fp16 range, and SOD_OUT_BIAS sets the share of salient pixels."""
    g = torch.Generator().manual_seed(60_000 + seed)
    sd = {}
    for name, cin, cout, _ in sod_rebnconvs():
        sd[name + ".conv_s1.weight"] = torch.randn(cout, cin, 3, 3, generator=g) * (1.4 / (9 * cin)) ** 0.5
        sd[name + ".conv_s1.bias"] = torch.randn(cout, generator=g) * 0.05
        sd[name + ".bn_s1.weight"] = 0.8 + 0.4 * torch.rand(cout, generator=g)
        sd[name + ".bn_s1.bias"] = 0.02 + torch.randn(cout, generator=g) * 0.05
        sd[name + ".bn_s1.running_mean"] = torch.randn(cout, generator=g) * 0.1
        sd[name + ".bn_s1.running_var"] = 0.5 + 1.5 * torch.rand(cout, generator=g)
        sd[name + ".bn_s1.num_batches_tracked"] = torch.tensor(1000, dtype=torch.int64)
    for k in range(1, 7):
        sd[f"u2netp.side{k}.weight"] = torch.randn(1, 64, 3, 3, generator=g) * (1.0 / (9 * 64)) ** 0.5
        sd[f"u2netp.side{k}.bias"] = torch.randn(1, generator=g) * 0.1
    sd["u2netp.outconv.weight"] = (0.5 + torch.rand(1, 6, 1, 1, generator=g)) / 3
    sd["u2netp.outconv.bias"] = torch.tensor([SOD_OUT_BIAS])
    return sd
