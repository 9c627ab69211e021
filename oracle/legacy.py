"""Oracle: UpConv7 / VGG7 forward from a state_dict (TEST INFRASTRUCTURE).

Functional fp32 restatement of waifu2x/models/upconv_7.py and vgg_7.py (eval mode).
Run under ``torch.autocast`` on a GPU it mimics the reference's CUDA path.
"""
import torch
import torch.nn.functional as F


def _stack(sd, x):
    """net.0 .. net.10: 3x3 valid convs, each followed by LeakyReLU(0.1) (upconv_7.py:12-24, vgg_7.py:12-24)."""
    for i in range(0, 12, 2):
        x = F.leaky_relu(F.conv2d(x, sd[f"net.{i}.weight"], sd[f"net.{i}.bias"]), 0.1)
    return x


def upconv7_forward(sd, x):
    """UpConv7.forward eval path (upconv_7.py:25,33-38)."""
    z = F.conv_transpose2d(_stack(sd, x), sd["net.12.weight"], sd["net.12.bias"], stride=2, padding=3)
    return torch.clamp(z, 0., 1.)


def vgg7_forward(sd, x):
    """VGG7.forward eval path (vgg_7.py:25,31-36)."""
    z = F.conv2d(_stack(sd, x), sd["net.12.weight"], sd["net.12.bias"])
    return torch.clamp(z, 0., 1.)


def any_tile_validator(size):
    """Neither model registers a tile-size validator (nunif/models/model.py:51-62)."""
    return True


UPCONV_7 = dict(scale=2, offset=14, blend_size=0)   # upconv_7.py:11
VGG_7 = dict(scale=1, offset=7, blend_size=0)       # vgg_7.py:11
