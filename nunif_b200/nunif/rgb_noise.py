"""Mirror of nunif/utils/rgb_noise.py (rgb_noise_like, apply_rgb_noise): waifu2x's film grain (csrc/rgb_noise.cu).

The noise is counter-based: every value is a pure function of (seed, offset, frame, channel, element), so the same
(seed, offset) gives the same field on every call and any field can be regenerated.  It is a different sample from the
same distribution as the reference's ``torch.randn`` draws, not their bits.  When no seed is given it is drawn from
torch's default CPU generator, so ``torch.manual_seed`` makes a run reproducible."""
import ctypes

import torch

from .. import _lib

_OUT_BITS = {torch.float32: 0, torch.uint8: 8, torch.uint16: 16}


def draw_seed():
    """A 64-bit seed from torch's default CPU generator."""
    return int(torch.empty((), dtype=torch.int64).random_())


def _check_frames(x, name):
    if not torch.is_tensor(x) or x.ndim not in (3, 4):
        raise ValueError(f"{name} must be a CHW or BCHW tensor")


def _check_level(level, H, W):
    if level not in (1, 2):
        raise ValueError(f"level must be 1 or 2, got {level!r}")
    if level == 2 and (H < 2 or W < 2):
        raise ValueError(f"level 2 needs H >= 2 and W >= 2 (its half-resolution field of {H // 2} x {W // 2} is empty)")


def _check_offset(offset, frames):
    if not 0 <= offset or offset + frames > 2 ** 32:
        raise ValueError(f"offset must be in [0, 2**32 - {frames}], got {offset}")


def rgb_noise_like(base, level=2, seed=None, offset=0):
    """rgb_noise.py:5-17: N(0, 1) noise of ``base``'s shape (level 1), or 0.5 * noise + 0.5 * nearest-upsampled
    half-resolution noise (level 2), as float32 on ``base``'s device.  Frame b of a BCHW ``base`` is frame b of the call
    (seed, offset)."""
    _check_frames(base, "base")
    H, W = base.shape[-2], base.shape[-1]
    _check_level(level, H, W)
    _check_offset(offset, 1)
    _lib.require_cuda(base, "base")
    seed = draw_seed() if seed is None else int(seed)
    B = 1 if base.ndim == 3 else base.shape[0]
    out = torch.empty(base.shape, dtype=torch.float32, device=base.device)
    with torch.cuda.device(base.device):
        _lib.check(_lib.lib().nb200_rgb_noise(seed & (2 ** 64 - 1), offset, level, B, base.shape[-3], H, W, _lib.ptr(out),
                                              _lib.stream_ptr(base.device)))
    return out


def _apply(rgb, noise=None, strength=0.2, gamma=2.2, light_decay=True, light_decay_strength=0.8, dtype=torch.float32,
           seed=0, offset=0, level=2, buffer=None, buffer_reset=False, speed=0.0):
    _check_frames(rgb, "rgb")
    if not 0 <= light_decay_strength <= 1:
        raise ValueError(f"light_decay_strength must be in [0, 1], got {light_decay_strength}")
    if not gamma > 0:
        raise ValueError(f"gamma must be positive, got {gamma}")
    if dtype not in _OUT_BITS:
        raise ValueError(f"dtype must be float32, uint8 or uint16, got {dtype}")
    C, H, W = rgb.shape[-3:]
    B = 1 if rgb.ndim == 3 else rgb.shape[0]
    if dtype != torch.float32 and C != 3:
        raise ValueError("uint8 / uint16 output needs 3 channels")
    if noise is None:
        _check_level(level, H, W)
        _check_offset(offset, B)
    if noise is not None and tuple(noise.shape) != tuple(rgb.shape):
        raise ValueError(f"noise shape {tuple(noise.shape)} != rgb shape {tuple(rgb.shape)}")
    _lib.require_cuda(rgb, "rgb")
    x = rgb.float().contiguous()
    if noise is not None:
        noise = noise.to(x.device, torch.float32).contiguous()
    if buffer is not None:
        assert buffer.dtype == torch.float32 and buffer.is_contiguous() and tuple(buffer.shape) == (C, H, W)
    if dtype == torch.float32:
        out = torch.empty(x.shape, dtype=dtype, device=x.device)
    else:
        out = torch.empty(x.shape[:-3] + (H, W, 3), dtype=dtype, device=x.device)
    params = (ctypes.c_double * 4)(strength, gamma, light_decay_strength, speed)
    with torch.cuda.device(x.device):
        _lib.check(_lib.lib().nb200_apply_rgb_noise(
            _lib.ptr(x), B, C, H, W, _lib.ptr(noise), int(seed) & (2 ** 64 - 1), offset, level, _lib.ptr(buffer),
            int(bool(buffer_reset)), params, int(bool(light_decay)), _OUT_BITS[dtype], _lib.ptr(out), _lib.stream_ptr(x.device)))
    return out


def apply_rgb_noise(rgb, noise, strength=0.2, gamma=2.2, light_decay=True, light_decay_strength=0.8, dtype=torch.float32):
    """rgb_noise.py:20-36 on CHW / BCHW float frames and a noise tensor of the same shape, in the reference's fp32 op order.
    ``dtype=torch.uint8 / torch.uint16`` returns the (H, W, 3) frames ``from_tensor`` would make of the result instead."""
    if noise is None:
        raise ValueError("noise is required (rgb_noise_like makes it)")
    return _apply(rgb, noise, strength, gamma, light_decay, light_decay_strength, dtype)


def apply_rgb_noise_like(rgb, strength=0.2, level=2, seed=None, offset=0, **kwargs):
    """``apply_rgb_noise(rgb, rgb_noise_like(rgb, level, seed, offset), strength, **kwargs)`` for one CHW frame, without
    the noise tensor: the kernel generates each value where it applies it."""
    if rgb.ndim != 3:
        raise ValueError("apply_rgb_noise_like takes one CHW frame")
    seed = draw_seed() if seed is None else seed
    return _apply(rgb, None, strength, seed=seed, offset=offset, level=level, **kwargs)


class TemporalGrain:
    """The video path's grain (waifu2x/ui_utils.py:167-175): a device noise buffer that each frame's
    ``rgb_noise_like(frame, seed=seed, offset=t)`` (t = the frame's index in the stream) blends into at ``speed``, applied
    at ``strength``.  The buffer is copied from the noise on the first frame and whenever the frame shape changes."""

    def __init__(self, strength, speed, seed=None):
        self.strength, self.speed = float(strength), float(speed)
        self.seed = draw_seed() if seed is None else int(seed)
        self.buffer = None
        self.frames = 0

    def __call__(self, frames, dtype=torch.float32):
        """Advance over ``frames`` (B, 3, H, W float, in stream order) and return them with grain, as float32 BCHW or,
        for dtype uint8 / uint16, as the encoder's (B, H, W, 3) frames."""
        _check_frames(frames, "frames")
        shape = tuple(frames.shape[-3:])
        reset = self.buffer is None or tuple(self.buffer.shape) != shape or self.buffer.device != frames.device
        if reset:
            self.buffer = torch.empty(shape, dtype=torch.float32, device=frames.device)
        B = 1 if frames.ndim == 3 else frames.shape[0]
        out = _apply(frames, None, self.strength, dtype=dtype, seed=self.seed, offset=self.frames, level=2, buffer=self.buffer,
                     buffer_reset=reset, speed=self.speed)
        self.frames += B
        return out
