"""CPU restatement of nunif/utils/rgb_noise.py (rgb_noise_like, apply_rgb_noise), of waifu2x's video noise buffer
(waifu2x/ui_utils.py:167-175) and of from_tensor's quantisation (nunif/utils/video.py:236-245), plus the engine's own
counter-based noise (csrc/rgb_noise.cu) restated in numpy.

rgb_noise_like draws exactly what the reference draws from torch's global generator (randn_like, then randn of the
half-resolution field) and upsamples with ATen's nearest rule written out, so after torch.manual_seed it reproduces the
reference's noise bit for bit.  apply_rgb_noise / temporal_step are torch ops in the reference's order and run on any
device: on CUDA they are the reference's own GPU evaluation."""
import hashlib

import numpy as np
import torch

# waifu2x/ui_utils.py:58-61, :167-175 and rgb_noise.py defaults
PARAMS = {
    "default": dict(strength=0.2, gamma=2.2, light_decay=True, light_decay_strength=0.8),
    "image": dict(strength=0.05 * 0.5, gamma=2.2, light_decay=True, light_decay_strength=0.8),
    "no_decay_g18": dict(strength=0.5, gamma=1.8, light_decay=False, light_decay_strength=0.8),
    "g2_lds03": dict(strength=0.35, gamma=2.0, light_decay=True, light_decay_strength=0.3),
    "g24_lds1": dict(strength=0.8, gamma=2.4, light_decay=True, light_decay_strength=1.0),
    "g3_lds0": dict(strength=0.2, gamma=3.0, light_decay=True, light_decay_strength=0.0),
}
# (name, shape, level, seed) of the noise cases; the 1080 x 1920 field is kept as a SHA-256 and CROPS
NOISE_CASES = [
    ("chw_5x7_l2", (3, 5, 7), 2, 11), ("chw_5x7_l1", (3, 5, 7), 1, 12), ("chw_6x8_l2", (3, 6, 8), 2, 13),
    ("bchw_7x5_l2", (2, 3, 7, 5), 2, 14), ("chw_2x3_l2", (3, 2, 3), 2, 15), ("chw_33x17_l2", (3, 33, 17), 2, 16),
    ("chw_1080x1920_l2", (3, 1080, 1920), 2, 17), ("chw_1081x1919_l2", (3, 1081, 1919), 2, 18),
]
FULL_NOISE = {"chw_1080x1920_l2", "chw_1081x1919_l2"}
CROPS = [(slice(0, 9), slice(0, 9)), (slice(536, 545), slice(955, 966)), (slice(-9, None), slice(-11, None))]
# (name, shape) of the apply inputs; each is run under every PARAMS entry
APPLY_CASES = [("chw_5x7", (3, 5, 7)), ("bchw_6x8", (2, 3, 6, 8)), ("chw_24x40", (3, 24, 40))]
# the temporal sequence: 6 frames, the shape changes at frame 3
TEMPORAL_SHAPES = [(3, 6, 8)] * 3 + [(3, 5, 7)] * 3
TEMPORAL_SPEED, TEMPORAL_STRENGTH = 0.8, 0.2


def nearest_index(out_size, in_size):
    """ATen's nearest source index for F.interpolate(size=...) (UpSample.h nearest_idx): out == in -> d,
    out == 2 in -> d >> 1, else min(int(d * ((float)in / out)), in - 1) in fp32."""
    d = np.arange(out_size)
    if out_size == in_size:
        return d
    if out_size == 2 * in_size:
        return d >> 1
    scale = np.float32(in_size) / np.float32(out_size)
    return np.minimum(np.floor(d.astype(np.float32) * scale).astype(np.int64), in_size - 1)


def rgb_noise_like(base, level=2):
    """rgb_noise.py:5-17 with the interpolate written as the index rule above: same draws, same order."""
    assert level in {1, 2}
    noise = torch.randn_like(base)
    if level == 2:
        H, W = base.shape[-2], base.shape[-1]
        noise2 = torch.randn(base.shape[:-2] + (H // 2, W // 2), dtype=base.dtype, device=base.device)
        iy = torch.from_numpy(nearest_index(H, H // 2)).to(base.device)
        ix = torch.from_numpy(nearest_index(W, W // 2)).to(base.device)
        noise2 = noise2.index_select(-2, iy).index_select(-1, ix)
        noise.mul_(0.5).add_(noise2, alpha=0.5)
    return noise


def apply_rgb_noise(rgb, noise, strength=0.2, gamma=2.2, light_decay=True, light_decay_strength=0.8):
    """rgb_noise.py:20-36, op for op."""
    assert 0 <= light_decay_strength <= 1
    output = rgb ** gamma
    correlated_noise = noise * output
    if light_decay:
        ld = (1.0 - output).mul_(light_decay_strength).add_(1.0 - light_decay_strength)
        ld = ld.pow_(gamma)
    else:
        ld = torch.tensor(1.0, device=rgb.device)
    weight = ld.mul_(strength)
    output = output.add_(correlated_noise.mul_(weight))
    return output.clamp_(0, 1).pow_(1.0 / gamma)


def temporal_step(buffer, noise, speed):
    """ui_utils.py:168-174: the buffer after one frame (None = no buffer yet)."""
    if buffer is None or noise.shape != buffer.shape:
        return noise.clone()
    return buffer.mul(1.0 - speed).add_(noise.mul(speed))


def from_tensor(x, bits):
    """video.py:236-245 without the PyAV frame: CHW float -> HWC uint8 / uint16."""
    dtype, scale = (torch.uint16, 65535.0) if bits == 16 else (torch.uint8, 255.0)
    return (x.permute(1, 2, 0).contiguous() * scale).round_().to(dtype)


def golden_rgb(shape, seed):
    """Seeded frames in [0, 1] with exact 0s and 1s and values just below 1 (the clamp's and pow's edges)."""
    g = torch.Generator().manual_seed(seed)
    x = torch.rand(shape, generator=g)
    flat = x.view(-1)
    k = flat.numel()
    flat[torch.randperm(k, generator=g)[: max(1, k // 16)]] = 0.0
    flat[torch.randperm(k, generator=g)[: max(1, k // 16)]] = 1.0
    flat[torch.randperm(k, generator=g)[: max(1, k // 32)]] = float(np.nextafter(np.float32(1), np.float32(0)))
    return x


def digest(a):
    return np.frombuffer(hashlib.sha256(np.ascontiguousarray(a).tobytes()).digest(), dtype=np.uint8)


# ---- the engine's noise (csrc/rgb_noise.cu), restated in numpy: Philox4x32-10 and Box-Muller in float64

def philox4x32_10(c0, c1, c2, c3, k0, k1):
    """Vectorised Philox4x32-10 over uint64 arrays holding 32-bit words."""
    M = np.uint64(0xFFFFFFFF)
    c = [np.asarray(v, dtype=np.uint64) & M for v in (c0, c1, c2, c3)]
    k0, k1 = np.uint64(k0), np.uint64(k1)
    for _ in range(10):
        p0 = np.uint64(0xD2511F53) * c[0]
        p1 = np.uint64(0xCD9E8D57) * c[2]
        c = [((p1 >> np.uint64(32)) ^ c[1] ^ k0) & M, p1 & M, ((p0 >> np.uint64(32)) ^ c[3] ^ k1) & M, p0 & M]
        k0 = (k0 + np.uint64(0x9E3779B9)) & M
        k1 = (k1 + np.uint64(0xBB67AE85)) & M
    return c


def philox_normal(seed, elem, stream, frame, offset):
    r = philox4x32_10(elem, stream, frame, offset, seed & 0xFFFFFFFF, (seed >> 32) & 0xFFFFFFFF)
    u1 = ((r[0] >> np.uint64(9)).astype(np.float64) + 0.5) * 2.0 ** -23
    a = (r[1] >> np.uint64(8)).astype(np.float64) * 2.0 ** -23
    return np.sqrt(-2.0 * np.log(u1)) * np.cos(np.pi * a)


def engine_noise(seed, offset, level, shape):
    """What nb200_rgb_noise returns for (seed, offset, level), in float64: shape (C, H, W) or (B, C, H, W)."""
    B, C, H, W = (1,) + tuple(shape) if len(shape) == 3 else tuple(shape)
    b, c, y, x = np.meshgrid(np.arange(B), np.arange(C), np.arange(H), np.arange(W), indexing="ij")
    n = philox_normal(seed, y * W + x, 2 * c, b, offset)
    if level == 2:
        hy, hx = nearest_index(H, H // 2)[y], nearest_index(W, W // 2)[x]
        n = 0.5 * n + 0.5 * philox_normal(seed, hy * (W // 2) + hx, 2 * c + 1, b, offset)
    return n.reshape(shape)
