"""float64 restatement of the engine's planar YUV <-> integer RGB conversions (csrc/yuv.cu, nunif_b200.nunif.video
yuv_to_rgb / rgb_to_yuv): the reference for the GPU tests.

Y'CbCr from ITU-R BT.601 / BT.709 / BT.2020 (non-constant luminance), with Kg = 1 - Kr - Kb:
    Y' = Kr R + Kg G + Kb B,   Cb = (B - Y') / (2 (1 - Kb)),   Cr = (R - Y') / (2 (1 - Kr))      (R, G, B in [0, 1])
codes at depth n (s = 2^(n-8)):
    limited (MPEG): Y = 16 s + 219 s Y',   C = 128 s + 224 s C
    full (JPEG):    Y = (2^n - 1) Y',      C = 2^(n-1) + (2^n - 1) C
RGB is full range, rgb24 (255) or rgb48 (65535).  yuv -> rgb replicates each chroma sample over its luma block; rgb -> yuv
gives each chroma sample the mean of the unrounded Cb / Cr of the pixels of its block that exist.  Round half to even,
clamp to the code range.  Frames are (Y [H][W], U [ch][cw], V [ch][cw]) numpy arrays here, cw = ceil(W/sx), ch = ceil(H/sy).
"""
import numpy as np

KR_KB = {"bt601": (0.299, 0.114), "bt709": (0.2126, 0.0722), "bt2020": (0.2627, 0.0593)}
SUBSAMPLING = {"420": (2, 2), "422": (2, 1), "444": (1, 1)}


def rgb_to_ycbcr_matrix(matrix):
    """3 x 3 float64 M with (Y', Cb, Cr) = M (R, G, B)."""
    kr, kb = KR_KB[matrix]
    kg = 1.0 - kr - kb
    return np.array([[kr, kg, kb],
                     [-kr / (2 * (1 - kb)), -kg / (2 * (1 - kb)), 0.5],
                     [0.5, -kg / (2 * (1 - kr)), -kb / (2 * (1 - kr))]])


def _range(bits, full):
    s, vmax = 2.0 ** (bits - 8), 2.0 ** bits - 1
    if full:
        return 0.0, vmax, 2.0 ** (bits - 1), vmax           # y offset, y span, chroma zero, chroma span
    return 16 * s, 219 * s, 128 * s, 224 * s


def _code(v, vmax):
    return np.clip(np.rint(v), 0, vmax)


def yuv_to_rgb(y, u, v, layout, bits, matrix, full, rgb_bits):
    """(Y, U, V) integer planes -> HWC RGB codes (uint8 for rgb_bits 8, uint16 for 16)."""
    sx, sy = SUBSAMPLING[layout]
    H, W = y.shape
    yo, ys, co, cs = _range(bits, full)
    yn = (y.astype(np.float64) - yo) / ys
    cb = (u.astype(np.float64) - co) / cs
    cr = (v.astype(np.float64) - co) / cs
    cb = np.repeat(np.repeat(cb, sy, axis=0), sx, axis=1)[:H, :W]
    cr = np.repeat(np.repeat(cr, sy, axis=0), sx, axis=1)[:H, :W]
    rgb = np.stack([yn, cb, cr], axis=-1) @ np.linalg.inv(rgb_to_ycbcr_matrix(matrix)).T
    omax = 2.0 ** rgb_bits - 1
    return _code(rgb * omax, omax).astype(np.uint16 if rgb_bits > 8 else np.uint8)


def _block_mean(c, sx, sy):
    H, W = c.shape
    ch, cw = -(-H // sy), -(-W // sx)
    pad = np.pad(c, ((0, ch * sy - H), (0, cw * sx - W)))
    cnt = np.pad(np.ones_like(c), ((0, ch * sy - H), (0, cw * sx - W)))
    s = pad.reshape(ch, sy, cw, sx).sum(axis=(1, 3))
    n = cnt.reshape(ch, sy, cw, sx).sum(axis=(1, 3))
    return s / n


def rgb_to_yuv(rgb, rgb_bits, layout, bits, matrix, full):
    """HWC RGB codes -> (Y, U, V) integer planes (uint8 for 8-bit, uint16 above)."""
    sx, sy = SUBSAMPLING[layout]
    yo, ys, co, cs = _range(bits, full)
    x = rgb.astype(np.float64) / (2.0 ** rgb_bits - 1)
    ycc = x @ rgb_to_ycbcr_matrix(matrix).T
    vmax = 2.0 ** bits - 1
    dt = np.uint16 if bits > 8 else np.uint8
    y = _code(yo + ys * ycc[..., 0], vmax).astype(dt)
    u = _code(co + cs * _block_mean(ycc[..., 1], sx, sy), vmax).astype(dt)
    v = _code(co + cs * _block_mean(ycc[..., 2], sx, sy), vmax).astype(dt)
    return y, u, v


def rgb_to_gbr(rgb, rgb_bits, bits):
    """HWC RGB codes -> the (G, B, R) planes of gbrp / gbrp10le / gbrp16le, each code rescaled to ``bits``."""
    vmax = 2.0 ** bits - 1
    x = _code(rgb.astype(np.float64) * (vmax / (2.0 ** rgb_bits - 1)), vmax).astype(np.uint16 if bits > 8 else np.uint8)
    return x[..., 1], x[..., 2], x[..., 0]


def pack(planes, W):
    """Concatenate planes into the engine's (rows, W) frame array, zero-padded to a whole row."""
    flat = np.concatenate([p.reshape(-1) for p in planes])
    rows = -(-flat.size // W)
    return np.concatenate([flat, np.zeros(rows * W - flat.size, flat.dtype)]).reshape(rows, W)


def unpack(arr, layout, H, W):
    """The (Y, U, V) planes of an engine frame array."""
    sx, sy = SUBSAMPLING.get(layout, (1, 1))
    ch, cw = -(-H // sy), -(-W // sx)
    flat = np.asarray(arr).reshape(-1)
    return flat[:H * W].reshape(H, W), flat[H * W:H * W + ch * cw].reshape(ch, cw), \
        flat[H * W + ch * cw:H * W + 2 * ch * cw].reshape(ch, cw)
