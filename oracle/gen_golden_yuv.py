"""Generate tests/golden/yuv.npz: the reference's colour policy over a grid of input streams, and a libswscale comparison.

policy  The REAL nunif/utils/video.py guess_color_range, guess_colorspace, guess_rgb24_options, guess_target_colorspace and
        configure_colorspace (its rgb24_options and the reformat() arguments of its reformatter), run with the stand-in
        `av` module of oracle/gen_golden_hdr2sdr.py on stand-in streams: every pix_fmt of YUV_SOURCE_FORMATS x codec colorspace
        unspecified / 601 / 709 / 2020 x codec range unspecified / MPEG / JPEG x height 480 / 720 / 2160, under every
        --colorspace value and every --pix-fmt of PIX_FMTS.  Integer table, one row per case (POLICY_COLUMNS; None = -1).
swscale Seeded in-gamut 32 x 16 frames through libswscale (sws_getContext + sws_setColorspaceDetails + sws_scale, SWS_BILINEAR as PyAV
        uses it), loaded by ctypes from the OpenCV wheel's bundled FFmpeg libraries.  Not PyAV's own FFmpeg build, so the
        tests only report the difference to the engine.  swscale/version holds av_version_info() and swscale_version().

Run from the repository root, as a module:
    PYTHONDONTWRITEBYTECODE=1 PYTHONPATH=<nunif checkout> python -m oracle.gen_golden_yuv
"""
import ctypes
import glob
import os
import types

import numpy as np

from oracle import yuv as oy
from oracle.gen_golden_hdr2sdr import install_av_stub

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
OUT = os.path.join(ROOT, "tests", "golden", "yuv.npz")

SOURCE_PIX_FMTS = ["yuv420p", "yuvj420p", "yuv422p", "yuv444p", "yuv420p10le", "yuv422p10le", "yuv444p10le"]
COLORSPACE_ARGS = ["unspecified", "auto", "copy", "bt709", "bt709-tv", "bt709-pc", "bt601", "bt601-tv", "bt601-pc",
                   "bt2020", "bt2020-tv", "bt2020-pc", "bt2020-pq-tv"]
PIX_FMTS = ["yuv420p", "yuv444p", "yuv420p10le", "gbrp", "gbrp10le", "gbrp16le", "rgb24",
            "yuvj420p", "yuvj444p", "rgb48le"]       # the last three only ever appear as outputs
STREAM_COLORSPACES = [2, 5, 1, 9]
STREAM_RANGES = [0, 1, 2]
HEIGHTS = [480, 720, 2160]
POLICY_COLUMNS = [
    # inputs
    "src_pix_fmt", "stream_colorspace", "stream_range", "height", "colorspace_arg", "pix_fmt_arg",
    # guess_color_range(stream), guess_colorspace(stream)
    "guess_color_range", "guess_colorspace",
    # guess_target_colorspace(stream, colorspace_arg, pix_fmt_arg); -2 = it raised
    "t_primaries", "t_trc", "t_colorspace", "t_range", "t_pix_fmt",
    # configure_colorspace: config.pix_fmt after it, state["rgb24_options"], the reformatter's reformat() kwargs
    "cfg_pix_fmt", "rgb_present", "rgb_format", "rgb_src_range", "rgb_dst_range", "rgb_src_colorspace", "rgb_dst_colorspace",
    "ref_present", "ref_format", "ref_src_colorspace", "ref_dst_colorspace", "ref_src_range", "ref_dst_range",
]
# guess_rgb24_options(stream, t) for each t of RGB24_TARGETS, per stream: present, format, src/dst range, src/dst colorspace
RGB24_TARGETS = [2, 1, 5, 9]
RGB_FORMATS = ["rgb24", "rgb48le"]


class Stream:
    def __init__(self, pix_fmt, colorspace, color_range, height):
        self.pix_fmt = pix_fmt
        self.height = height
        self.width = height * 16 // 9
        bits = 10 if pix_fmt.endswith("10le") else 8
        self.format = types.SimpleNamespace(components=[types.SimpleNamespace(bits=bits)])
        self.codec_context = types.SimpleNamespace(colorspace=colorspace, color_range=color_range, color_primaries=colorspace,
                                                   color_trc=16 if colorspace == 9 else 1)


class OutputStream:
    def __init__(self):
        self.codec_context = types.SimpleNamespace(colorspace=None, color_range=None, color_primaries=None, color_trc=None)


class RecordingFrame:
    def reformat(self, **kw):
        return kw


def _i(v):
    return -1 if v is None else int(v)


def _rgb24_row(opts):
    if not opts:
        return [0, -1, -1, -1, -1, -1]
    return [1, RGB_FORMATS.index(opts["format"]), _i(opts["src_color_range"]), _i(opts["dst_color_range"]),
            _i(opts["src_colorspace"]), _i(opts["dst_colorspace"])]


def policy_table(VU):
    rows, rgb24 = [], []
    for pi, pix_fmt in enumerate(SOURCE_PIX_FMTS):
        for cs in STREAM_COLORSPACES:
            for cr in STREAM_RANGES:
                for h in HEIGHTS:
                    s = Stream(pix_fmt, cs, cr, h)
                    rgb24.append(sum((_rgb24_row(VU.guess_rgb24_options(s, t)) for t in RGB24_TARGETS), []))
                    for ai, arg in enumerate(COLORSPACE_ARGS):
                        for fi, pf in enumerate(PIX_FMTS[:7]):
                            row = [pi, cs, cr, h, ai, fi, _i(VU.guess_color_range(s)), _i(VU.guess_colorspace(s))]
                            try:
                                t = VU.guess_target_colorspace(s, arg, pf)
                                row += [_i(v) for v in t[:4]] + [PIX_FMTS.index(t[4])]
                            except UnboundLocalError:        # "unspecified" names no target (configure returns first)
                                row += [-2] * 5
                            config = VU.VideoOutputConfig(pix_fmt=pf, colorspace=arg)
                            VU.configure_colorspace(OutputStream(), s, config)
                            row += [PIX_FMTS.index(config.pix_fmt)] + _rgb24_row(config.state["rgb24_options"])
                            kw = config.state["reformatter"](RecordingFrame())
                            if isinstance(kw, RecordingFrame):
                                row += [0, -1, -1, -1, -1, -1]
                            else:
                                row += [1, PIX_FMTS.index(kw["format"]), _i(kw["src_colorspace"]), _i(kw["dst_colorspace"]),
                                        _i(kw["src_color_range"]), _i(kw["dst_color_range"])]
                            rows.append(row)
    return np.array(rows, np.int16), np.array(rgb24, np.int16)


# ---- libswscale
SWS_BILINEAR = 2
W, H = 32, 16
SWS_SOURCES = SOURCE_PIX_FMTS
SWS_TARGETS = ["yuv420p", "yuv444p", "yuv420p10le", "gbrp", "gbrp10le", "gbrp16le"]
SWS_MATRICES = {"bt601": 5, "bt709": 1, "bt2020": 9}


def load_swscale():
    import cv2
    libdir = glob.glob(os.path.join(os.path.dirname(cv2.__file__), "..", "opencv_python*.libs"))[0]
    for dep in ("libdrm", "libcrypto", "libavutil", "libswscale"):
        ctypes.CDLL(glob.glob(os.path.join(libdir, dep + "-*.so*"))[0], mode=ctypes.RTLD_GLOBAL)
    avutil = ctypes.CDLL(glob.glob(os.path.join(libdir, "libavutil-*.so*"))[0])
    sws = ctypes.CDLL(glob.glob(os.path.join(libdir, "libswscale-*.so*"))[0])
    avutil.av_get_pix_fmt.restype = ctypes.c_int
    avutil.av_get_pix_fmt.argtypes = [ctypes.c_char_p]
    avutil.av_version_info.restype = ctypes.c_char_p
    sws.swscale_version.restype = ctypes.c_uint
    sws.sws_getContext.restype = ctypes.c_void_p
    sws.sws_getContext.argtypes = [ctypes.c_int] * 7 + [ctypes.c_void_p] * 3
    sws.sws_getCoefficients.restype = ctypes.c_void_p
    sws.sws_getCoefficients.argtypes = [ctypes.c_int]
    sws.sws_setColorspaceDetails.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_void_p, ctypes.c_int,
                                             ctypes.c_int, ctypes.c_int, ctypes.c_int]
    sws.sws_scale.argtypes = [ctypes.c_void_p, ctypes.c_void_p, ctypes.c_void_p, ctypes.c_int, ctypes.c_int, ctypes.c_void_p,
                              ctypes.c_void_p]
    sws.sws_freeContext.argtypes = [ctypes.c_void_p]
    return avutil, sws


def sws_convert(avutil, sws, src_fmt, src_planes, dst_fmt, dst_shapes, dtype_out, colorspace, full):
    """One sws_scale of planar / packed numpy arrays; colorspace and range apply to whichever side is YUV."""
    sf, df = avutil.av_get_pix_fmt(src_fmt.encode()), avutil.av_get_pix_fmt(dst_fmt.encode())
    assert sf >= 0 and df >= 0, (src_fmt, dst_fmt)
    ctx = sws.sws_getContext(W, H, sf, W, H, df, SWS_BILINEAR, None, None, None)
    assert ctx
    coef = sws.sws_getCoefficients(colorspace)
    src_is_rgb = src_fmt.startswith("rgb")
    sws.sws_setColorspaceDetails(ctx, coef, 1 if (full or src_is_rgb) else 0, coef, 1 if (full or not src_is_rgb) else 0,
                                 0, 1 << 16, 1 << 16)
    src = [np.ascontiguousarray(p) for p in src_planes]
    dst = [np.zeros(s, dtype_out) for s in dst_shapes]
    sp = (ctypes.c_void_p * 4)(*[p.ctypes.data for p in src] + [None] * (4 - len(src)))
    ss = (ctypes.c_int * 4)(*[p.strides[0] for p in src] + [0] * (4 - len(src)))
    dp = (ctypes.c_void_p * 4)(*[p.ctypes.data for p in dst] + [None] * (4 - len(dst)))
    ds = (ctypes.c_int * 4)(*[p.strides[0] for p in dst] + [0] * (4 - len(dst)))
    n = sws.sws_scale(ctx, sp, ss, 0, H, dp, ds)
    sws.sws_freeContext(ctx)
    assert n == H, n
    return dst


def swscale_cases():
    avutil, sws = load_swscale()
    rng = np.random.default_rng(2024)
    out = {"swscale/version": np.array(f"{avutil.av_version_info().decode()} swscale {sws.swscale_version() >> 16}."
                                        f"{(sws.swscale_version() >> 8) & 255}.{sws.swscale_version() & 255}")}
    for pix_fmt in SWS_SOURCES:
        bits = 10 if pix_fmt.endswith("10le") else 8
        sx, sy = oy.SUBSAMPLING[{"yuv420p": "420", "yuvj420p": "420", "yuv422p": "422", "yuv444p": "444"}.get(
            pix_fmt.replace("10le", ""), "420")]
        dt = np.uint16 if bits > 8 else np.uint8
        # in-gamut planes: a seeded rgb24 frame through the oracle's BT.709 limited-range conversion (random YUV codes
        # are mostly outside the RGB cube, where libswscale's 10-bit paths wrap instead of clamping)
        layout = {(2, 2): "420", (2, 1): "422", (1, 1): "444"}[(sx, sy)]
        y, u, v = oy.rgb_to_yuv(rng.integers(0, 256, (H, W, 3)).astype(np.uint8), 8, layout, bits, "bt709", 0)
        out[f"swscale/y2r/{pix_fmt}/in"] = oy.pack([y, u, v], W)
        for mname, cs in SWS_MATRICES.items():
            for full in (0, 1):
                rgb_fmt = "rgb48le" if bits > 8 else "rgb24"
                (rgb,) = sws_convert(avutil, sws, pix_fmt, [y, u, v], rgb_fmt, [(H, W * 3)], dt if bits == 8 else np.uint16,
                                     cs, full)
                out[f"swscale/y2r/{pix_fmt}/{mname}/{full}"] = rgb.reshape(H, W, 3)
    for target in SWS_TARGETS:
        rgb_bits = 16 if target.endswith("le") else 8
        dt_in = np.uint16 if rgb_bits > 8 else np.uint8
        rgb = rng.integers(0, 1 << rgb_bits, (H, W, 3)).astype(dt_in)
        out[f"swscale/r2y/{target}/in"] = rgb
        bits = 16 if target == "gbrp16le" else 10 if target.endswith("10le") else 8
        dt = np.uint16 if bits > 8 else np.uint8
        if target.startswith("gbrp"):
            shapes, configs = [(H, W)] * 3, [("none", 1, 1)]
        else:
            sx, sy = (1, 1) if target == "yuv444p" else (2, 2)
            shapes = [(H, W), (H // sy, W // sx), (H // sy, W // sx)]
            configs = [(m, cs, f) for m, cs in SWS_MATRICES.items() for f in (0, 1)]
        for mname, cs, full in configs:
            planes = sws_convert(avutil, sws, "rgb48le" if rgb_bits > 8 else "rgb24", [rgb.reshape(H, W * 3)], target, shapes,
                                 dt, cs, full)
            out[f"swscale/r2y/{target}/{mname}/{full}"] = oy.pack(planes, W)
    return out


def main():
    install_av_stub()
    import nunif.utils.video as VU
    table, rgb24 = policy_table(VU)
    out = {"policy/table": table, "policy/columns": np.array(POLICY_COLUMNS), "policy/rgb24": rgb24,
           "policy/rgb24_targets": np.array(RGB24_TARGETS), "policy/source_pix_fmts": np.array(SOURCE_PIX_FMTS),
           "policy/colorspace_args": np.array(COLORSPACE_ARGS), "policy/pix_fmts": np.array(PIX_FMTS),
           "policy/rgb_formats": np.array(RGB_FORMATS)}
    out.update(swscale_cases())
    np.savez_compressed(OUT, **out)
    print(OUT, os.path.getsize(OUT), table.shape, out["swscale/version"])


if __name__ == "__main__":
    main()
