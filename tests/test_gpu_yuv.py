"""GPU: the planar YUV <-> integer RGB kernels (csrc/yuv.cu) against the float64 oracle (oracle/yuv.py), the libswscale
frames of tests/golden/yuv.npz (reported, not gated), and FrameBatchPipeline's source= / target= stages against the RGB
pipeline fed with the oracle's frames."""
import itertools
import types
from argparse import Namespace

import numpy as np
import pytest
import torch

from oracle import yuv as oy
from tests.util import load_golden, log_metric

pytestmark = pytest.mark.gpu
DEV = "cuda:0"
MATRICES = {"bt601": 5, "bt709": 1, "bt2020": 9}
RANGES = {0: 1, 1: 2}           # oracle full flag -> PyAV color_range (MPEG, JPEG)
SIZES = [(1, 1), (23, 37), (1080, 1920)]


def _layout(pix_fmt):
    from nunif_b200.nunif.video import YUV_SOURCE_FORMATS, YUV_TARGET_FORMATS
    return (YUV_SOURCE_FORMATS.get(pix_fmt) or YUV_TARGET_FORMATS[pix_fmt])


def _compare(got, want, name, acc):
    d = np.abs(got.astype(np.int64) - want.astype(np.int64))
    assert d.max() <= 1, (name, int(d.max()))
    acc[0] += int((d != 0).sum())
    acc[1] += d.size
    acc[2] = max(acc[2], int(d.max()))


@pytest.mark.parametrize("pix_fmt", ["yuv420p", "yuvj420p", "yuv422p", "yuv444p", "yuv420p10le", "yuv422p10le", "yuv444p10le"])
def test_yuv_to_rgb_vs_oracle(pix_fmt):
    from nunif_b200.nunif.video import yuv_to_rgb
    layout, bits = _layout(pix_fmt)
    sx, sy = oy.SUBSAMPLING[layout]
    rng = np.random.default_rng(bits)
    for m, full in itertools.product(MATRICES, RANGES):
        acc = [0, 0, 0]
        for H, W in SIZES:
            dt = np.uint16 if bits > 8 else np.uint8
            chroma = (-(-H // sy), -(-W // sx))
            batch = [oy.pack([rng.integers(0, 1 << bits, s).astype(dt) for s in [(H, W), chroma, chroma]], W) for _ in range(2)]
            got = yuv_to_rgb(torch.from_numpy(np.stack(batch)), pix_fmt, MATRICES[m], RANGES[full], use_16bit=bits > 8,
                             device=DEV).cpu().numpy()
            for b, a in enumerate(batch):
                want = oy.yuv_to_rgb(*oy.unpack(a, layout, H, W), layout, bits, m, full, 16 if bits > 8 else 8)
                _compare(got[b], want, (pix_fmt, m, full, H, W, b), acc)
        log_metric(f"yuv/y2r/{pix_fmt}/{m}/{full}", mismatched=acc[0], total=acc[1], max=acc[2])
        assert acc[0] <= acc[1] * 1e-3, (pix_fmt, m, full, acc)


@pytest.mark.parametrize("pix_fmt", ["yuv420p", "yuvj420p", "yuv444p", "yuvj444p", "yuv420p10le", "gbrp", "gbrp10le", "gbrp16le"])
def test_rgb_to_yuv_vs_oracle(pix_fmt):
    from nunif_b200.nunif.video import rgb_to_yuv, plane_shape
    layout, bits = _layout(pix_fmt)
    rgb_bits = 16 if bits > 8 else 8
    rng = np.random.default_rng(bits + 1)
    configs = [("bt709", 0)] if layout == "gbr" else list(itertools.product(MATRICES, RANGES))
    for m, full in configs:
        acc = [0, 0, 0]
        for H, W in SIZES:
            rgb = rng.integers(0, 1 << rgb_bits, (2, H, W, 3)).astype(np.uint16 if rgb_bits > 8 else np.uint8)
            got = rgb_to_yuv(torch.from_numpy(rgb).to(DEV), pix_fmt, MATRICES[m], RANGES[full]).cpu().numpy()
            assert got.shape == (2,) + plane_shape(pix_fmt, H, W)
            for b in range(2):
                if layout == "gbr":
                    planes = oy.rgb_to_gbr(rgb[b], rgb_bits, bits)
                else:
                    planes = oy.rgb_to_yuv(rgb[b], rgb_bits, layout, bits, m, full)
                _compare(got[b], oy.pack(planes, W), (pix_fmt, m, full, H, W, b), acc)
        log_metric(f"yuv/r2y/{pix_fmt}/{m}/{full}", mismatched=acc[0], total=acc[1], max=acc[2])
        assert acc[0] <= acc[1] * 1e-3, (pix_fmt, m, full, acc)


def test_swscale_frames_report():
    """libswscale's conversions of the golden frames (another FFmpeg build than PyAV's): logged, not gated."""
    from nunif_b200.nunif.video import rgb_to_yuv, yuv_to_rgb
    g = load_golden("yuv")
    print("libswscale", g["swscale/version"])
    for key in sorted(k for k in g if k.startswith("swscale/") and not k.endswith("/in") and k != "swscale/version"):
        _, kind, pix_fmt, m, full = key.split("/")
        cs, cr = MATRICES.get(m, 1), RANGES[int(full)]
        src = torch.from_numpy(g[f"swscale/{kind}/{pix_fmt}/in"])
        if kind == "y2r":
            got = yuv_to_rgb(src, pix_fmt, cs, cr, use_16bit=pix_fmt.endswith("10le"), device=DEV)
        else:
            got = rgb_to_yuv(src.to(DEV), pix_fmt, cs, cr)
        d = (got.cpu().numpy().astype(np.int64) - g[key].astype(np.int64))
        log_metric(f"yuv/swscale/{kind}/{pix_fmt}/{m}/{full}", max=int(np.abs(d).max()), mean=float(np.abs(d).mean()))
        assert got.shape == g[key].shape


# ---- pipeline
SRC = ("yuv420p", 1, 1)                     # BT.709 limited
FRAME_SIZES = [(72, 128)] * 5 + [(54, 96)] * 4   # 9 frames, batch 4: a size change inside the second batch, a partial last


def _rgb_frames(bits, seed=0):
    from nunif_b200 import synth
    frames = []
    for i, (H, W) in enumerate(FRAME_SIZES):
        x = synth.synth_image(seed + i, 3, H, W).permute(1, 2, 0)
        frames.append((x * (65535 if bits > 8 else 255)).round().to(torch.uint16 if bits > 8 else torch.uint8).numpy())
    return frames


def _as_source(frames, fmt):
    """Planes of each RGB frame (through the oracle) and the oracle's RGB frame decoded back from them."""
    from nunif_b200.nunif.video import _YuvFormat, YUV_SOURCE_FORMATS
    f = _YuvFormat(fmt, YUV_SOURCE_FORMATS, "source")
    layout = {0: "420", 1: "422", 2: "444"}[f.layout]
    m = {0: "bt601", 1: "bt709", 2: "bt2020"}[f.matrix]
    rgb_bits = 16 if f.bits > 8 else 8
    planes, rgb = [], []
    for x in frames:
        p = oy.rgb_to_yuv(x, rgb_bits, layout, f.bits, m, f.range)
        planes.append(torch.from_numpy(oy.pack(p, x.shape[1])))
        rgb.append(torch.from_numpy(oy.yuv_to_rgb(*p, layout, f.bits, m, f.range, rgb_bits)))
    return planes, rgb


def _run(pipe, frames):
    out = []
    for f in frames:
        out += pipe(f)
    return out + pipe.finish()


def _iw3_factory(pix_fmt):
    from nunif_b200.iw3 import bind_batch_frame_callback
    from nunif_b200.iw3.null_depth_model import NullDepthModel

    def make():
        dm = NullDepthModel("NULL").load(gpu=0)
        dm.disable_ema()
        args = Namespace(method="forward_fill", divergence=2.0, convergence=0.5, synthetic_view="both", ipd_offset=0,
                         mapper="none", edge_dilation=0, tta=False, low_vram=False, disable_amp=False, depth_aa=False,
                         rotate_left=False, rotate_right=False, max_output_height=None, max_output_width=None,
                         keep_aspect_ratio=False, pad=None, pad_mode=None, vr180=False, half_sbs=False, tb=False,
                         half_tb=False, cross_eyed=False, anaglyph=None, rgbd=False, half_rgbd=False, debug_depth=False,
                         preserve_screen_border=False, pix_fmt=pix_fmt, batch_size=4, cuda_stream=False, stereo_width=None,
                         warp_steps=None, state={"device": DEV, "convergence_model": None})
        cb = bind_batch_frame_callback(dm, None, set(), args)
        pts = itertools.count()
        return lambda x: cb(x, [next(pts) for _ in range(x.shape[0])], False)
    return make


class _StubCtx:
    def convert(self, x, alpha, method, noise_level, tile_size=None, batch_size=None, tta=False, enable_amp=True,
                output_device="cpu"):
        return (x * 0.8 + 0.1).to(output_device), alpha


def _waifu2x_pipe(use_16bit, grain, **kw):
    from nunif_b200.waifu2x.ui_utils import make_video_pipeline
    args = types.SimpleNamespace(rotate_left=False, rotate_right=False, method="scale", noise_level=0, tile_size=64,
                                 batch_size=1, tta=False, disable_amp=False, grain=grain, grain_strength=0.3,
                                 grain_speed=0.6, state={"device": torch.device(DEV)})
    return make_video_pipeline(_StubCtx(), args, batch_size=4, use_16bit=use_16bit, seed=17, **kw)


def _check(path, source, target, bits, hdr2sdr=None, grain=False):
    from nunif_b200.nunif.video import FrameBatchPipeline, rgb_to_yuv
    use_16bit = bits > 8
    frames = _rgb_frames(bits)
    planes, rgb = _as_source(frames, source) if source else (None, [torch.from_numpy(f) for f in frames])

    def pipe(**kw):
        if path == "iw3":
            return FrameBatchPipeline(_iw3_factory("yuv420p10le" if use_16bit else "yuv420p")(), 4, DEV,
                                      use_16bit=use_16bit, hdr2sdr=hdr2sdr, **kw)
        return _waifu2x_pipe(use_16bit, grain, **kw)

    want = _run(pipe(), rgb)
    got = _run(pipe(source=source, target=target), planes if source else rgb)
    assert len(got) == len(want) == len(frames)
    for i, (g, w) in enumerate(zip(got, want)):
        if target is not None:
            w = rgb_to_yuv(w.to(DEV), *target).cpu()
        assert g.shape == w.shape and g.dtype == w.dtype, (i, g.shape, w.shape)
        assert torch.equal(g, w), (path, i, int((g.int() - w.int()).abs().max()))


@pytest.mark.parametrize("path", ["iw3", "waifu2x"])
@pytest.mark.parametrize("source,target", [(SRC, None), (None, ("yuv420p", 1, 1)), (SRC, ("yuv420p", 1, 1))])
def test_pipeline_8bit(path, source, target):
    _check(path, source, target, 8)


def test_pipeline_10bit_hdr2sdr():
    """PQ BT.2020 yuv420p10le in, tone-mapped to BT.709 by hdr2sdr=, through the iw3 callback, written as yuv420p10le
    BT.709 limited."""
    _check("iw3", ("yuv420p10le", 9, 1), ("yuv420p10le", 1, 1), 10, hdr2sdr=(16, "bt709"))


@pytest.mark.parametrize("bits", [8, 10])
def test_pipeline_grain(bits):
    src = SRC if bits == 8 else ("yuv420p10le", 1, 2)
    tgt = ("yuv420p", 1, 1) if bits == 8 else ("yuv420p10le", 9, 1)
    _check("waifu2x", src, tgt, bits, grain=True)
