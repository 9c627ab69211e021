"""CPU: the colour policy mirror of nunif_b200.nunif.video against the reference's own functions (tests/golden/yuv.npz),
the float64 YUV oracle (oracle/yuv.py), and the argument checks of yuv_to_rgb / rgb_to_yuv / FrameBatchPipeline."""
import types

import numpy as np
import pytest
import torch

from oracle import yuv as oy
from tests.util import load_golden


@pytest.fixture(scope="module")
def golden():
    return load_golden("yuv")


def _stream(pix_fmt, colorspace, color_range, height):
    bits = 10 if pix_fmt.endswith("10le") else 8
    return types.SimpleNamespace(
        pix_fmt=pix_fmt, height=height, format=types.SimpleNamespace(components=[types.SimpleNamespace(bits=bits)]),
        codec_context=types.SimpleNamespace(colorspace=colorspace, color_range=color_range, color_primaries=colorspace,
                                            color_trc=16 if colorspace == 9 else 1))


def _i(v):
    return -1 if v is None else int(v)


def test_policy_mirror_equals_reference(golden):
    """Every (stream, --colorspace, --pix-fmt) case of the grid: guess_color_range, guess_colorspace,
    guess_target_colorspace and the rgb24_options / reformatter that configure_colorspace picks."""
    from nunif_b200.nunif import video as V
    cols = [str(c) for c in golden["policy/columns"]]
    src_fmts, args_, pix_fmts = (list(map(str, golden[k])) for k in
                                 ("policy/source_pix_fmts", "policy/colorspace_args", "policy/pix_fmts"))
    rgb_formats = list(map(str, golden["policy/rgb_formats"]))
    table = golden["policy/table"]
    assert len(table) == 7 * 4 * 3 * 3 * 13 * 7
    checked_source = checked_target = 0
    for row in table:
        r = dict(zip(cols, (int(v) for v in row)))
        s = _stream(src_fmts[r["src_pix_fmt"]], r["stream_colorspace"], r["stream_range"], r["height"])
        arg, pf = args_[r["colorspace_arg"]], pix_fmts[r["pix_fmt_arg"]]
        assert _i(V.guess_color_range(s)) == r["guess_color_range"], r
        assert _i(V.guess_colorspace(s)) == r["guess_colorspace"], r
        if r["t_pix_fmt"] == -2:
            with pytest.raises(ValueError):
                V.guess_target_colorspace(s, arg, pf)
        else:
            t = V.guess_target_colorspace(s, arg, pf)
            assert [_i(v) for v in t[:4]] + [pix_fmts.index(t[4])] == \
                [r["t_primaries"], r["t_trc"], r["t_colorspace"], r["t_range"], r["t_pix_fmt"]], r
        out_fmt, source, target = V.configure_colorspace(s, arg, pf)
        assert pix_fmts.index(out_fmt) == r["cfg_pix_fmt"], r
        if r["rgb_present"]:
            assert source == (s.pix_fmt, r["rgb_src_colorspace"], r["rgb_src_range"]), r
            assert rgb_formats[r["rgb_format"]] == ("rgb48le" if V.pix_fmt_requires_16bit(s.pix_fmt) else "rgb24")
            checked_source += 1
        else:
            assert source is None, r
        if r["ref_present"]:
            assert target == (pix_fmts[r["ref_format"]], r["ref_dst_colorspace"], r["ref_dst_range"]), r
            # the reformatter's RGB side is always what rgb24_options produced: full range, of the rgb24 dst colorspace
            assert r["ref_src_range"] == 2 and r["ref_src_colorspace"] == r["rgb_dst_colorspace"], r
            checked_target += 1
        else:
            assert target is None, r
    assert checked_source > 10000 and checked_target > 10000


def test_rgb24_options_mirror(golden):
    from nunif_b200.nunif import video as V
    src_fmts = list(map(str, golden["policy/source_pix_fmts"]))
    rgb_formats = list(map(str, golden["policy/rgb_formats"]))
    targets = [int(t) for t in golden["policy/rgb24_targets"]]
    i = 0
    for pix_fmt in src_fmts:
        for cs in (2, 5, 1, 9):
            for cr in (0, 1, 2):
                for h in (480, 720, 2160):
                    s = _stream(pix_fmt, cs, cr, h)
                    want = golden["policy/rgb24"][i].reshape(len(targets), 6)
                    for t, w in zip(targets, want):
                        o = V.guess_rgb24_options(s, t)
                        got = [1, rgb_formats.index(o["format"]), o["src_color_range"], o["dst_color_range"],
                               o["src_colorspace"], o["dst_colorspace"]] if o else [0, -1, -1, -1, -1, -1]
                        assert got == [int(v) for v in w], (pix_fmt, cs, cr, h, t)
                    i += 1
    assert i == len(golden["policy/rgb24"])


@pytest.mark.parametrize("matrix", ["bt601", "bt709", "bt2020"])
def test_oracle_matrices_are_itu_tables(matrix):
    """Rows of the RGB -> Y'CbCr matrix as ITU-R BT.601-7, BT.709-6 and BT.2020-2 print them (4 decimals)."""
    itu = {"bt601": [[0.299, 0.587, 0.114], [-0.1687, -0.3313, 0.5], [0.5, -0.4187, -0.0813]],
           "bt709": [[0.2126, 0.7152, 0.0722], [-0.1146, -0.3854, 0.5], [0.5, -0.4542, -0.0458]],
           "bt2020": [[0.2627, 0.6780, 0.0593], [-0.1396, -0.3604, 0.5], [0.5, -0.4598, -0.0402]]}[matrix]
    m = oy.rgb_to_ycbcr_matrix(matrix)
    np.testing.assert_allclose(m, itu, atol=5e-5)
    np.testing.assert_allclose(m.sum(axis=1), [1, 0, 0], atol=1e-12)     # white is Y' = 1, no chroma


@pytest.mark.parametrize("bits", [8, 10])
@pytest.mark.parametrize("full", [0, 1])
@pytest.mark.parametrize("matrix", ["bt601", "bt709", "bt2020"])
def test_oracle_round_trip_444(matrix, full, bits):
    """rgb24 -> yuv444p (8-bit) / yuv444p10le -> rgb24 stays within one code value.  The one exception is inherent to 8-bit
    limited range: its 219 luma and 224 chroma steps cannot hold 256 RGB levels, and R = Y + 1.4 Cr adds both rounding
    errors, so a few samples move by two; 10-bit YUV returns every rgb24 code exactly."""
    rng = np.random.default_rng(bits * 10 + full)
    rgb = rng.integers(0, 256, (128, 128, 3)).astype(np.uint8)
    back = oy.yuv_to_rgb(*oy.rgb_to_yuv(rgb, 8, "444", bits, matrix, full), "444", bits, matrix, full, 8)
    err = np.abs(back.astype(np.int64) - rgb)
    if bits == 10:
        assert err.max() == 0
    elif full:
        assert err.max() <= 1
    else:
        assert err.max() <= 2 and (err <= 1).mean() > 0.995, (err.max(), (err <= 1).mean())


def test_oracle_plane_packing():
    for layout, (H, W) in [("420", (23, 37)), ("422", (1, 1)), ("444", (4, 6)), ("420", (48, 64))]:
        sx, sy = oy.SUBSAMPLING[layout]
        planes = [np.arange(H * W).reshape(H, W) % 251, np.full((-(-H // sy), -(-W // sx)), 7), np.full((-(-H // sy), -(-W // sx)), 9)]
        arr = oy.pack([p.astype(np.uint8) for p in planes], W)
        from nunif_b200.nunif.video import plane_shape
        assert arr.shape == plane_shape({"420": "yuv420p", "422": "yuv422p", "444": "yuv444p"}[layout], H, W)
        for a, b in zip(oy.unpack(arr, layout, H, W), planes):
            np.testing.assert_array_equal(a, b)


def test_plane_shape_is_pyav_layout_and_invertible():
    from nunif_b200.nunif import video as V
    assert V.plane_shape("yuv420p", 1080, 1920) == (1620, 1920)
    assert V.plane_shape("yuv422p10le", 1080, 1920) == (2160, 1920)
    assert V.plane_shape("yuv444p", 1080, 1920) == (3240, 1920)
    assert V.plane_shape("gbrp16le", 1080, 1920) == (3240, 1920)
    for pix_fmt in V.YUV_SOURCE_FORMATS:
        fmt = V._YuvFormat((pix_fmt, 1, 1), V.YUV_SOURCE_FORMATS, "source")
        for H in range(1, 40):
            for W in range(1, 24):
                assert fmt.size(V.plane_shape(pix_fmt, H, W)) == (H, W)


def test_bad_arguments_raise():
    from nunif_b200.nunif import video as V
    with pytest.raises(ValueError, match="supported: yuv420p"):
        V.yuv_to_rgb(np.zeros((6, 4), np.uint8), "nv12", 1, 1)
    with pytest.raises(ValueError, match="supported: yuv420p"):
        V.rgb_to_yuv(torch.zeros((4, 4, 3), dtype=torch.uint8), "yuv422p", 1, 1)
    with pytest.raises(ValueError, match="colorspace"):
        V.yuv_to_rgb(np.zeros((6, 4), np.uint8), "yuv420p", 7, 1)          # SMPTE 240M
    with pytest.raises(ValueError, match="color_range"):
        V.yuv_to_rgb(np.zeros((6, 4), np.uint8), "yuv420p", 1, 0)
    # odd-size plane shapes: no yuv420p frame has 4 rows of width 2 (rows are H + ceil(H / 2) for even widths)
    with pytest.raises(ValueError, match="not the plane array"):
        V.yuv_to_rgb(np.zeros((4, 2), np.uint8), "yuv420p", 1, 1)
    with pytest.raises(ValueError, match="not the plane array"):
        V.yuv_to_rgb(np.zeros((5, 2), np.uint8), "yuv444p", 1, 1)
    # bit depth: 10-bit planes need rgb48 (use_16bit) and uint16 planes; 8-bit ones refuse rgb48
    with pytest.raises(ValueError, match="use_16bit=True"):
        V.yuv_to_rgb(np.zeros((6, 4), np.uint16), "yuv420p10le", 1, 1)
    with pytest.raises(ValueError, match="use_16bit=False"):
        V.yuv_to_rgb(np.zeros((6, 4), np.uint8), "yuv420p", 1, 1, use_16bit=True)
    with pytest.raises(ValueError, match="uint16"):
        V.yuv_to_rgb(np.zeros((6, 4), np.uint8), "yuv420p10le", 1, 1, use_16bit=True)
    with pytest.raises(ValueError, match="use_16bit=True"):
        V.rgb_to_yuv(torch.zeros((4, 4, 3), dtype=torch.uint8), "gbrp16le", 1, 1)
    with pytest.raises(ValueError, match="CUDA"):
        V.yuv_to_rgb(np.zeros((6, 4), np.uint8), "yuv420p", 1, 1)
    with pytest.raises(ValueError, match="colorspace"):
        V.configure_colorspace(_stream("yuv420p", 1, 1, 1080), "bt2100", "yuv420p")


def test_pipeline_validates_formats():
    from nunif_b200.nunif import video as V
    # construction checks run before any CUDA object is created, so this needs no GPU
    for kw, msg in [(dict(source=("yuv420p10le", 9, 1)), "use_16bit=True"),
                    (dict(target=("yuv420p", 1, 1), use_16bit=True), "use_16bit=False"),
                    (dict(source=("p010le", 9, 1), use_16bit=True), "supported: yuv420p"),
                    (dict(target=("yuv422p", 1, 1)), "supported: yuv420p"),
                    (dict(source=("yuv420p", 1)), "tuple")]:
        with pytest.raises(ValueError, match=msg):
            V.FrameBatchPipeline(lambda x: x, 2, **kw)
