"""CPU-only: the C-ABI library builds, loads without a GPU, exports every symbol that
include/nunif_b200.h declares, and fails loudly (no fallback) when asked to compute."""
import ctypes
import os
import re
import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from nunif_b200 import build, _lib
    build.build()
    return _lib.lib()


def declared_symbols():
    src = open(os.path.join(ROOT, "include", "nunif_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(nb200_[a-z0-9_]+)\s*\(", src)))


def test_header_symbols_exported(lib):
    from nunif_b200 import _lib
    syms = declared_symbols()
    assert len(syms) >= 20
    for s in syms:
        assert hasattr(lib, s), f"{s} declared in include/nunif_b200.h but not exported"
        assert s in _lib.SIGNATURES, f"{s} has no ctypes signature in nunif_b200/_lib.py"
    for s in _lib.SIGNATURES:
        assert s in syms, f"{s} bound in _lib.py but not declared in the header"


def test_model_kinds_match_header():
    """_lib.MODEL_KINDS is the header's NB200_MODEL_* enum, name for name and value for value."""
    from nunif_b200 import _lib
    src = open(os.path.join(ROOT, "include", "nunif_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    declared = {name: int(v) for name, v in re.findall(r"\bNB200_MODEL_([A-Z0-9_]+)\s*=\s*(\d+)", src)}
    assert declared == _lib.MODEL_KINDS


def test_abi_version(lib):
    assert lib.nb200_abi_version() == 1


def test_tile_config_host_planner_bit_exact(lib):
    """create_config is host integer code: check it against the reference goldens without a GPU."""
    from nunif_b200.nunif.render import create_config
    from tests.util import load_golden
    g = load_golden("seam_config")
    for case, want in zip(g["cases"], g["configs"]):
        h, w, scale, offset, tile, blend = (int(v) for v in case)
        p = create_config((h, w), scale, offset, tile, blend)
        got = [p["y_h"], p["y_w"], p["h_blocks"], p["w_blocks"], *p["pad"],
               p["y_buffer_h"], p["y_buffer_w"], p["input_tile_step"], p["output_tile_step"]]
        assert got == [int(v) for v in want], (case, got, want)


@pytest.mark.skipif(torch.cuda.is_available(), reason="checks the no-GPU failure mode")
def test_no_cpu_fallback(lib):
    from nunif_b200.iw3 import apply_divergence_grid_sample, dilate_edge
    from nunif_b200.nunif.models import create_model
    from nunif_b200 import synth
    assert lib.nb200_check_device(0) != 0
    assert b"no CPU fallback" in lib.nb200_last_error()
    with pytest.raises(RuntimeError):
        apply_divergence_grid_sample(torch.rand(1, 3, 8, 8), torch.rand(1, 1, 8, 8), 2.0, 0.5)
    with pytest.raises(RuntimeError):
        dilate_edge(torch.rand(1, 1, 8, 8), 2)
    with pytest.raises(RuntimeError):
        create_model("waifu2x.upcunet", synth.upcunet_state_dict(0), device="cpu")


def test_find_valid_tile_size_host():
    from tests.util import load_golden
    from nunif_b200.nunif import models
    g = load_golden("tile_size")
    m_c = object.__new__(models.B200I2IModel)
    m_c._validator = models._cunet_validator
    m_c.i2i_default_tile_size = 256
    m_s = object.__new__(models.B200I2IModel)
    m_s._validator = models._swin_validator
    m_s.i2i_default_tile_size = 256
    for q, c, s in zip(g["query"], g["cunet"], g["swin"]):
        assert m_c.find_valid_tile_size(int(q)) == int(c)
        assert m_s.find_valid_tile_size(int(q)) == int(s)
    assert m_s.find_valid_tile_size(None) == 256


def test_da_preprocess_size_host_rule_bit_exact(lib):
    """nb200_da_preprocess_size is host integer logic (depth_anything_model.py:69-101): check it against the sizes the
    reference produced (tests/golden/frames.npz) without a GPU."""
    from tests.util import load_golden
    from nunif_b200.iw3.depth_anything_preprocess import preprocess_size
    g = load_golden("frames")
    for H, W, lb, lim, nh, nw in g["sizes"]:
        assert preprocess_size(int(H), int(W), int(lb), 4, bool(lim)) == (int(nh), int(nw)), (H, W, lb, lim)
    assert preprocess_size(1080, 1920) == (392, 686)


def test_zoe_preprocess_size_host_rule_bit_exact(lib):
    """nb200_zoe_preprocess_size (zoedepth_model.py:30-71, incl. Python's round-half-even) against the reference's sizes."""
    from tests.util import load_golden
    from nunif_b200.iw3.zoedepth_preprocess import preprocess_size
    g = load_golden("frames")
    for H, W, oh, ow, ph, pw in g["zoe_sizes"]:
        nh, nw, p_h, p_w, fh, fw = preprocess_size(int(H), int(W))
        assert (fh + 2 * p_h, fw + 2 * p_w, p_h, p_w) == (int(oh), int(ow), int(ph), int(pw)), (H, W)


def test_launch_recorder_mask_bits_0_to_5(lib):
    """nb200_record_launches takes a mask of the recorded kinds (bit 0: GEMM / attention / Swin, bit 1: the kernels between
    them, bit 2: the waifu2x stem / tail / head convolutions, SE, to_image and the SOD REBNCONV, bit 3: the stereo networks'
    input / output stages, row_flow_v2 and the hole mask, bit 4: the backward stereo warps and the AA depth resize, bit 5: the
    depth networks' patch, token, hook-cast, readout and DPT kernels) and refuses other bits; host only, no device needed."""
    for on in (1, 2, 3, 4, 7, 8, 15, 16, 31, 32, 63, 0):
        assert lib.nb200_record_launches(on) == 0, on
    for on in (64, 127):
        assert lib.nb200_record_launches(on) != 0, on
        assert b"unknown recorder bits" in lib.nb200_last_error()
    buf = ctypes.create_string_buffer(16)
    assert lib.nb200_recorded_launches(buf, 16) == 0 and buf.value == b""


def test_stereo_entry_points_refuse_bad_geometry(lib):
    """The stereo test entry points refuse a padded grid that does not hold the image, an L without an instantiation and a hole
    head with L != 2 before their first CUDA call: dummy host pointers, no device needed, and nothing is recorded."""
    d = ctypes.create_string_buffer(4096)
    cases = [
        (lambda: lib.nb200_row_flow_prep_f16(d, 1, 13, 16, 12, 2, d, None), b"padded height"),            # Hp < h
        (lambda: lib.nb200_row_flow_prep_f16(d, 1, 12, 17, 12, 2, d, None), b"padded width"),             # 8 Wt < w
        (lambda: lib.nb200_row_flow_last_conv_f32(d, 1, 12, 2, 12, 17, d, d, d, None), b"padded width"),
        (lambda: lib.nb200_row_flow_last_conv_f32(d, 0, 12, 2, 12, 16, d, d, d, None), b"empty input"),
        (lambda: lib.nb200_mlbw_prep_f16(d, 1, 4, 16, 1, 1, 4, 3, 8, d, d, d, None), b"padded height"),   # ph1 + H > Hp
        (lambda: lib.nb200_mlbw_prep_f16(d, 1, 4, 16, 1, 1, 6, 2, 8, d, d, d, None), b"padded width"),    # pw1 + W > 8 Wt
        (lambda: lib.nb200_mlbw_prep_f16(d, 1, 4, 16, -1, 0, 6, 4, 8, d, d, d, None), b"negative leading pad"),
        (lambda: lib.nb200_mlbw_out_f32(d, d, 1, 4, 16, 1, 8, 6, 2, 8, 2, d, d, d, d, None, None), b"padded width"),
        (lambda: lib.nb200_mlbw_out_f32(d, d, 1, 4, 16, 1, 8, 6, 4, 8, 3, d, d, d, d, None, None), b"L must be 2 or 4"),
        (lambda: lib.nb200_mlbw_out_f32(d, d, 1, 4, 16, 1, 8, 6, 4, 16, 4, d, d, d, d, d, None), b"hole head"),
        (lambda: lib.nb200_depth_aa_minmax_f32(d, 0, d, None), b"empty input"),
        (lambda: lib.nb200_depth_aa_prep_f16(d, None, 1, 16, 16, 8, 0, 8, 8, d, d, d, None), b"padded height"),   # ph1 + H > 2 Hh
        (lambda: lib.nb200_depth_aa_out_f32(d, d, None, 1, 16, 17, 0, 0, 8, 8, d, d, 1, d, None), b"padded width"),
    ]
    assert lib.nb200_record_launches(8) == 0
    try:
        for i, (call, msg) in enumerate(cases):
            assert call() != 0, i
            assert msg in lib.nb200_last_error(), (i, lib.nb200_last_error())
    finally:
        lib.nb200_record_launches(0)
    buf = ctypes.create_string_buffer(16)
    assert lib.nb200_recorded_launches(buf, 16) == 0 and buf.value == b""


def test_depth_entry_points_refuse_bad_shapes(lib):
    """The depth networks' kernel entry points refuse, before their first CUDA call, an image that is not a whole number of
    patches, a patch row narrower than its 588 columns, element counts and widths their vector loads cannot take, a head
    width other than 32, a channel pad below the channel count, and an x0 without s: dummy host pointers, no device needed,
    and nothing is recorded."""
    d = ctypes.create_string_buffer(4096)
    cases = [
        (lambda: lib.nb200_da_patch_im2col_f16(d, 1, 28, 27, 640, d, None), b"multiples of the 14-pixel patch"),
        (lambda: lib.nb200_da_patch_im2col_f16(d, 1, 15, 28, 640, d, None), b"multiples of the 14-pixel patch"),
        (lambda: lib.nb200_da_patch_im2col_f16(d, 1, 28, 28, 584, d, None), b"kpad below"),
        (lambda: lib.nb200_zoe_patch_im2col_f16(d, 1, 32, 40, d, None), b"multiples of the 16-pixel patch"),
        (lambda: lib.nb200_zoe_patch_im2col_f16(d, 1, 14, 32, d, None), b"multiples of the 16-pixel patch"),
        (lambda: lib.nb200_vit_assemble_tokens_f32(d, d, d, d, 1, 0, 384, None), b"bad shape"),
        (lambda: lib.nb200_zoe_add_cast_f16(d, d, d, 1026, None), b"multiple of 4"),
        (lambda: lib.nb200_zoe_add_cast_f16(d, None, d, 6, None), b"multiple of 4"),
        (lambda: lib.nb200_zoe_readout_concat_f16(d, 1, 4, 100, d, None), b"multiple of 8"),
        (lambda: lib.nb200_dpt_depth_to_space4_f16(d, 1, 2, 3, 48, 40, d, None), b"padded channel count"),
        (lambda: lib.nb200_dpt_im2col_s2_f16(d, 1, 3, 3, 12, d, None), b"multiple of 8"),
        (lambda: lib.nb200_dpt_relu_add_f16(d, d, d, d, 1020, None), b"multiple of 8"),
        (lambda: lib.nb200_dpt_relu_add_f16(d, None, d, None, 12, None), b"multiple of 8"),
        (lambda: lib.nb200_dpt_relu_add_f16(d, d, d, None, 16, None), b"x0 and s go together"),
        (lambda: lib.nb200_dpt_head_final_f32(d, 64, 64, d, 0.5, d, None), b"32 input channels"),
        (lambda: lib.nb200_dpt_head_final_f32(d, 64, 16, d, 0.5, d, None), b"32 input channels"),
    ]
    assert lib.nb200_record_launches(32) == 0
    try:
        for i, (call, msg) in enumerate(cases):
            assert call() != 0, i
            assert msg in lib.nb200_last_error(), (i, lib.nb200_last_error())
    finally:
        lib.nb200_record_launches(0)
    buf = ctypes.create_string_buffer(16)
    assert lib.nb200_recorded_launches(buf, 16) == 0 and buf.value == b""


def test_backward_warp_entry_points_refuse_bad_geometry(lib):
    """nb200_backward_warp / _conv refuse a batch or a height beyond a grid axis (65535) for either kernel, and the
    learned-delta warps a row too wide for the row-staged kernel's 200 KB of shared memory (W = 7313 with a full-resolution
    delta), all before their first CUDA call: dummy host pointers, no device needed, and nothing is recorded."""
    d = ctypes.create_string_buffer(4096)
    bw = lambda B, H: lib.nb200_backward_warp(d, d, B, H, 8, 4, 4, 2.0, 0.5, 0, 0, d, d, None)
    bwc = lambda B, H: lib.nb200_backward_warp_conv(d, d, B, H, 8, 4, 4, 2.0, d, 0, 1, d, None, None)
    cases = [
        (lambda: bw(65536, 8), b"batch too large"),
        (lambda: bw(1, 65536), b"image too tall"),
        (lambda: bwc(65536, 8), b"batch too large"),
        (lambda: bwc(1, 65536), b"image too tall"),
        (lambda: lib.nb200_backward_warp_delta(d, d, 1, 2, 7313, 2, 7313, 0.001, d, None), b"image row too wide"),
        (lambda: lib.nb200_backward_warp_delta_f16(d, d, 1, 2, 7313, 2, 7313, 0.001, d, None), b"image row too wide"),
        (lambda: lib.nb200_backward_warp_delta_sym(d, d, 1, 2, 7313, 2, 7313, 0.001, 1, 1, d, d, None), b"image row too wide"),
        (lambda: lib.nb200_backward_warp_delta(d, d, 65536, 2, 8, 2, 8, 0.001, d, None), b"image row too wide"),
    ]
    assert lib.nb200_record_launches(16) == 0
    try:
        for i, (call, msg) in enumerate(cases):
            assert call() != 0, i
            assert msg in lib.nb200_last_error(), (i, lib.nb200_last_error())
    finally:
        lib.nb200_record_launches(0)
    buf = ctypes.create_string_buffer(16)
    assert lib.nb200_recorded_launches(buf, 16) == 0 and buf.value == b""


def test_forward_warp_entry_points_refuse_bad_geometry(lib):
    """nb200_forward_warp / _conv refuse, before their first CUDA call: a divergence whose row padding
    P = (int)(base * divergence * 0.01 + 2) is negative (W = 64, divergence -5: P = -1), a padded row over 227 KB at 28 B per
    cell with a depth that upsamples on both axes and a workspace (H = 3 from h = 2, W = 8002 from w = 3000, P = 150:
    Wp = 8302), so that checking after the column-table launch would fail on that launch instead,
    B over the grid's 65535, a misaligned workspace that the column table would use, and empty sizes.  Dummy host pointers,
    no device needed, and nothing is recorded."""
    d = ctypes.create_string_buffer(4096)
    ws = ctypes.addressof(d) + (16 - ctypes.addressof(d) % 16) % 16      # 16-byte aligned inside d
    fw = lambda B, H, W, h, w, div, work=ws: lib.nb200_forward_warp(d, d, B, H, W, h, w, div, 0.5, 1, 0, 1, 0, d, d, d, d, work, None)
    fwc = lambda B, H, W, h, w, div, work=ws: lib.nb200_forward_warp_conv(d, d, B, H, W, h, w, div, d, 1, 0, 1, 1, d, None, None,
                                                                          None, work, None)
    cases = []
    for f in (fw, fwc):
        cases += [
            (lambda f=f: f(1, 4, 64, 4, 64, -5.0), b"divergence too negative"),
            (lambda f=f: f(1, 3, 8002, 2, 3000, 1.85), b"does not fit shared memory"),
            (lambda f=f: f(65536, 4, 64, 2, 32, 2.0), b"batch too large"),
            (lambda f=f: f(1, 4, 64, 2, 32, 2.0, ws + 4), b"16-byte aligned"),
            (lambda f=f: f(0, 4, 64, 2, 32, 2.0), b"bad shape"),
            (lambda f=f: f(1, 4, 64, 0, 32, 2.0), b"bad shape"),
            (lambda f=f: f(1, 4, 0, 2, 32, 2.0), b"bad shape"),
        ]
    assert lib.nb200_record_launches(16) == 0
    try:
        for i, (call, msg) in enumerate(cases):
            assert call() != 0, i
            assert msg in lib.nb200_last_error(), (i, lib.nb200_last_error())
    finally:
        lib.nb200_record_launches(0)
    buf = ctypes.create_string_buffer(16)
    assert lib.nb200_recorded_launches(buf, 16) == 0 and buf.value == b""


def test_launch_recorder_names_each_field(lib):
    """A recorded line is `kind,name=value,...` with the names the replay tests read, and nb200_recorded_launches returns
    the same values without the names.  zoe_expand_rel_bias records its launch before it checks ldb, so a call with dummy
    host pointers and ldb < ph * pw + 1 is refused without touching the device and still leaves its line: no GPU needed."""
    dummy = ctypes.create_string_buffer(64)
    assert lib.nb200_record_launches(2) == 0
    try:
        assert lib.nb200_zoe_expand_rel_bias_f32(dummy, 3, 5, 4, dummy, 10, None) != 0
        assert b"bias row stride too small" in lib.nb200_last_error()
    finally:
        lib.nb200_record_launches(0)
    buf = ctypes.create_string_buffer(256)
    assert lib.nb200_recorded_launches_named(buf, 256) == 0
    assert buf.value == b"zrelbias,ph=3,pw=5,heads=4,ldb=10\n"
    assert lib.nb200_recorded_launches(buf, 256) == 0
    assert buf.value == b"zrelbias,3,5,4,10\n"
