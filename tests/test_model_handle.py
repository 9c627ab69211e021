"""The model handle (csrc/model.cu): nb200_model_create refuses a kind outside the kind table before any CUDA call, and every
entry point that takes a handle refuses one of another network family with its own error, before any CUDA call."""
import ctypes
import pytest
import torch


@pytest.fixture(scope="module")
def lib():
    from nunif_b200 import build, _lib
    build.build()
    return _lib.lib()


@pytest.mark.parametrize("kind", [0, 24])
def test_create_refuses_unknown_kind(lib, kind):
    """Kinds 0 and 24 lie outside NB200_MODEL_*: refused before the device is queried, so also without a GPU."""
    names = (ctypes.c_char_p * 1)(b"w")
    value = ctypes.c_float(0.0)
    datas = (ctypes.c_void_p * 1)(ctypes.addressof(value))
    numels = (ctypes.c_int64 * 1)(1)
    h = ctypes.c_void_p()
    assert lib.nb200_model_create(kind, 1, names, datas, numels, 0, ctypes.byref(h)) != 0
    assert b"unknown model kind" in lib.nb200_last_error()
    assert not h


@pytest.mark.gpu
def test_entry_points_refuse_a_handle_of_another_family(lib):
    """A row_flow_v3 handle (and a sod_v1 handle for the row_flow_v3 entry point) passed to every entry point of another family:
    each call fails with that entry point's message and launches nothing.  The buffers are dummy host memory: a refusal
    happens before the first CUDA call."""
    from nunif_b200 import _lib, synth
    rf = _lib.Model("ROW_FLOW_V3", synth.row_flow_v3_state_dict(0), "cuda:0")
    sod = _lib.Model("SOD_V1", synth.sod_v1_state_dict(0), "cuda:0")
    d = ctypes.create_string_buffer(4096)
    cases = [
        (lambda: lib.nb200_model_forward(rf, d, 1, 64, 1, d, None), b"not an image-to-image model"),
        (lambda: lib.nb200_tiled_render(rf, d, 3, 64, 64, 64, 1, 1, d, None), b"not an image-to-image model"),
        (lambda: lib.nb200_tiled_render_host(rf, d, 3, 64, 64, 64, 1, 1, d, None), b"not an image-to-image model"),
        (lambda: lib.nb200_depth_anything_forward(rf, d, 1, 14, 14, d, None), b"model is not a Depth-Anything network"),
        (lambda: lib.nb200_zoedepth_forward(rf, d, 1, 32, 32, d, None), b"model is not a ZoeDepth network"),
        (lambda: lib.nb200_depth_aa(rf, d, 1, 8, 8, 0, d, None), b"model is not iw3.depth_aa"),
        (lambda: lib.nb200_mlbw_delta(rf, d, 1, 8, 8, d, d, None), b"model is not sbs.mlbw"),
        (lambda: lib.nb200_mlbw_delta_hole(rf, d, 1, 8, 8, d, d, d, None), b"model is not sbs.mlbw"),
        (lambda: lib.nb200_row_flow_delta(sod, d, 1, 8, 8, d, None), b"model is not sbs.row_flow_v3"),
        (lambda: lib.nb200_row_flow_v2_delta(rf, d, 1, 8, 8, d, None), b"model is not sbs.row_flow_v2"),
        (lambda: lib.nb200_light_inpaint(rf, d, d, 1, 8, 8, 0, d, None), b"model is not inpaint.light_inpaint_v1"),
        (lambda: lib.nb200_sod_forward(rf, d, 1, 8, 8, d, 8, 8, d, d, None), b"model is not iw3.sod_v1"),
        (lambda: lib.nb200_transnetv2_forward(rf, d, 1, 4, d, d, None), b"model is not TransNetV2"),
    ]
    torch.cuda.synchronize()
    launches = lib.nb200_launch_count()
    for i, (call, msg) in enumerate(cases):
        assert call() != 0, i
        assert msg in lib.nb200_last_error(), (i, lib.nb200_last_error())
    assert lib.nb200_mlbw_num_layers(rf) == 0
    assert lib.nb200_mlbw_has_hole_mask(rf) == 0
    assert lib.nb200_launch_count() == launches
