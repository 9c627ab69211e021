"""ctypes binding of libnunif_b200.so (the C ABI in include/nunif_b200.h).

PyTorch is only used for device memory and streams: tensors are passed to the
library as raw device pointers.  There is NO fallback: if the shared library is
missing, or no sm_90 device is present, calls raise RuntimeError.
"""
import ctypes
import os
import threading

_HERE = os.path.dirname(os.path.abspath(__file__))
LIB_PATH = os.path.join(_HERE, "libnunif_b200.so")
_lib = None
_lock = threading.Lock()

c_void_p, c_int, c_float, c_size_t, c_char_p = (ctypes.c_void_p, ctypes.c_int, ctypes.c_float,
                                                 ctypes.c_size_t, ctypes.c_char_p)
c_double = ctypes.c_double


class TileConfig(ctypes.Structure):
    """nb200_tile_config == SeamBlending.create_config (seam_blending.py:109-143)."""
    _fields_ = [(n, ctypes.c_int32) for n in (
        "y_h", "y_w", "h_blocks", "w_blocks", "pad_l", "pad_r", "pad_t", "pad_b",
        "y_buffer_h", "y_buffer_w", "input_tile_step", "output_tile_step")]

    def as_dict(self):
        return {
            "y_h": self.y_h, "y_w": self.y_w, "h_blocks": self.h_blocks, "w_blocks": self.w_blocks,
            "pad": (self.pad_l, self.pad_r, self.pad_t, self.pad_b),
            "y_buffer_h": self.y_buffer_h, "y_buffer_w": self.y_buffer_w,
            "input_tile_step": self.input_tile_step, "output_tile_step": self.output_tile_step,
        }


class GemmDesc(ctypes.Structure):
    """nb200_gemm_desc: every field of one implicit-GEMM launch (csrc/gemm.h ConvGemm) but the pointers."""
    _fields_ = ([(n, ctypes.c_int) for n in ("kind", "pad", "dil", "B", "Hi", "Wi", "Ci", "Cin")]
                + [("a_row_stride", ctypes.c_longlong), ("a_img_stride", ctypes.c_longlong), ("a_planes", ctypes.c_int),
                   ("a_plane_stride", ctypes.c_longlong)]
                + [(n, ctypes.c_int) for n in ("N", "act", "ldo", "out_mode", "cout")]
                + [("split_stride", ctypes.c_longlong)]
                + [(n, ctypes.c_int) for n in ("ldr", "res_H", "res_W", "res_cy", "res_cx", "res_before_act", "Cin2", "ld2")])


MAPPER_MAX_STAGES = 8


class MapperFn(ctypes.Structure):
    """nb200_mapper_fn: one function of iw3/mapper.py resolve_mapper_function and its fp32 constants."""
    _fields_ = [("kind", ctypes.c_int32), ("k", ctypes.c_float * 5)]


class MapperStage(ctypes.Structure):
    """nb200_mapper_stage: one function, or the blend a(x) * (1 - w) + b(x) * w."""
    _fields_ = [("a", MapperFn), ("b", MapperFn), ("blend", ctypes.c_int32), ("one_minus_w", ctypes.c_float),
                ("w", ctypes.c_float), ("pad", ctypes.c_float)]


class Mapper(ctypes.Structure):
    """nb200_mapper: a parsed get_mapper(name) chain (nunif_b200/iw3/mapper.py builds it)."""
    _fields_ = [("n_stages", ctypes.c_int32), ("pad", ctypes.c_int32 * 3), ("stage", MapperStage * MAPPER_MAX_STAGES)]


# name -> (restype, argtypes).  Must list every symbol declared in include/nunif_b200.h
# (tests/test_abi.py parses the header and checks this table and the .so against it).
SIGNATURES = {
    "nb200_last_error": (c_char_p, []),
    "nb200_abi_version": (c_int, []),
    "nb200_check_device": (c_int, [c_int]),
    "nb200_launch_count": (ctypes.c_uint64, []),
    "nb200_tile_config_create": (c_int, [c_int] * 6 + [ctypes.POINTER(TileConfig)]),
    "nb200_tile_unfold": (c_int, [c_void_p, c_int, c_int, c_int, ctypes.POINTER(TileConfig), c_int, c_int, c_int,
                                  c_void_p, c_int, c_void_p]),
    "nb200_tile_gather_blend": (c_int, [c_void_p, c_int, ctypes.POINTER(TileConfig), c_int, c_int, c_int, c_int,
                                        c_void_p, c_void_p]),
    "nb200_model_create": (c_int, [c_int, c_int, ctypes.POINTER(c_char_p), ctypes.POINTER(c_void_p),
                                   ctypes.POINTER(ctypes.c_int64), c_int, ctypes.POINTER(c_void_p)]),
    "nb200_model_destroy": (None, [c_void_p]),
    "nb200_model_info": (c_int, [c_void_p, ctypes.POINTER(c_int), ctypes.POINTER(c_int), ctypes.POINTER(c_int)]),
    "nb200_model_weight_blob": (c_int, [c_void_p, ctypes.POINTER(c_void_p), ctypes.POINTER(c_size_t)]),
    "nb200_model_forward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_tiled_render": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_tiled_render_host": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_depth_anything_forward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_zoedepth_forward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_zoe_rel_pos_table": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p]),
    "nb200_depth_aa": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_mlbw_delta": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "nb200_mlbw_num_layers": (c_int, [c_void_p]),
    "nb200_mlbw_has_hole_mask": (c_int, [c_void_p]),
    "nb200_mlbw_delta_hole": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nb200_hole_mask": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_float, c_int, c_void_p, c_void_p]),
    "nb200_row_flow_delta": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_row_flow_v2_delta": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_inpaint_mask": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_inpaint_blur": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_resize_bilinear_aa": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_light_inpaint": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_backward_warp_delta": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_double, c_void_p, c_void_p]),
    "nb200_backward_warp_delta_f16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_double, c_void_p, c_void_p]),
    "nb200_backward_warp_delta_sym": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_double, c_int, c_int, c_void_p,
                                              c_void_p, c_void_p]),
    "nb200_alpha_border_padding_workspace": (c_size_t, [c_int, c_int]),
    "nb200_alpha_border_padding": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "nb200_tta_transform": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_tta_merge": (c_int, [ctypes.POINTER(c_void_p), c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_hwc_to_chw_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_chw_f32_to_hwc": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_hdr2sdr": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, ctypes.POINTER(c_double), c_int, c_void_p, c_void_p]),
    "nb200_rgb_noise": (c_int, [ctypes.c_uint64, ctypes.c_uint32, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_apply_rgb_noise": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, ctypes.c_uint64, ctypes.c_uint32, c_int,
                                      c_void_p, c_int, ctypes.POINTER(c_double), c_int, c_int, c_void_p, c_void_p]),
    "nb200_da_preprocess_size": (c_int, [c_int, c_int, c_int, c_int, c_int, ctypes.POINTER(c_int), ctypes.POINTER(c_int)]),
    "nb200_da_preprocess": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_null_depth": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_zoe_preprocess_size": (c_int, [c_int] * 5 + [ctypes.POINTER(c_int)] * 6),
    "nb200_zoe_preprocess": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_anaglyph": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_resize_bicubic_aa": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_resize_bicubic_aa_ac": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_rot90": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_autocrop_detect": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int] + [c_void_p] * 7),
    "nb200_autocrop_bounds": (c_int, [c_void_p, c_int, c_void_p, c_int, c_int, c_float, c_void_p, c_void_p]),
    "nb200_equirectangular_size": (c_int, [c_int, c_int, ctypes.POINTER(c_int), ctypes.POINTER(c_int)]),
    "nb200_equirectangular": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_backward_warp": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_double, c_double, c_int, c_int,
                                    c_void_p, c_void_p, c_void_p]),
    "nb200_backward_warp_conv": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_double, c_void_p, c_int, c_int,
                                         c_void_p, c_void_p, c_void_p]),
    "nb200_forward_warp_conv": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_double, c_void_p, c_int, c_int,
                                        c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nb200_sod_forward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "nb200_sod_position": (c_int, [c_void_p, c_void_p, c_int, c_int, c_double, c_void_p, c_void_p]),
    "nb200_sod_ema": (c_int, [c_void_p, c_void_p, c_int, c_void_p, c_double, c_void_p, c_void_p]),
    "nb200_transnetv2_forward": (c_int, [c_void_p, c_void_p, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "nb200_forward_warp_workspace": (c_size_t, [c_int] * 5),
    "nb200_forward_warp": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_double, c_double, c_int, c_int,
                                   c_int, c_int, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p]),
    "nb200_depth_resize_aa": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_dilate_edge_workspace": (c_size_t, [c_int] * 3),
    "nb200_dilate_edge": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_void_p, c_void_p, c_void_p]),
    "nb200_minmax_map": (c_int, [c_void_p, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p]),
    "nb200_ema_scaler_create": (c_int, [c_int, c_double, c_int, ctypes.POINTER(c_void_p)]),
    "nb200_ema_scaler_destroy": (None, [c_void_p]),
    "nb200_ema_scaler_reset": (c_int, [c_void_p, c_double, c_int]),
    "nb200_ema_scaler_update": (c_int, [c_void_p, c_void_p, c_int, ctypes.POINTER(c_int), c_void_p]),
    "nb200_ema_scaler_normalize": (c_int, [c_void_p, c_void_p, c_int, c_int, c_float, c_void_p, c_void_p, c_void_p]),
    "nb200_depth_mapper": (c_int, [c_void_p, ctypes.c_longlong, c_float, c_void_p, c_void_p]),
    "nb200_mapper_apply": (c_int, [c_void_p, ctypes.c_longlong, ctypes.POINTER(Mapper), c_void_p, c_void_p]),
    "nb200_minmax_mapper": (c_int, [c_void_p, c_int, c_int, ctypes.POINTER(Mapper), c_void_p, c_void_p, c_void_p]),
    "nb200_depth_export_u16": (c_int, [c_void_p, c_int, c_int, c_int, ctypes.POINTER(Mapper), c_int, c_int, c_int, c_int, c_void_p,
                                       c_void_p]),
    "nb200_depth_import": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_double, c_double, c_int, c_void_p, c_void_p]),
    "nb200_anaglyph_dubois": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_conv_gemm_f16": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_int,
                                    c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int,
                                    c_void_p]),
    "nb200_conv_gemm_pixshuf_a2_f16": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_void_p, c_int, c_void_p,
                                               c_int, c_int, c_void_p, c_int, c_int, c_void_p]),
    "nb200_conv_gemm_ex_f16": (c_int, [ctypes.POINTER(GemmDesc), c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_void_p,
                                       c_void_p]),
    "nb200_flash_attention_f16": (c_int, [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    "nb200_window_mha_f16": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p] + [c_int] * 8 + [c_void_p]),
    "nb200_reppad1_f16": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_void_p]),
    "nb200_add_layernorm_f32": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, ctypes.c_longlong, c_int, c_void_p]),
    "nb200_upsample_bilinear_f16": (c_int, [c_void_p, c_int, c_int, c_int, c_int, c_void_p, c_int, c_int, c_void_p]),
    "nb200_zoe_add_upsampled_f16": (c_int, [c_void_p, c_void_p] + [c_int] * 6 + [c_void_p, c_void_p]),
    "nb200_zoe_softplus_f32": (c_int, [c_void_p, c_void_p, ctypes.c_longlong, c_void_p]),
    "nb200_zoe_seed_normed_f32": (c_int, [c_void_p, ctypes.c_longlong, c_float, c_float, c_void_p, c_void_p]),
    "nb200_zoe_attractor_f32": (c_int, [c_void_p, c_int, c_int, c_void_p] + [c_int] * 6 + [c_float, c_float, c_void_p, c_void_p,
                                                                                            c_void_p]),
    "nb200_zoe_clb_concat_f16": (c_int, [c_void_p, c_void_p, c_void_p] + [c_int] * 5 + [c_void_p, c_void_p]),
    "nb200_zoe_clb_final_f32": (c_int, [c_void_p, c_int, c_void_p, c_void_p, c_void_p] + [c_int] * 5 + [c_void_p, c_void_p]),
    "nb200_zoe_expand_rel_bias_f32": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_int, c_void_p]),
    "nb200_stem_conv_f16": (c_int, [c_void_p, c_void_p, c_void_p] + [c_int] * 5 + [c_void_p, c_int, c_void_p]),
    "nb200_tail_conv_f16": (c_int, [c_void_p, c_void_p, c_void_p] + [c_int] * 5 + [c_void_p, c_void_p, c_int, c_int, c_int, c_void_p]),
    "nb200_head_conv_f16": (c_int, [c_void_p, c_void_p, c_void_p] + [c_int] * 5 + [c_void_p, c_void_p]),
    "nb200_se_block_f16": (c_int, [c_void_p] * 5 + [c_int] * 4 + [c_void_p]),
    "nb200_to_image_f16": (c_int, [c_void_p] + [c_int] * 6 + [c_void_p, c_void_p]),
    "nb200_sod_conv_f16": (c_int, [c_void_p, c_int, c_int, c_int, c_void_p, c_void_p, c_int, c_int, c_void_p, c_int, c_int, c_void_p,
                                   c_int, c_int, c_int, c_int, c_void_p]),
    "nb200_row_flow_prep_f16": (c_int, [c_void_p] + [c_int] * 5 + [c_void_p, c_void_p]),
    "nb200_row_flow_last_conv_f32": (c_int, [c_void_p] + [c_int] * 5 + [c_void_p] * 4),
    "nb200_mlbw_prep_f16": (c_int, [c_void_p] + [c_int] * 8 + [c_void_p] * 4),
    "nb200_mlbw_out_f32": (c_int, [c_void_p, c_void_p] + [c_int] * 9 + [c_void_p] * 6),
    "nb200_depth_aa_minmax_f32": (c_int, [c_void_p, ctypes.c_longlong, c_void_p, c_void_p]),
    "nb200_depth_aa_prep_f16": (c_int, [c_void_p, c_void_p] + [c_int] * 7 + [c_void_p] * 4),
    "nb200_depth_aa_out_f32": (c_int, [c_void_p, c_void_p, c_void_p] + [c_int] * 7 + [c_void_p, c_void_p, c_int, c_void_p, c_void_p]),
    "nb200_swin_mlp_fused_y_f16": (c_int, [c_void_p, c_void_p, ctypes.c_longlong, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                           c_void_p, c_void_p, c_void_p, c_int, c_void_p, c_void_p, c_void_p]),
    "nb200_record_launches": (c_int, [c_int]),
    "nb200_recorded_launches": (c_int, [c_char_p, c_size_t]),
    "nb200_recorded_launches_named": (c_int, [c_char_p, c_size_t]),
    "nb200_tune_set": (c_int, [c_int, c_int]),
    "nb200_debug_tap": (c_int, [c_int, c_void_p, ctypes.c_size_t]),
    "nb200_profile_enable": (c_int, [c_int]),
    "nb200_profile_report": (c_int, [ctypes.c_char_p, c_size_t]),
    "nb200_profile_dump": (c_int, [c_char_p, c_size_t]),
    "nb200_swin_mlp_fused_f16": (c_int, [c_void_p, c_void_p, ctypes.c_longlong, c_int, c_void_p, c_void_p, c_void_p, c_void_p,
                                         c_void_p, c_void_p, c_void_p]),
    "nb200_swin_attn_fused_f16": (c_int, [c_void_p, c_void_p, c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int,
                                          c_void_p]),
    "nb200_window_attention_f16": (c_int, [c_void_p, c_void_p, c_void_p, c_int, c_int, c_int, c_int, c_int, c_int, c_void_p]),
}


def lib():
    """Load the shared library (once).  Raises if it has not been built."""
    global _lib
    if _lib is not None:
        return _lib
    with _lock:
        if _lib is not None:
            return _lib
        if not os.path.exists(LIB_PATH):
            raise RuntimeError(
                f"{LIB_PATH} is missing: build it with `python -m nunif_b200.build` "
                "(nvcc, sm_90a).  nunif_b200 has no CPU / PyTorch fallback.")
        l = ctypes.CDLL(LIB_PATH)
        for name, (res, args) in SIGNATURES.items():
            fn = getattr(l, name)
            fn.restype = res
            fn.argtypes = args
        _lib = l
    return _lib


def check(status):
    if status != 0:
        raise RuntimeError("nunif_b200: " + lib().nb200_last_error().decode("utf-8", "replace"))


def require_cuda(t, name="tensor"):
    import torch
    if not torch.is_tensor(t) or not t.is_cuda:
        raise RuntimeError(f"nunif_b200: {name} must be a CUDA tensor (the engine has no CPU fallback)")


# NB200_MODEL_<NAME> -> value: the network kinds nb200_model_create packs.  Must match the enum in include/nunif_b200.h
# (tests/test_abi.py parses the header and checks this table against it).
MODEL_KINDS = {
    "UPCUNET": 1, "CUNET": 2, "SWIN_UNET_1X": 3, "SWIN_UNET_2X": 4, "SWIN_UNET_4X": 5, "DEPTH_ANYTHING_V2_S": 6,
    "ROW_FLOW_V3": 7, "DEPTH_ANYTHING_V2_B": 8, "DEPTH_ANYTHING_V2_L": 9, "DEPTH_AA": 10, "MLBW": 11, "ZOEDEPTH_N": 12,
    "UPCONV_7": 13, "VGG_7": 14, "LIGHT_INPAINT_V1": 15, "ROW_FLOW_V2": 16, "SOD_V1": 17, "ZOEDEPTH_ANY_N": 18,
    "ZOEDEPTH_ANY_K": 19, "DEPTH_ANYTHING_V1_S": 20, "DEPTH_ANYTHING_V1_B": 21, "DEPTH_ANYTHING_V1_L": 22, "TRANSNET_V2": 23,
}


def cuda_device(device):
    """``torch.device(device)``; raises unless it is a CUDA device."""
    import torch
    device = torch.device(device)
    if device.type != "cuda":
        raise RuntimeError("nunif_b200 models live on a CUDA (sm_90) device; there is no CPU path")
    return device


class Model:
    """One packed network (``nb200_model*``) of kind ``MODEL_KINDS[kind]`` on ``device``, built from a state_dict with the
    reference's key names (strict: a missing or unexpected key raises) and destroyed with this object.  It passes directly as
    the ``nb200_model*`` argument of the library's entry points (ctypes reads ``_as_parameter_``)."""
    _as_parameter_ = None

    def __init__(self, kind, state_dict, device, no_clip=False):
        import torch
        # the tensors must outlive nb200_model_create: the ctypes arrays hold only their raw pointers
        items = [(k, v.detach().to("cpu", torch.float32).contiguous()) for k, v in state_dict.items()]
        n = len(items)
        names = (c_char_p * n)(*[k.encode() for k, _ in items])
        datas = (c_void_p * n)(*[v.data_ptr() for _, v in items])
        numels = (ctypes.c_int64 * n)(*[v.numel() for _, v in items])
        h = c_void_p()
        with torch.cuda.device(device):
            check(lib().nb200_model_create(MODEL_KINDS[kind], n, names, datas, numels, 1 if no_clip else 0, ctypes.byref(h)))
        self._as_parameter_ = h

    def __del__(self):
        try:
            if self._as_parameter_:
                lib().nb200_model_destroy(self._as_parameter_)
                self._as_parameter_ = None
        except Exception:
            pass


def stream_ptr(device=None):
    import torch
    return ctypes.c_void_p(torch.cuda.current_stream(device).cuda_stream)


def ptr(t):
    return ctypes.c_void_p(t.data_ptr()) if t is not None else ctypes.c_void_p(0)
