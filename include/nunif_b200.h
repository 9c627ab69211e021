/*
 * nunif_b200 - C ABI of the H100 (sm_90a) engine for nunif's two hot paths.
 *
 * The reference (nagadomi/nunif) is pure Python; it has no FFI.  The boundary a
 * maintainer binds is therefore "one C entry point per reference callable on
 * the hot path" (SURVEY.md section 8b).  Each declaration cites the reference
 * callable it replaces (paths relative to nagadomi/nunif @ d23721f).  The
 * ctypes binding the reference would add is shown in INTEGRATION.md and
 * implemented in nunif_b200/_lib.py.
 *
 * Conventions
 *   - all pointers are DEVICE pointers unless the name ends in _host
 *   - images are planar float32 CHW / BCHW exactly as the reference passes them
 *   - `stream` is a cudaStream_t passed as void* (0 = legacy default stream)
 *   - divergence / convergence are doubles: the reference folds them into fp32 constants from
 *     Python floats (e.g. float(shift_size * convergence)), and bit-exactness needs the same rounding
 *   - every function returns 0 on success, non-zero on error;
 *     nb200_last_error() returns a thread-local message
 *   - there is no CPU fallback: a call without a usable sm_90 device fails
 */
#ifndef NUNIF_B200_H
#define NUNIF_B200_H

#include <stddef.h>
#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

#define NB200_ABI_VERSION 1

const char* nb200_last_error(void);
int nb200_abi_version(void);
/* device 0..n-1 must be compute capability 10.x; returns non-zero otherwise */
int nb200_check_device(int device);
/* number of kernels this library has launched in this process (bench `gpu_launches`) */
uint64_t nb200_launch_count(void);

/* ------------------------------------------------------------------ *
 * Path A: tiled render (nunif/utils/seam_blending.py)
 * ------------------------------------------------------------------ */

typedef struct nb200_tile_config {
    /* SeamBlending.create_config, seam_blending.py:109-143 */
    int32_t y_h, y_w, h_blocks, w_blocks;
    int32_t pad_l, pad_r, pad_t, pad_b;
    int32_t y_buffer_h, y_buffer_w;
    int32_t input_tile_step, output_tile_step;
} nb200_tile_config;

/* host-side integer planner; bit-exact with the reference. */
int nb200_tile_config_create(int x_h, int x_w, int scale, int offset, int tile_size,
                             int blend_size, nb200_tile_config* out_host);

/* seam_blending.py:82-92: replicate-pad + unfold of tiles [tile0, tile0+n) in raster
 * order into an NHWC fp16 tile batch  dst[n][T][T][cpad]  (channels >= C zero). */
int nb200_tile_unfold(const float* x, int C, int H, int W, const nb200_tile_config* cfg_host,
                      int tile_size, int tile0, int n, void* dst_nhwc_f16, int cpad, void* stream);

/* seam_blending.py:156-174 (update) + :39-40 (get_output) in closed form:
 *   out[C][y_h][y_w] = clamp( sum_t w_t*z_t / sum_t w_t , 0, 1 )
 * over the (at most 4) tiles covering each output pixel, summed in raster tile order.
 * z_all: fp16 planar [h_blocks*w_blocks][C][S][S], S = tile_size*scale - 2*offset.
 * w = create_blend_filter (seam_blending.py:146-153) evaluated in closed form;
 * blend_size==0 reproduces the plain store of :173. */
int nb200_tile_gather_blend(const void* z_all_f16, int C, const nb200_tile_config* cfg_host,
                            int scale, int offset, int tile_size, int blend_size,
                            float* out, void* stream);

/* ------------------------------------------------------------------ *
 * Path A: models.  A model handle owns packed fp16 weights on one device.
 * ------------------------------------------------------------------ */

typedef struct nb200_model nb200_model;

enum {
    NB200_MODEL_UPCUNET = 1,        /* waifu2x.upcunet  (waifu2x/models/cunet.py:139-170) */
    NB200_MODEL_CUNET = 2,          /* waifu2x.cunet    (cunet.py:173-203)                */
    NB200_MODEL_SWIN_UNET_1X = 3,   /* waifu2x.swin_unet_1x (swin_unet.py:208-226)        */
    NB200_MODEL_SWIN_UNET_2X = 4,   /* waifu2x.swin_unet_2x (swin_unet.py:229-251)        */
    NB200_MODEL_SWIN_UNET_4X = 5,   /* waifu2x.swin_unet_4x (swin_unet.py:261-303)        */
    /* Depth-Anything-V2 ViT-S: third-party net the reference loads through torch.hub
     * (iw3/depth_anything_model.py:223-230); state_dict keys `pretrained.*`, `depth_head.*` */
    NB200_MODEL_DEPTH_ANYTHING_V2_S = 6,
    NB200_MODEL_ROW_FLOW_V3 = 7,    /* sbs.row_flow_v3, iw3's default learned stereo warp (iw3/models/row_flow_v3.py) */
    NB200_MODEL_DEPTH_ANYTHING_V2_B = 8,   /* Any_V2_B: ViT-B encoder, 128 head features */
    NB200_MODEL_DEPTH_ANYTHING_V2_L = 9,   /* Any_V2_L: ViT-L encoder (24 blocks), 256 head features */
    NB200_MODEL_DEPTH_AA = 10,             /* iw3.depth_aa, learned anti-aliasing of the depth map (iw3/models/depth_aa.py) */
    NB200_MODEL_MLBW = 11,                 /* sbs.mlbw, multi-layer learned stereo warp, num_layers 2 | 4 (iw3/models/mlbw.py) */
    /* ZoeD_N metric depth: third-party net the reference loads through torch.hub "nagadomi/ZoeDepth_iw3" (iw3/zoedepth_model.py:151-157);
     * state_dict keys of ZoeD_M12_N.pt (`core.core.pretrained.*`, `core.core.scratch.*`, `conv2`, `seed_bin_regressor`, ...).
     * The widths are read off the tensor sizes (BEiT-L/16 for the released checkpoint). */
    NB200_MODEL_ZOEDEPTH_N = 12,
    NB200_MODEL_UPCONV_7 = 13,             /* waifu2x.upconv_7 (waifu2x/models/upconv_7.py:6-38): scale 2, offset 14 */
    NB200_MODEL_VGG_7 = 14,                /* waifu2x.vgg_7    (waifu2x/models/vgg_7.py:6-36): scale 1, offset 7 */
    NB200_MODEL_LIGHT_INPAINT_V1 = 15,     /* inpaint.light_inpaint_v1, iw3's image-mode hole inpainting (iw3/models/light_inpaint_v1.py) */
    NB200_MODEL_ROW_FLOW_V2 = 16,          /* sbs.row_flow_v2, the learned row-flow warp of `--method row_flow_v2` (iw3/models/row_flow_v2.py) */
    NB200_MODEL_SOD_V1 = 17,               /* iw3.sod_v1, the U^2-Net-p saliency network of `--convergence-mode sod_v1` (iw3/models/sod_v1.py) */
    /* ZoeD_Any_N / ZoeD_Any_K, iw3's default depth model: third-party net the reference loads through torch.hub
     * "nagadomi/Depth-Anything_iw3" DepthAnythingMetricDepth (iw3/zoedepth_model.py:12-20,154-170); a Depth-Anything V1 encoder
     * and DPT head under the ZoeDepth bins head, keys `core.core.pretrained.*`, `core.core.depth_head.*`, `conv2`, ...
     * N (indoor) has the "softplus" bins head of ZoeD_N, K (outdoor) the "normed" one (max_depth 80).  Widths read off the
     * tensor sizes.  Run through nb200_zoedepth_forward. */
    NB200_MODEL_ZOEDEPTH_ANY_N = 18,
    NB200_MODEL_ZOEDEPTH_ANY_K = 19,
    /* Depth-Anything V1 Any_S / Any_B / Any_L (iw3/depth_anything_model.py:36-38): the V2 S/B/L networks with the hooks on the
     * last four blocks; checkpoints depth_anything_vit{s,b,l}14.pth.  Run through nb200_depth_anything_forward. */
    NB200_MODEL_DEPTH_ANYTHING_V1_S = 20,
    NB200_MODEL_DEPTH_ANYTHING_V1_B = 21,
    NB200_MODEL_DEPTH_ANYTHING_V1_L = 22,
    /* TransNetV2, the shot-boundary network of iw3's --scene-detect (nunif/utils/transnetv2.py, F=16 L=3 S=2 D=1024); keys
     * `SDDCNN.*`, `frame_sim_layer.*`, `color_hist_layer.fc.*`, `fc1.*`, `cls_layer1.*`, `cls_layer2.*`.  Every BatchNorm is
     * folded into its branch's temporal conv.  Run through nb200_transnetv2_forward. */
    NB200_MODEL_TRANSNET_V2 = 23
};

/* Create a model from named fp32 host tensors using the reference's state_dict
 * keys (nunif/models/utils.py:42-74 load_model / load_state_dict).
 * names[i] is the key, data_host[i] a contiguous float32 buffer of numel[i]
 * elements.  Missing/extra keys are an error, like strict load_state_dict. */
int nb200_model_create(int kind, int n_tensors, const char* const* names,
                       const float* const* data_host, const int64_t* numel,
                       int no_clip, nb200_model** out);
void nb200_model_destroy(nb200_model* m);
/* i2i contract of nunif/models/model.py:65-86 */
int nb200_model_info(const nb200_model* m, int* scale, int* offset, int* blend_size);
/* raw packed weight blob (for the one-time NCCL broadcast that replaces
 * torch.nn.parallel.replicate, nunif/models/data_parallel.py:16,58) */
int nb200_model_weight_blob(nb200_model* m, void** dev_ptr, size_t* bytes);

/* model(minibatch) of seam_blending.py:94-95 under autocast fp16:
 * x: NHWC fp16 [n][T][T][8] (from nb200_tile_unfold, channels 3..7 zero)
 * z: planar [n][3][S][S], S = T*unet_scale/downscale - 2*offset; fp16 for downscale == 1 (the reference's model
 *    output is fp16 under autocast as well), fp32 for downscale 2 | 4 (SwinUNetDownscaled resizes z.float() and
 *    returns fp32, waifu2x/models/swin_unet.py:366-379).
 * downscale in {1,2,4}: 2/4 apply SwinUNetDownscaled (swin_unet.py:366-379). */
int nb200_model_forward(nb200_model* m, const void* x_nhwc_f16, int n, int tile_size,
                        int downscale, void* z_f16, void* stream);

/* nunif.utils.render.tiled_render (render.py:8-19): whole image, device pointers. */
int nb200_tiled_render(nb200_model* m, const float* x, int C, int H, int W, int tile_size,
                       int batch_size, int downscale, float* out, void* stream);

/* The same render with HOST buffers (planar fp32, pinned for full overlap): one H2D copy of the
 * frame, then the output is blended and copied back in bands of finished tile rows on a side
 * stream while later tile batches compute.  `stream` completes after the last band has landed
 * in out_host.  This is the entry point a non-torch binding uses (INTEGRATION.md) and the one
 * bench.py's e2e figure times.  Replaces the host<->device hops around
 * Waifu2x.render (waifu2x/utils.py:218-243; SeamBlending.tiled_render moves each minibatch with .to(device),
 * seam_blending.py:94). */
int nb200_tiled_render_host(nb200_model* m, const float* x_host, int C, int H, int W, int tile_size,
                            int batch_size, int downscale, float* out_host, void* stream);

/* DepthAnythingV2.forward (or the V1 DepthAnything.forward) as called by DepthAnythingModel._forward (iw3/depth_anything_model.py:113-119):
 * x [B][3][H][W] fp32, ImageNet-normalised (nb200_da_preprocess), H and W multiples of 14
 * -> depth [B][H][W] fp32 (relative inverse depth, larger = nearer). */
int nb200_depth_anything_forward(nb200_model* m, const float* x, int B, int H, int W, float* depth,
                                 void* stream);

/* ZoeDepth.forward(x)['metric_depth'] as called by zoedepth_model._forward (iw3/zoedepth_model.py:23-27):
 * x [B][3][H][W] fp32, normalised (x - 0.5) / 0.5 and reflection padded (nb200_zoe_preprocess), H and W multiples of 32
 * (ZoeD_N) or of 14 (ZoeD_Any_N / ZoeD_Any_K, prep_mod 14) -> depth [B][H][W] fp32 (metric depth, larger = farther; batch_infer
 * negates it, zoedepth_model.py:124-130). */
int nb200_zoedepth_forward(nb200_model* m, const float* x, int B, int H, int W, float* depth, void* stream);
/* Host-only helper of the same path: the per-block relative-position table ((2g-1)^2 + 3 rows x heads, learned on a g x g token
 * grid) resampled for a ph x pw grid as MiDaS backbones/beit.py `_get_rel_pos_bias` does (bilinear, the 3 class-token rows kept). */
int nb200_zoe_rel_pos_table(const float* table, int g, int heads, int ph, int pw, float* out);

/* iw3.depth_aa (iw3/models/depth_aa.py:46-87; applied by batch_infer when depth_aa is set, iw3/depth_anything_model.py:153-154):
 * x [B][1][H][W] fp32 -> out, same shape.  mode 0 = forward in eval mode (clamp to [0,1]), 1 = infer (normalise by the
 * min / max of the WHOLE tensor, filter without clamp, de-normalise), 2 = forward(clamp=False). */
int nb200_depth_aa(nb200_model* m, const float* x, int B, int H, int W, int mode, float* out, void* stream);

/* sbs.row_flow_v3 in delta_output mode (iw3/models/row_flow_v3.py:57-68,111-116): x [B][3][h][w] fp32 = depth,
 * divergence feature, convergence feature (make_input_tensor, iw3/backward_warp.py:18-63) -> delta [B][1][h][w]
 * fp32 (the x component; the y component is zero). */
int nb200_row_flow_delta(nb200_model* m, const float* x, int B, int h, int w, float* delta, void* stream);
/* sbs.row_flow_v2 in delta_output mode (iw3/models/row_flow_v2.py:43-47,80-86): same x as nb200_row_flow_delta -> delta
 * [B][1][h][w] fp32 holding the fp16 values of the reference's autocast output (the x component).  Replaces the pre_pad,
 * the convolutions and the crop of _forward_delta_only with one kernel. */
int nb200_row_flow_v2_delta(nb200_model* m, const float* x, int B, int h, int w, float* delta, void* stream);

/* sbs.mlbw in delta_output mode (iw3/models/mlbw.py:96-127,237-245): x [B][3][h][w] fp32 (depth, divergence feature,
 * convergence feature) -> delta [B][L][h][w] (x component of each flow layer) and layer_weight [B][L][h][w] (softmax over
 * the L layers); L = nb200_mlbw_num_layers (2 or 4, read off the state_dict).  A hole_mask model (sbs.mask_mlbw_l2,
 * nb200_mlbw_has_hole_mask = 1) fails here: it runs through nb200_mlbw_delta_hole. */
int nb200_mlbw_delta(nb200_model* m, const float* x, int B, int h, int w, float* delta, float* layer_weight, void* stream);
int nb200_mlbw_num_layers(const nb200_model* m);
/* 1 for a hole_mask model (lv1_out.1.bias with 2 * 2 + 1 = 5 elements, iw3/models/mlbw.py:70-74), else 0. */
int nb200_mlbw_has_hole_mask(const nb200_model* m);
/* _forward_delta_only of a hole_mask model (mlbw.py:232-240): delta and layer_weight as nb200_mlbw_delta, plus
 * hole_logits [B][1][h][w] fp32 (the fp16 conv output of channel 2L, .float()). */
int nb200_mlbw_delta_hole(nb200_model* m, const float* x, int B, int h, int w, float* delta, float* layer_weight,
                          float* hole_logits, void* stream);
/* postprocess_hole_mask(logits, (H, W), threshold) (iw3/backward_warp.py:382-393) up to the threshold: closing(logits, n_iter=1)
 * (iw3/dilation.py:41-64), the align_corners=True bilinear resize to H x W when the size differs, sigmoid(.) > threshold.
 * logits [B][1][h][w] -> out [B][1][H][W] binary fp32.  mirror = 1 gives the mask forward_left computes on the flipped logits
 * (iw3/mlbw_inpaint.py:28-34), flipped back.  threshold = NaN writes the resized closed logits instead of the mask (a view
 * of the first two steps, for tests).  The dilate_inner / dilate_outer steps are nb200_inpaint_mask(binarize=1, closing=0,
 * outer, inner, base_width = w, mirror). */
int nb200_hole_mask(const float* logits, int B, int h, int w, int H, int W, float threshold, int mirror, float* out, void* stream);

/* iw3 forward_inpaint, image mode (iw3/forward_inpaint.py:18-40,69-103).  All tensors planar fp32 in image coordinates.
 * nb200_inpaint_mask: the mask chain of forward_right / forward_left (:18-40): binarize => mask > 0; closing => mask_closing
 *   (iw3/dilation.py:41-64,145-152); then dilate_outer(., outer_iter, base_width) and dilate_inner(., inner_iter, base_width)
 *   (dilation.py:67-98; base_width <= 0 means None).  mirror = 1 gives the result forward_left computes on the flipped mask,
 *   flipped back.  mask, out [B][1][H][W]; any stage may be switched off, so each reference function is available alone.
 * nb200_inpaint_blur: clamp(blur15(mask) + mask, 0, 1), the mask half of LightInpaintV1.preprocess (light_inpaint_v1.py:88-100).
 * nb200_light_inpaint: LightInpaintV1.infer(x, mask) (light_inpaint_v1.py:102-154) of a model of kind
 *   NB200_MODEL_LIGHT_INPAINT_V1: x [B][3][H][W] (the warped eye), mask [B][1][H][W] (from nb200_inpaint_mask) -> out, same
 *   shape as x.  mirror = 1 runs the network on x.flip(-1), mask.flip(-1) and flips the result (forward_left). */
int nb200_inpaint_mask(const float* mask, int B, int H, int W, int binarize, int closing, int outer_iter, int inner_iter,
                       int base_width, int mirror, float* out, void* stream);
/* forward_inpaint.py:74-81: F.interpolate(x, (new_h, new_w), bilinear, antialias=True, align_corners=False) of x [B][3][H][W]
 * (the max_width resize; no clamp). */
int nb200_resize_bilinear_aa(const float* x, int B, int H, int W, int new_h, int new_w, float* out, void* stream);
int nb200_inpaint_blur(const float* mask, int B, int H, int W, float* out, void* stream);
int nb200_light_inpaint(nb200_model* m, const float* x, const float* mask, int B, int H, int W, int mirror, float* out,
                        void* stream);

/* backward_warp(c, grid, delta, delta_scale) of the learned warps (iw3/backward_warp.py:67-83,213-226):
 * c [B][3][H][W], delta [B][1][h][w] fp32 -> out [B][3][H][W] = clamp(grid_sample(c, grid + delta*delta_scale)). */
int nb200_backward_warp_delta(const float* c, const float* delta, int B, int H, int W, int h, int w,
                              double delta_scale, float* out, void* stream);
/* The same warp for an fp16 delta (sbs.row_flow_v2, whose _forward_delta_only returns the autocast fp16 tensor,
 * row_flow_v2.py:80-86): `delta * delta_scale` is then an fp16 tensor op, i.e. delta_scale is rounded to fp16 and so is the
 * product, and only `grid +` runs in fp32 (backward_warp.py:68).  delta holds fp16 values. */
int nb200_backward_warp_delta_f16(const float* c, const float* delta, int B, int H, int W, int h, int w,
                                  double delta_scale, float* out, void* stream);
/* apply_divergence_nn_symmetric's warps (iw3/backward_warp.py:344-379, sbs.row_flow_v3 with symmetric = True) in one launch:
 * left = backward_warp(c, grid, delta, delta_scale), right = backward_warp(c, grid, -delta, delta_scale).  warp_left /
 * warp_right = 0 writes a copy of c for that eye instead (synthetic_view "right" / "left"). */
int nb200_backward_warp_delta_sym(const float* c, const float* delta, int B, int H, int W, int h, int w, double delta_scale,
                                  int warp_left, int warp_right, float* left, float* right, void* stream);

/* iw3 auto-convergence (--convergence-mode sod_v1, iw3/convergence_estimator.py).
 * nb200_sod_forward: SODV1.infer(rgb, depth) (iw3/models/sod_v1.py:47-54) of a NB200_MODEL_SOD_V1 model under CUDA autocast:
 *   rgb [B][3][H][W], depth [B][1][h][w] fp32 -> saliency [B][1][192][192] (fp32 holding the fp16 sigmoid(d0)) and depth192
 *   [B][1][192][192] fp32 (F.interpolate(depth, (192, 192), bilinear, align_corners=False)).
 * nb200_sod_position: ConvergenceEstimator.depth_position_from_ratio(saliency, depth192, pos) (:33-58): per image the depth
 *   values where saliency > 0.5, their torch.quantile 0.1 / 0.9, the centre / range rule, clamp [0, 1] -> out [B] fp32.
 *   saliency, depth [B][n]; n <= 49152.  No host synchronisation.
 * nb200_sod_ema: the EMA of ConvergenceEstimator.__call__ (:60-81) over z [B] in batch order -> out [B].  state: 2 floats on
 *   the device {ema, has_value}; zero them for reset().  reset_host: B host ints (NULL = none), a non-zero entry clears the
 *   state after that frame.  B <= 1024. */
int nb200_sod_forward(nb200_model* m, const float* rgb, int B, int H, int W, const float* depth, int h, int w, float* saliency,
                      float* depth192, void* stream);
int nb200_sod_position(const float* saliency, const float* depth, int B, int n, double pos, float* out, void* stream);
int nb200_sod_ema(float* state, const float* z, int B, const int* reset_host, double decay, float* out, void* stream);

/* TransNetV2.forward (nunif/utils/transnetv2.py:49-87) of a NB200_MODEL_TRANSNET_V2 model on B windows of T frames each
 * (T >= 1; each window is zero-padded in time on its own, as a separate batch entry of the reference):
 *   x [B][T][3][27][48] fp32 (any scale; the colour histograms truncate it to int) -> one_hot [B][T], many_hot [B][T] fp32
 *   logits.  No host synchronisation.  Debug taps 200..205 (DESIGN.md §5). */
int nb200_transnetv2_forward(nb200_model* m, const float* x, int B, int T, float* one_hot, float* many_hot, void* stream);

/* AlphaBorderPadding.forward (nunif/utils/alpha.py:32-57): rgb [3][H][W], alpha [1][H][W] fp32 ->
 * out [3][H][W]: transparent pixels are filled from their opaque neighbours, `offset` rounds
 * (offset = the model's i2i_offset, waifu2x/utils.py:271), then clamped to [0,1]. */
size_t nb200_alpha_border_padding_workspace(int H, int W);
int nb200_alpha_border_padding(const float* rgb, const float* alpha, int H, int W, int offset,
                               float* out, void* workspace, void* stream);

/* tta_split (nunif/transforms/tta.py:20-33): view k in 0..7 of x [C][H][W]
 * (identity, hflip, vflip, vflip+hflip, then the same four of rot90) -> out [C][H][W] (k<4)
 * or [C][W][H] (k>=4).  tta_merge (:36-48): views[k] is the render of view k, i.e.
 * [C][H][W] for k<4 and [C][W][H] for k>=4 (H, W = merged size) -> out = clamp(mean of the
 * inverse-transformed views).  `views` is a host array of 8 device pointers. */
int nb200_tta_transform(const float* x, int C, int H, int W, int k, float* out, void* stream);
int nb200_tta_merge(const float* const* views, int C, int H, int W, float* out, void* stream);

/* ------------------------------------------------------------------ *
 * Path B: iw3 depth post-processing and stereo warps
 * ------------------------------------------------------------------ */

enum { NB200_VIEW_BOTH = 0, NB200_VIEW_LEFT = 1, NB200_VIEW_RIGHT = 2 };
enum { NB200_COMPOSE_NONE = 0,      /* separate left/right planar tensors            */
       NB200_COMPOSE_SBS = 1,       /* iw3/utils.py:466-469 cat([L,R], dim=2)+clamp  */
       NB200_COMPOSE_ANAGLYPH_DUBOIS = 2 /* iw3/anaglyph.py:51-92                    */ };

/* iw3/backward_warp.py:96-121 apply_divergence_grid_sample.
 * c: [B][3][H][W], depth: [B][1][h][w] (any resolution).
 * compose NONE: left,right = [B][3][H][W]; SBS: left = [B][3][H][2W], right unused;
 * ANAGLYPH: left = [B][3][H][W], right unused. */
int nb200_backward_warp(const float* c, const float* depth, int B, int H, int W, int h, int w,
                        double divergence, double convergence, int synthetic_view, int compose,
                        float* left, float* right, void* stream);

/* The same warp with a per-frame convergence tensor (auto-convergence, iw3/utils.py:303-307): convergence is a device array
 * of B fp32 values, and shift_size * convergence is then the fp32 tensor op fp32(shift_size) * convergence[b]. */
int nb200_backward_warp_conv(const float* c, const float* depth, int B, int H, int W, int h, int w,
                             double divergence, const float* convergence, int synthetic_view, int compose,
                             float* left, float* right, void* stream);

/* iw3/forward_warp.py:246-256 apply_divergence_forward_warp (inconsistent_shift=False).
 * depth: [B][1][h][w]; if (h,w)!=(H,W) it is resized like forward_warp.py:146-148.
 * fill!=0 <=> method=="forward_fill".  masks may be NULL (return_mask=False).
 * workspace: nb200_forward_warp_workspace() bytes (may be NULL if depth is full-res). */
size_t nb200_forward_warp_workspace(int B, int H, int W, int h, int w);
int nb200_forward_warp(const float* c, const float* depth, int B, int H, int W, int h, int w,
                       double divergence, double convergence, int fill, int synthetic_view,
                       int width_base, int compose, float* left, float* right,
                       float* left_mask, float* right_mask, void* workspace, void* stream);

/* nb200_forward_warp with a per-frame convergence tensor: device array of B fp32 values, as nb200_backward_warp_conv. */
int nb200_forward_warp_conv(const float* c, const float* depth, int B, int H, int W, int h, int w,
                            double divergence, const float* convergence, int fill, int synthetic_view,
                            int width_base, int compose, float* left, float* right,
                            float* left_mask, float* right_mask, void* workspace, void* stream);

/* iw3/dilation.py:115-142 dilate_edge(x, [x_iter, y_iter]); x,out: [B][1][h][w];
 * workspace: nb200_dilate_edge_workspace() bytes. */
size_t nb200_dilate_edge_workspace(int B, int h, int w);
int nb200_dilate_edge(const float* x, int B, int h, int w, int x_iter, int y_iter,
                      float* out, void* workspace, void* stream);

/* iw3/depth_scaler.py:4-17 with per-frame amin/amax (base_depth_model.py:176-194)
 * followed by the mapper (iw3/mapper.py:29-32): mapper_c < 0 => "none",
 * else distance_to_disparity(x, mapper_c) (div_6 => 0.6).  In place allowed. */
int nb200_minmax_map(const float* depth, int B, int n_per_frame, float mapper_c,
                     float* out, float* minmax_out /* [B][2] or NULL */, void* stream);

/* Stateful depth normaliser: MinMaxBuffer + EMAMinMaxScaler (iw3/depth_scaler.py:33-142; BaseDepthModel.enable_ema /
 * minmax_normalize_chw / flush_minmax_normalize, iw3/base_depth_model.py:152-194).  All values stay on the device; the
 * host only counts calls, so a frame costs three small launches and no synchronisation (csrc/ema_scaler.cu).
 * mode: 0 = "minmax", 1 = "max".  reset: decay < 0 / buffer_size <= 0 keep the current value (:76-86).
 * update: pushes the frame's amin/amax, *filled = the look-ahead buffer is full, i.e. the OLDEST queued frame can now be
 *   normalised (the frame queue itself lives with the caller).
 * normalize: from_ring = 0 uses the EMA values (:108-116), 1 the ring's amin/amax (flush before a value exists, :127-128);
 *   mapper_c >= 0 applies distance_to_disparity(x, mapper_c) afterwards; minmax_out: optional 2 floats on the device. */
typedef struct nb200_ema_scaler nb200_ema_scaler;
int nb200_ema_scaler_create(int buffer_size, double decay, int mode, nb200_ema_scaler** out);
void nb200_ema_scaler_destroy(nb200_ema_scaler* s);
int nb200_ema_scaler_reset(nb200_ema_scaler* s, double decay, int buffer_size);
int nb200_ema_scaler_update(nb200_ema_scaler* s, const float* frame, int n, int* filled, void* stream);
int nb200_ema_scaler_normalize(nb200_ema_scaler* s, const float* frame, int n, int from_ring,
                               float mapper_c, float* out, float* minmax_out, void* stream);
/* iw3/mapper.py:29-32 get_mapper("div_*") alone: distance_to_disparity(x, mapper_c); in place allowed. */
int nb200_depth_mapper(const float* depth, long long n, float mapper_c, float* out, void* stream);

/* Disparity mapper descriptor: iw3/mapper.py:129-151 get_mapper(name) parsed once on the host
 * (nunif_b200/iw3/mapper.py) into up to NB200_MAPPER_MAX_STAGES chained stages, each one function
 * (resolve_mapper_function, :64-120) or the blend a(x)*(1-w) + b(x)*w (:136-147).  Every constant
 * is already rounded to fp32 the way the reference rounds it, so the device evaluates in fp32 in the
 * reference's op order (csrc/mapper.cuh).  Function kinds and their constants k[]:
 *   0 none  identity                        1 pow2  x*x
 *   2 softplus  softplus01_legacy (:7-11)   3 softplus2  its square           k = {min_v, max_v - min_v}
 *   4 softplus01 (mul_*, :14-19)            k = {bias, scale, min_v, max_v - min_v}
 *   5 inv_softplus01 (inv_mul_*, :22-26)    k = {bias, scale, min_v, max_v - min_v}  (fp32 tensor values)
 *   6 distance_to_disparity (div_*, :29-32) k = {c, 1 + c, c / (1 + c), 1 - c / (1 + c)}
 *   7 shift_relative_depth (shift_*, :39-61) k = {A, B, 1 - min_distance, 1 / 17, 1 - 1 / 17}
 * n_stages = 0 is "none".  Fixed size: 528 bytes. */
#define NB200_MAPPER_MAX_STAGES 8
typedef struct nb200_mapper_fn {
    int32_t kind;
    float k[5];
} nb200_mapper_fn;
typedef struct nb200_mapper_stage {
    nb200_mapper_fn a, b;         /* b is read only when blend != 0 */
    int32_t blend;
    float one_minus_w, w, pad;
} nb200_mapper_stage;
typedef struct nb200_mapper {
    int32_t n_stages, pad[3];
    nb200_mapper_stage stage[NB200_MAPPER_MAX_STAGES];
} nb200_mapper;

/* iw3/utils.py:310 get_mapper(args.mapper)(depth) for any mapper name: out = mapper(depth), n elements;
 * in place allowed. */
int nb200_mapper_apply(const float* depth, long long n, const nb200_mapper* mapper_host, float* out, void* stream);
/* nb200_minmax_map with any mapper: iw3/depth_scaler.py:4-17 per frame, then get_mapper(name)
 * (iw3/utils.py:310), in one pass (what stereo_sbs runs).  In place allowed. */
int nb200_minmax_mapper(const float* depth, int B, int n_per_frame, const nb200_mapper* mapper_host,
                        float* out, float* minmax_out /* [B][2] or NULL */, void* stream);

/* Depth export (iw3/utils.py:1323-1328 images, :1378-1382 video, then iw3/base_depth_model.py:203-204
 * save_normalized_depth): depth [B][1][h][w] normalised -> out uint16 [B][H][W] = (0xffff * clamp(d', 0, 1)) truncated,
 * where d' is the mapper applied to each source pixel (mapper_host NULL or 0 stages: none), then, with fit != 0, the
 * antialiased bilinear resize to H x W (align_corners 1: F.interpolate(..., align_corners=True) of the image path,
 * 0: TF.resize of the video path).  fit = 0 ignores H, W and align_corners and writes h x w. */
int nb200_depth_export_u16(const float* depth, int B, int h, int w, const nb200_mapper* mapper_host, int fit, int H, int W,
                           int align_corners, uint16_t* out, void* stream);
/* Depth import (iw3/base_depth_model.py:225-232 load_depth) of B decoded depth maps, channels interleaved as the
 * decoder leaves them, of element type dtype:
 *   NB200_DEPTH_U8   uint8, C = 1..4      NB200_DEPTH_U16  uint16, C = 1   (PNG "L" / "RGB" / "RGBA", "I;16")
 *   NB200_DEPTH_I32  int32, C = 1         NB200_DEPTH_F32  float32, C = 1  (Pillow modes "I" and "F")
 * Integer channels are divided by 0xffff (8-bit maps too) and clamped to [0, 1]; float maps are taken as they are.  The
 * channels are averaged (alpha included), and with has_range != 0 (the iw3_min_depth_value / iw3_max_depth_value text
 * keys) d * (float)(hi - lo) + (float)lo.  out fp32 [B][1][H][W]. */
#define NB200_DEPTH_U8 1
#define NB200_DEPTH_U16 2
#define NB200_DEPTH_I32 3
#define NB200_DEPTH_F32 4
int nb200_depth_import(const void* src, int dtype, int C, int B, int H, int W, double lo, double hi, int has_range,
                       float* out, void* stream);

/* iw3/anaglyph.py:51-92 on already-warped eyes: l,r,out [B][3][H][W] */
int nb200_anaglyph_dubois(const float* l, const float* r, int B, int H, int W, int clip_before,
                          float* out, void* stream);

/* ------------------------------------------------------------------ *
 * Low-level ops (exported for unit tests and micro-benchmarks; the model
 * entry points above are sequences of these)
 * ------------------------------------------------------------------ */

/* F.interpolate(depth, size=(H,W), mode="bilinear", align_corners=True, antialias=True)
 * as used at iw3/forward_warp.py:146-148 (the forward warp fuses this; this entry
 * materialises it). depth [B][1][h][w] -> out [B][1][H][W]. */
int nb200_depth_resize_aa(const float* depth, int B, int h, int w, int H, int W, float* out, void* stream);

/* wgmma implicit GEMM on NHWC fp16 activations (csrc/gemm_wgmma.cuh).
 * kind: 0 linear over flattened pixels, 1 linear with 2-D tiling, 2 conv3x3 valid (4 = conv3x3 zero-padded by 1),
 *       3 conv2x2 stride 2.  Wt: fp16 [N][taps*Cin] with K ordered (ky, kx, c).
 * act: 0 none, 1 LeakyReLU(0.1), 2 GELU(erf), 3 ReLU.
 * out_mode 1: N = 4*cout ordered (dy,dx,co), pixel-shuffle(2) scatter (ConvTranspose2d
 * k2 s2 / Linear+pixel_shuffle).  res: optional residual read at (y+res_cy, x+res_cx). */
int nb200_conv_gemm_f16(const void* A, int B, int Hi, int Wi, int Ci, int Cin, int kind,
                        const void* Wt, int N, const float* bias, int act, void* out, int ldo,
                        int out_mode, int cout, const void* res, int ldr, int res_H, int res_W,
                        int res_cy, int res_cx, int res_before_act, void* stream);

/* kind 1 with out_mode 1 and, instead of a residual, a second A operand A2 [B][2 Hi][2 Wi][ld2] fp16: output pixel
 * (2y+dy, 2x+dx) also multiplies the first Cin2 channels of A2 at that pixel with K columns [Ci, Ci + Cin2) of
 * Wt [N][Ci + Cin2] (a Linear of the skip tensor folded into the GEMM).  cout must be a multiple of 64 or 96. */
int nb200_conv_gemm_pixshuf_a2_f16(const void* A, int B, int Hi, int Wi, int Ci, const void* Wt, int N,
                                   const float* bias, int act, void* out, int ldo, int cout, const void* A2,
                                   int Cin2, int ld2, void* stream);

/* Every field of the engine's implicit-GEMM launch (csrc/gemm.h ConvGemm), for tests that replay the engine's launches.
 * kind: 0 linear over flattened pixels, 1 linear with 2-D tiling, 2 conv3x3 (pad 0 or 1), 3 conv2x2 stride 2,
 *       5 (3,1,1) conv over time: A viewed as [B][T = Hi][Wi][Ci], taps t - dil, t, t + dil, zero padding dil.
 * A: [B][Hi][Wi] pixels of Ci channels, of which the first Cin are read; a_row_stride / a_img_stride (elements, 0 = dense)
 * let A be a cropped view; kind 0 with a_planes > 1 reads K as a_planes planes of Cin channels, a_plane_stride apart.
 * out_mode 0: NHWC output, channel stride ldo; 1: pixel shuffle(2), N = 4*cout; 2: N/cout dense planes split_stride apart.
 * res (optional): residual [B][res_H][res_W][ldr] read at (y + res_cy, x + res_cx), added before the activation when
 * res_before_act.  A2 (out_mode 1, no res): second A operand [B][2 Ho][2 Wo][ld2], its first Cin2 channels are the last
 * Cin2 K columns of Wt. */
typedef struct nb200_gemm_desc {
    int kind, pad, dil, B, Hi, Wi, Ci, Cin;
    long long a_row_stride, a_img_stride;
    int a_planes;
    long long a_plane_stride;
    int N, act, ldo, out_mode, cout;
    long long split_stride;
    int ldr, res_H, res_W, res_cy, res_cx, res_before_act;
    int Cin2, ld2;
} nb200_gemm_desc;
int nb200_conv_gemm_ex_f16(const nb200_gemm_desc* desc, const void* A, const void* Wt, const float* bias, void* out,
                           const void* res, const void* A2, void* stream);

/* The ViT / BEiT attention of the depth models: qkv [B][N][3][heads][64] fp16 -> out [B][N][heads][64] fp16,
 * softmax(q k^T / 8 + bias) v.  bias_log2e (optional): fp32 [heads][N][ldb], already multiplied by log2(e);
 * ldb is even and >= N rounded up to 64. */
int nb200_flash_attention_f16(const void* qkv, void* out, int B, int N, int heads, const float* bias_log2e, int ldb,
                              void* stream);

/* The WindowMHA2d core of the WABlock (row_flow_v3, mlbw, depth_aa; csrc/window_mha.h): qkv fp16 [B][H][W][3C] (q | k | v),
 * ws x ws windows, `heads` heads of C / heads channels, bias fp32 [N][N] (N = ws * ws) added to the scaled scores,
 * out fp16 [B][H][W][C].  pad_y / pad_x are 0 or ws / 2 (a shifted direction; the padded grid must tile into whole windows):
 * padded tokens have k | v = qkv_bias[C..3C) (fp32, required with padding).  Layouts: 3x3 and 4x4 with 2 heads of 32, 4x4
 * with 4 heads of 32, 8x8 with 2 heads of 16. */
int nb200_window_mha_f16(const void* qkv, const float* qkv_bias, const float* bias, void* out, int B, int H, int W, int C,
                         int ws, int heads, int pad_y, int pad_x, void* stream);
/* ReplicationPad2d(1) of x fp16 [B][H][W][C] -> out [B][H+2][W+2][C]; C % 8 == 0. */
int nb200_reppad1_f16(const void* x, int B, int H, int W, int C, void* out, void* stream);
/* The ViT block's residual add + LayerNorm (eps 1e-6) on the fp32 residual stream: x32 [rows][dim] += fp32(delta) (delta
 * fp16, may be NULL: no add, x32 is not written), out fp16 = LayerNorm(x32) * w + b (may be NULL: no output).
 * dim in {256, 384, 768, 1024}. */
int nb200_add_layernorm_f32(float* x32, const void* delta, const float* w, const float* b, void* out, long long rows, int dim,
                            void* stream);
/* Bilinear resize, align_corners=True, of x fp16 [B][h][w][C] -> out [B][H][W][C] (fp32 interpolation); C % 8 == 0. */
int nb200_upsample_bilinear_f16(const void* x, int B, int h, int w, int C, void* out, int H, int W, void* stream);

/* ZoeDepth bins head kernels (csrc/zoe_kernels.h, where each is specified): y = e + bilinear(prev) (fp16 NHWC, C % 8 == 0);
 * out = softplus(x) (fp32); the normed seed bin centres; the attractor layer (normed = 0: AttractorLayerUnnormed, sorted
 * must be NULL; normed = 1: AttractorLayer, sorted optional); the ConditionalLogBinomial input concat and its final 4-output
 * conv + log-binomial mixture; and the BEiT relative-position bias expansion (bias [heads][N][ldb], N = ph * pw + 1,
 * columns N..ldb-1 are not written). */
int nb200_zoe_add_upsampled_f16(const void* e, const void* prev, int B, int h, int w, int C, int H, int W, void* y,
                                void* stream);
int nb200_zoe_softplus_f32(const void* x, float* out, long long n, void* stream);
int nb200_zoe_seed_normed_f32(const void* s, long long npix, float min_depth, float max_depth, float* out, void* stream);
int nb200_zoe_attractor_f32(const void* apre, int lda, int na, const float* prev_bin, int B, int h, int w, int H, int W,
                            int normed, float min_depth, float max_depth, float* out, float* sorted, void* stream);
int nb200_zoe_clb_concat_f16(const void* act, const float* rel, const void* emb, int B, int h, int w, int H, int W, void* A,
                             void* stream);
int nb200_zoe_clb_final_f32(const void* g, int ldg, const float* w2, const float* b2, const float* bins, int B, int h, int w,
                            int H, int W, float* depth, void* stream);
int nb200_zoe_expand_rel_bias_f32(const float* table, int ph, int pw, int heads, float* bias, int ldb, void* stream);

/* The hand-written convolutions of the waifu2x models and the SE block, through the host functions the networks call (so
 * nb200_tune_set(7, 1) selects their SIMT kernels here too).  w / b / w1 / b1 / w2 / b2 are HOST fp32 tensors in the PyTorch
 * layout (Conv2d [co][ci][kh][kw], ConvTranspose2d [ci][co][kh][kw], bias [co]), packed by the networks' own packers into a
 * stream-ordered workspace; activations are device fp16.
 *   stem: x [n][Hi][Wi][8] (channel 3 must be 0, channels 4..7 are not read), w [cout][3][3][3] -> out [n][Hi-2][Wi-2][ldo],
 *         LeakyReLU(0.1); channels cout..cout_pad-1 are written as 0, cout_pad..ldo-1 are not written.  cout_pad 32 or 64.
 *   tail: x [n][Hi][Wi][64]; mode 0: Conv2d(64, 3, 3) valid, mode 1: ConvTranspose2d(64, 3, 4, 2, 3).  epi 0: out NHWC8
 *         [n][Ho][Wo][8] (3 channels, optional clamp(0, 1), 5 zeros); epi 1 (mode 0 only): out planar [n][3][Ho][Wo] =
 *         clamp(conv + z1[:, 20:20+Ho, 20:20+Wo, :3]) with z1 NHWC8 [n][z1H][z1W][8].
 *   head: x [n][Hi][Wi][cin]; mode 0 (cin 128): Conv2d(cin, 3, 3), mode 1 (cin 256): ConvTranspose2d(cin, 3, 4, 2, 3);
 *         out planar [n][3][Ho][Wo] = clamp(conv, 0, 1).
 *   se:   x [n][H][W][C] fp16 scaled in place by sigmoid(conv2(relu(conv1(mean over H, W)))); C 64 or 128, conv1 [C/8][C],
 *         conv2 [C][C/8]. */
int nb200_stem_conv_f16(const void* x, const float* w, const float* b, int cout, int cout_pad, int n, int Hi, int Wi, void* out,
                        int ldo, void* stream);
int nb200_tail_conv_f16(const void* x, const float* w, const float* b, int mode, int epi, int n, int Hi, int Wi, void* out,
                        const void* z1, int z1H, int z1W, int clip, void* stream);
int nb200_head_conv_f16(const void* x, const float* w, const float* b, int mode, int cin, int n, int Hi, int Wi, void* out,
                        void* stream);
int nb200_se_block_f16(void* x, const float* w1, const float* b1, const float* w2, const float* b2, int n, int H, int W, int C,
                       void* stream);
/* SwinUNet's to_image tail: y fp16 [n][Hs][Ws][cs] with channel c*r*r + dy*r + dx (F.pixel_shuffle) -> z planar [n][3][S][S],
 * S = Hs * r / down; down 1: fp16 clamp(pixel_shuffle(y), 0, 1); down 2 / 4: fp32 clamp(bicubic antialias resize (ATen
 * upsample_bicubic2d_aa) of that clamp, 0, 1).  Hs == Ws. */
int nb200_to_image_f16(const void* y, int n, int Hs, int Ws, int cs, int r, int down, void* z, void* stream);
/* One REBNCONV of iw3.sod_v1 (csrc/sod.cu sod_conv_kernel): out[..., out_off:out_off+cout] = fp16(relu(fp16(fp16(conv3x3(
 * in[..., in_off:in_off+cin], dilation and padding dil)) + bias)) [+ res[..., :cout]]), NHWC fp16 with pixel strides in_ld /
 * out_ld / res_ld (res may be NULL).  wt fp16 [cout][9][cin] (k = tap * cin + c), bias fp32; cin % 16 == 0, cout 16 or 64. */
int nb200_sod_conv_f16(const void* in, int in_ld, int in_off, int cin, const void* wt, const float* bias, int cout, int dil,
                       void* out, int out_ld, int out_off, const void* res, int res_ld, int B, int H, int W, void* stream);

/* The input and output stages of the learned stereo networks and of depth_aa (csrc/rowflow_kernels.h, mlbw_kernels.h,
 * depth_aa_kernels.h, where each is specified), with the geometry their model forwards compute; weight / bias are HOST fp32
 * tensors in the PyTorch layout.  A geometry whose padded grid does not hold the image is refused before any launch.
 *   row_flow_prep:      x [B][3][h][w] fp32 -> tokens [B][Hp][Wt][32] fp16 (replicate pad to Hp x 8 Wt, pixel_unshuffle (1, 8)).
 *   row_flow_last_conv: tokens [B][Hp][Wt][64] fp16 -> delta [B][1][h][w] (pixel_shuffle, crop, ReplicationPad2d(1), conv 3x3
 *                       8 -> 1, fp16 values); weight [1][8][3][3], bias [1].
 *   mlbw_prep:          x [B][3][H][W] -> tokens [B][Hp][Wt][8 C1] fp16 (pads ph1 / pw1 leading, lv1_in); weight [C1][3][1][9].
 *   mlbw_out:           tokens t, t0 [B][Hp][Wt][8 C1] fp16 -> delta, layer_weight [B][L][H][W] and, with hole (L = 2 only),
 *                       the hole logits [B][1][H][W]; weight [2L (+1)][C1][1][9].  L 2 or 4.
 *   depth_aa_minmax:    minmax[0], minmax[1] = min, max of x[0..n) (device fp32).
 *   depth_aa_prep:      x [B][1][H][W] -> tokens [B][Hh][Wh][32] fp16, normalised by minmax unless it is NULL; weight [32][4][1][1].
 *   depth_aa_out:       tokens [B][Hh][Wh][32] fp16, x -> out [B][1][H][W]: x + filter, clamped to [0, 1] with clamp, or with
 *                       minmax the de-normalised infer output; weight [4][32][1][1]. */
int nb200_row_flow_prep_f16(const float* x, int B, int h, int w, int Hp, int Wt, void* out, void* stream);
int nb200_row_flow_last_conv_f32(const void* x, int B, int Hp, int Wt, int h, int w, const float* weight, const float* bias,
                                 float* delta, void* stream);
int nb200_mlbw_prep_f16(const float* x, int B, int H, int W, int ph1, int pw1, int Hp, int Wt, int C1, const float* weight,
                        const float* bias, void* out, void* stream);
int nb200_mlbw_out_f32(const void* t, const void* t0, int B, int H, int W, int ph1, int pw1, int Hp, int Wt, int C1, int L,
                       const float* weight, const float* bias, float* delta, float* layer_weight, float* hole, void* stream);
int nb200_depth_aa_minmax_f32(const float* x, long long n, float* minmax, void* stream);
int nb200_depth_aa_prep_f16(const float* x, const float* minmax, int B, int H, int W, int ph1, int pw1, int Hh, int Wh,
                            const float* weight, const float* bias, void* out, void* stream);
int nb200_depth_aa_out_f32(const void* tok, const float* x, const float* minmax, int B, int H, int W, int ph1, int pw1, int Hh,
                           int Wh, const float* weight, const float* bias, int clamp, float* out, void* stream);

/* shifted-window attention core between the qkv and proj Linears
 * (torchvision swin_transformer.py:166-221), window 6x6, 6 heads.
 * qkv: three dense planes q | k | v, each [B][H][W][C] fp16 (how the engine's qkv GEMM writes them)
 * -> out [B][H][W][C] fp16; bias_table fp32 [121][6].  A shift > 0 needs H and W both 6 (no shift) or both larger. */
int nb200_window_attention_f16(const void* qkv, const float* bias_table, void* out, int B,
                               int H, int W, int C, int heads, int shift, void* stream);

/* Tail of one SwinTransformerBlock (torchvision swin_transformer.py:228 proj, :453-455; MLP = Linear-GELU-Linear,
 * ratio 2, Identity norms: waifu2x/models/swin_unet.py:16-17,31), on the engine's GEMM (csrc/swin_block.cu):
 *   x1 = x + att @ wp^T + bp   (att == NULL: x1 = x);   x <- x1 + gelu(x1 @ w1^T + b1) @ w2^T + b2
 * x, att: [T][C] fp16 (x updated in place); wp [C][C], w1 [2C][C], w2 [C][2C] fp16; biases fp32.  C in {96, 192}. */
int nb200_swin_mlp_fused_f16(void* x, const void* att, long long T, int C, const void* wp,
                             const float* bp, const void* w1, const float* b1, const void* w2,
                             const float* b2, void* stream);

/* The same tail as the network's last block runs it, with to_image's Linear fused: the block output is not written to x
 * (x is left unchanged); y [T][cs] = output @ wy^T + by is written instead.  att is required; wy [cs][C] fp16, by [cs]
 * fp32; cs = 48 at C = 192, 16 at C = 96. */
int nb200_swin_mlp_fused_y_f16(void* x, const void* att, long long T, int C, const void* wp,
                               const float* bp, const void* w1, const float* b1, const void* w2,
                               const float* b2, void* y, int cs, const void* wy, const float* by,
                               void* stream);

/* Head of one SwinTransformerBlock: qkv Linear + shifted 6x6 window attention (swin_transformer.py:166-221;
 * everything but the proj Linear), the engine's fused block head (csrc/swin_attention_mma.cu).
 * x, att: [B][H][W][C] fp16; wqkv [3C][C] fp16 and bqkv [3C] fp32 in the reference's row order
 * (q | k | v), bias_table = relative_position_bias_table [121][6] fp32.  C in {96, 192}, H and W multiples of 6.
 * A shift > 0 needs H and W both 6 (no shift) or both larger; exactly one side of 6 is refused. */
int nb200_swin_attn_fused_f16(const void* x, const void* wqkv, const float* bqkv,
                              const float* bias_table, void* att, int B, int H, int W, int C,
                              int shift, void* stream);

/* Frame-edge conversions (nunif/utils/video.py:218-223 to_tensor, :236-246 from_tensor,
 * iw3/utils.py:274-289 hwc_to_chw_float): x [B][H][W][3] uint8 (bits=8) or uint16 (bits=16)
 * <-> [B][3][H][W] fp32 in [0,1]; the fp32 -> integer direction rounds half to even. */
int nb200_hwc_to_chw_f32(const void* x, int bits, int B, int H, int W, float* out, void* stream);
int nb200_chw_f32_to_hwc(const float* x, int bits, int B, int H, int W, void* out, void* stream);

/* nunif/utils/video.py:309-416 hdr2sdr (steps 1-6), the HDR input stage of input_reformatter (:1025-1041): PQ (HDR10) or
 * HLG BT.2020 -> Hable tone map -> BT.709 / BT.601 SDR, one fused pass.  x [B][H][W][3] uint16 rgb48, full range;
 * trc = the stream's color_trc code (16 PQ, 18 HLG); params_host = {pq_exposure, pq_white_point, hlg_exposure,
 * hlg_white_point, hlg_saturation_gain} as the Python floats (defaults 110, 5, 1.2, 0.8, 0.9).
 * out_float = 0: out [B][H][W][3] uint16, the rgb48 frame hdr2sdr returns (truncating cast);
 * out_float = 1: out [B][3][H][W] fp32, that frame / 65535 exactly as nb200_hwc_to_chw_f32 makes it.
 * Every op rounds to fp32 as ATen's CUDA kernels do; the 3x3 matrix (torch.mm) sums in its own order. */
enum { NB200_TRC_PQ = 16, NB200_TRC_HLG = 18, NB200_SDR_BT709 = 0, NB200_SDR_BT601 = 1 };
int nb200_hdr2sdr(const uint16_t* x, int B, int H, int W, int trc, int colorspace, const double* params_host,
                  int out_float, void* out, void* stream);

/* Film grain (waifu2x --grain: waifu2x/ui_utils.py:58-61 images, :167-175 video) through nunif/utils/rgb_noise.py.
 * Noise: each normal is Philox4x32-10 keyed by seed at the counter (element, 2 * channel + field, frame, offset), turned
 * into N(0, 1) by Box-Muller; field 0 = the full-resolution field, field 1 = level 2's (H / 2) x (W / 2) field.  A different
 * sample from the distribution of the reference's torch.randn draws, not their bits.
 * nb200_rgb_noise: rgb_noise_like (rgb_noise.py:5-17) -> out [B][C][H][W] fp32; frame b of the batch uses frame word b.
 *   level 1: the full field; level 2: 0.5 * full + 0.5 * half upsampled by F.interpolate's nearest rule (H, W >= 2). */
int nb200_rgb_noise(uint64_t seed, uint32_t offset, int level, int B, int C, int H, int W, float* out, void* stream);
/* nb200_apply_rgb_noise: apply_rgb_noise (rgb_noise.py:20-36) of rgb [B][C][H][W] fp32, in the reference's fp32 op order.
 *   noise [B][C][H][W], or null: frame b's noise is nb200_rgb_noise(seed, offset + b, level) of that frame alone.
 *   buffer [C][H][W], or null: the video path's temporal noise buffer (ui_utils.py:167-175), advanced over the B frames in
 *   order, b = b * (1 - speed) + n * speed, and the blended buffer applied; buffer_reset = 1: frame 0 copies its noise into
 *   the buffer (the reference's first frame and every frame-shape change).
 *   params_host = {strength, gamma, light_decay_strength, speed} as the Python floats.
 *   out_bits = 0: out [B][C][H][W] fp32; 8 / 16: out [B][H][W][3] uint8 / uint16, (y * 255 | 65535).round_() as
 *   from_tensor (nunif/utils/video.py:236-245) makes the encoder's frame (C must be 3). */
int nb200_apply_rgb_noise(const float* rgb, int B, int C, int H, int W, const float* noise, uint64_t seed, uint32_t offset,
                          int level, float* buffer, int buffer_reset, const double* params_host, int light_decay, int out_bits,
                          void* out, void* stream);

/* DepthAnything batch_preprocess (iw3/depth_anything_model.py:69-110): size rule (host,
 * integers) and the fused antialiased-bilinear resize + clamp + ImageNet normalise:
 * x [B][3][H][W] fp32 in [0,1] -> out [B][3][new_h][new_w] fp32. */
int nb200_da_preprocess_size(int H, int W, int lower_bound, int max_aspect_ratio,
                             int limit_resolution, int* new_h, int* new_w);
int nb200_da_preprocess(const float* x, int B, int H, int W, int new_h, int new_w, float* out,
                        void* stream);

/* iw3's NULL depth model (iw3/null_depth_model.py:17-21 NullDepth.forward): F.interpolate(x, (R, R), mode="bilinear",
 * align_corners=False) then x.mean(dim=1, keepdim=True) in one pass, with the arithmetic of ATen's CUDA kernels:
 * x [B][3][H][W] fp32 -> out [B][1][R][R] fp32.  out must not alias x. */
int nb200_null_depth(const float* x, int B, int H, int W, int R, float* out, void* stream);

/* ZoeDepth batch_preprocess (iw3/zoedepth_model.py:30-85): size rule (host integers) and the fused
 * antialiased resize + reflection pad (nunif/modules/reflection_pad2d.py:57-68) + clamp + normalise:
 * x [B][3][H][W] -> out [B][3][frame_h + 2*pad_h][frame_w + 2*pad_w] (== new_h x new_w in landscape). */
int nb200_zoe_preprocess_size(int H, int W, int h_height, int v_height, int mod, int* new_h,
                              int* new_w, int* pad_h, int* pad_w, int* frame_h, int* frame_w);
int nb200_zoe_preprocess(const float* x, int B, int H, int W, int frame_h, int frame_w, int pad_h,
                         int pad_w, float* out, void* stream);

/* iw3/anaglyph.py:95-110 apply_anaglyph_redcyan: l, r [B][3][H][W] fp32 -> out [B][3][H][W]. */
enum { NB200_ANAGLYPH_DUBOIS = 0, NB200_ANAGLYPH_DUBOIS2 = 1, NB200_ANAGLYPH_COLOR = 2, NB200_ANAGLYPH_GRAY = 3,
       NB200_ANAGLYPH_HALF_COLOR = 4, NB200_ANAGLYPH_WIMMER = 5, NB200_ANAGLYPH_WIMMER2 = 6 };
int nb200_anaglyph(const float* l, const float* r, int B, int H, int W, int type, float* out, void* stream);

/* TF.resize(x, (oh, ow), BICUBIC, antialias=True) on `planes` fp32 H x W planes (half-SBS / half-TB and the
 * max-output-size resize of postprocess_image, iw3/utils.py:445-485); clamp01_out applies the following clamp. */
int nb200_resize_bicubic_aa(const float* x, int planes, int H, int W, int oh, int ow, int clamp01_out,
                            float* out, void* stream);
/* The same resize with F.interpolate's align_corners flag (preprocess_image's --max-output-height resize,
 * iw3/utils.py:247-271, uses align_corners=True): ATen's scale becomes (in - 1) / (out - 1); align_corners = 0 is
 * nb200_resize_bicubic_aa. */
int nb200_resize_bicubic_aa_ac(const float* x, int planes, int H, int W, int oh, int ow, int clamp01_out,
                               int align_corners, float* out, void* stream);

/* torch.rot90(x, k, (-2, -1)) of `planes` fp32 H x W planes (--rotate-left k = 1, --rotate-right k = 3,
 * iw3/utils.py:247-252): x [planes][H][W] -> out [planes][W][H], bit-exact.  out must not alias x. */
int nb200_rot90(const float* x, int planes, int H, int W, int k, float* out, void* stream);

/* The autocrop detector (nunif/utils/autocrop.py:6-207) on x [B][3][H][W] fp32, one frame at a time as the reference's
 * detect_tb / detect_lr:  Y = r*0.299 + g*0.587 + b*0.114 (fp32, no contraction).
 *   black != 0 (black, black_tb, black_lr): Y clamped to [16/255, 235/255]; a line is a bar when its mean <= 32/255 and
 *     max|Y - mean| < 16/255 (mean = sum * fl(1/n) as ATen's CUDA mean; the summation order is the kernel's own).
 *   black == 0 (flat, flat_tb, flat_lr): a line is a bar when fl(count(|Y - median| < 16/255) * fl(1/n)) > 0.99, median
 *     the exact lower median (torch.median).
 * axes: bit 0 rows (detect_tb), bit 1 columns (detect_lr).  Every output may be NULL: mask_tb [B][H] / mask_lr [B][W]
 * (uint8 0 / 1), count_tb [H] / count_lr [W] int32 (+= the mask, summed over the B frames: AutoCropDetector.update),
 * stat_tb [B][H] / stat_lr [B][W] (black: the mean, flat: the median).  Makes no host synchronisation.
 * Rows in flat mode need W <= 12544, columns need H <= 6144 (shared-memory staging). */
int nb200_autocrop_detect(const float* x, int B, int H, int W, int black, int axes, unsigned char* mask_tb,
                          unsigned char* mask_lr, int* count_tb, int* count_lr, float* stat_tb, float* stat_lr,
                          void* stream);
/* AutoCropDetector.get_crop (:47-69) on the device: bar_i = fl(count_i * fl(1 / frame_count)) >= threshold (ATen's
 * CUDA division by a host scalar); out[0], out[1] = first / last non-bar row, out[2], out[3] = first / last non-bar
 * column, -1 when there is none or the counts are NULL.  out: 4 int32 on the device. */
int nb200_autocrop_bounds(const int* count_tb, int H, const int* count_lr, int W, int frame_count, float threshold,
                          int* out, void* stream);

/* VR180 output (iw3/equirectangular.py:7-40; iw3/utils.py:441-443): zero-pad to 1.5 x the longer edge, bicubic grid_sample
 * (zeros, align_corners=True) through x' = k tan(az), y' = k tan(el)/cos(az), clamp [0,1].
 * c [C][H][W] -> out [C][out_h][out_w] with (out_h, out_w) from nb200_equirectangular_size (host rule). */
int nb200_equirectangular_size(int H, int W, int* out_h, int* out_w);
int nb200_equirectangular(const float* c, int C, int H, int W, float* out, void* stream);

/* Kernel-class device timing (CUDA events around every launch of this library) used by
 * bench.py for the live roofline figure.  report writes a JSON object
 * {"gemm": {"launches": n, "ms": t, "work": flops_or_bytes}, ...} and synchronises the device. */
int nb200_tune_set(int key, int value);   /* kernel-selection knobs (csrc/gemm.cu g_tune), for tests and A/B runs */
int nb200_debug_tap(int id, void* dev_buf, size_t capacity);  /* copy intermediate `id` of nb200_zoedepth_forward (ids 0..14,
                                                               15 = the sorted centres of a normed head, DESIGN.md §5)
                                                               or nb200_light_inpaint (ids 100..173, DESIGN.md §5)
                                                               or nb200_transnetv2_forward (ids 200..205) to dev_buf */
int nb200_profile_enable(int on);
int nb200_profile_report(char* buf, size_t cap);
int nb200_profile_dump(char* buf, size_t cap);   /* one CSV line per timed launch: class,ms,work,read_bytes,write_bytes */

/* Launch recorder for tests: a non-zero `on` clears the record and appends one line per launch of the kinds its bits
 * select; on = 0 stops.  Off by default; recording changes no launch.  Other bits are refused.
 *   bit 0 (on = 1): gemm attn swin_attn swin_mlp (the implicit GEMM, the ViT attention, the fused Swin-block head and tail)
 *   bit 1 (on = 2): wmha reppad ln upbl zadd_up zsoftplus zseed zattr zclb_concat zclb_final zrelbias (the WABlock core and
 *                   pad, the ViT add + LayerNorm, the DPT upsample and the ZoeDepth bins head)
 *   bit 2 (on = 4): stem tail head se toimg sodconv (the waifu2x stem, tail and head convolutions, the SE block, to_image
 *                   and the SOD REBNCONV)
 *   bit 3 (on = 8): rfprep rflast rf2 mlprep mlout holemask aaminmax aaprep aaout (the input and output stages of row_flow_v3,
 *                   mlbw and depth_aa, the fused row_flow_v2 delta kernel and the hole mask of mask_mlbw_l2)
 * A line is `kind,name=value,name=value,...`: the launch's fields without its pointers, named where the host code writes
 * them.  Values are integers (flags 0 or 1) or fp32 values printed with 9 significant digits.  recorded_launches_named copies
 * the lines (NUL-terminated) like nb200_profile_dump; recorded_launches copies them without the names (`kind,value,...`, the
 * values in the same order).  Both fail if cap is too small.  A few kinds record before their last argument check (zrelbias
 * before its ldb check, mlout before its L check), so a refused call of those can leave a line for a launch that never ran. */
int nb200_record_launches(int on);
int nb200_recorded_launches(char* buf, size_t cap);
int nb200_recorded_launches_named(char* buf, size_t cap);

#ifdef __cplusplus
}
#endif
#endif /* NUNIF_B200_H */
