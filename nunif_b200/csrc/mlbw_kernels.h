// Non-GEMM kernels of the multi-layer learned stereo warp sbs.mlbw (mlbw.cu); wiring in mlbw_model.inl.
#pragma once
#include "common.cuh"

namespace nb200 {

// replicate-pad (ph1 / pw1 leading) + lv1_in (ReplicationPad (4,4,0,0) + Conv2d(3, C1, (1,9)) + LeakyReLU(0.2)) + pixel_unshuffle (1, 8):
// x fp32 [B][3][H][W] -> tokens fp16 [B][Hp][Wt][8 * C1] (channel = c * 8 + sw)
int mlbw_prep(cudaStream_t st, const float* x, int B, int H, int W, int ph1, int pw1, int Hp, int Wt, int C1, const float* w_in,
              const float* b_in, __half* out);
// pixel_shuffle (1, 8) of (t + t0) + lv1_out (ReplicationPad (4,4,0,0) + Conv2d(C1, 2L [+ 1], (1,9))) + crop + chunk + softmax over the
// layers: -> delta fp32 [B][L][H][W], layer_weight fp32 [B][L][H][W]; hole != nullptr (hole_mask head, L = 2): the fp16-rounded hole
// logits fp32 [B][1][H][W] of output channel 2L
int mlbw_out(cudaStream_t st, const __half* t, const __half* t0, int B, int H, int W, int ph1, int pw1, int Hp, int Wt, int C1, int L,
             const float* w_out, const float* b_out, float* delta, float* lw, float* hole);
// The first three steps of postprocess_hole_mask (iw3/backward_warp.py:382-393): closing(logits, n_iter=1) (3x3 max then 3x3 min,
// -inf padding, dilation.py:41-64), the align-corners bilinear resize from h x w to H x W (skipped when the sizes are equal), and
// sigmoid(.) > threshold: logits fp32 [B][1][h][w] -> binary mask fp32 [B][1][H][W].  mirror = 1: the mask computed on the flipped
// logits (forward_left, iw3/mlbw_inpaint.py:28-34), flipped back.  threshold = NaN: out = the resized closed logits.
int hole_mask(cudaStream_t st, const float* logits, int B, int h, int w, int H, int W, float threshold, int mirror, float* out);

}  // namespace nb200
