#pragma once
#include "common.cuh"

namespace nb200 {
// iw3 forward_inpaint / inpaint.light_inpaint_v1 (csrc/inpaint_kernels.cu).  Masks and frames are planar fp32 [B][1|3][H][W]
// in image coordinates; `mirror` = the network sees the frame flipped left-right (forward_left, iw3/forward_inpaint.py:28-40).

// mask > 0 (binarize), mask_closing (closing), then the OR of each pixel's run [x - n_left, x + n_right] of the same row
// (dilate_outer / dilate_inner in image coordinates).  tmp: B*H*W floats.
int inpaint_mask(cudaStream_t st, const float* mask, int B, int H, int W, int binarize, int closing, int n_left, int n_right,
                 float* tmp, float* out);
// clamp(blur15(mask) + mask, 0, 1) written in network coordinates (flipped when mirror).  tmp: B*H*W floats.
int inpaint_blur(cudaStream_t st, const float* mask, int B, int H, int W, int mirror, float* tmp, float* out);
// stem: hole zeroing, (x - 0.5) / 0.5, replicate pad to Hp x Wp, pixel_unshuffle(4), 1x1 conv 48 -> 96 + LeakyReLU(0.2), and the
// mask token where the blurred mask's 4x4 amax > 0.99.  w: fp32 [48][96], b, mask_bias: [96].  out: [B][Hp/4][Wp/4][96] fp16.
int inpaint_stem(cudaStream_t st, const float* x, const float* hole, const float* blur, int B, int H, int W, int Hp, int Wp,
                 int mirror, const float* w, const float* b, const float* mask_bias, __half* out);
// LN1 (no bias, eps 1e-5) of x [B][H][W][C] into t [B][H+2p][W+2p][C] with a zero ring of p, and x <- 2x (the block's
// doubled shortcut, attention.py:643-660 + light_inpaint_v1.py:46).  C in {96, 192}.
int inpaint_ln_pad(cudaStream_t st, __half* x, const float* g, __half* t, int B, int H, int W, int C, int p);
// Token mixing of every ws x ws window of u [B][Hq][Wq][4C] (proj_in output, u | v): v' = Ws . LN2(v) + bs, u <- u * v'.
// wfrag: Ws as fp16 mma.sync A fragments, wf: Ws fp32 [N][N] (SIMT cross-check), bs [N], g2 [2C].
int inpaint_token_mix(cudaStream_t st, __half* u, int B, int Hq, int Wq, int C, int ws, const __half* wfrag, const float* wf,
                      const float* bs, const float* g2);
// Replicate-pad x [B][H][W][cs] by 1 into out [B][H+2][W+2][co]; glu: out = x[:cs/2] * sigmoid(x[cs/2:]), channels >= cs/2 zero.
int inpaint_pad(cudaStream_t st, const __half* x, int B, int H, int W, int cs, int co, int glu, __half* out);
// Tail: pixel_shuffle(4) of y [B][Hp/4][Wp/4][48], crop, composite with the hole-zeroed frame and the blurred mask, clamp,
// un-mirror: out [B][3][H][W] fp32.
int inpaint_tail(cudaStream_t st, const __half* y, const float* x, const float* hole, const float* blur, int B, int H, int W,
                 int Hp, int Wp, int mirror, float* out);
}  // namespace nb200
