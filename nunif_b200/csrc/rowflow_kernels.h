// Non-GEMM kernels of the learned stereo warp sbs.row_flow_v3 (rowflow_kernels.cu); wiring in rowflow_model.inl.
#pragma once
#include "common.cuh"

namespace nb200 {

// x fp32 [B][3][h][w] -> tokens fp16 [B][Hp][Wt][32]: replicate-pad to (Hp, Wt*8), pixel_unshuffle (1, 8) (channel = c*8 + sw),
// channels 24..31 zero
int rf_prep(cudaStream_t st, const float* x, int B, int h, int w, int Hp, int Wt, __half* out);
// pixel_shuffle (1, 8) + crop to (h, w) + replication pad 1 + conv3x3 (8 -> 1): tokens [B][Hp][Wt][64] -> delta fp32 [B][1][h][w]
int rf_last_conv(cudaStream_t st, const __half* x, int B, int Hp, int Wt, int h, int w, const float* wt72, float bias, float* delta);

// sbs.row_flow_v2 (rowflow_v2.cu): one fused kernel, RF2_ROWS x RF2_T output pixels per CTA.  Its weights are one parameter
// block of RF2_PARAM_BYTES (packed by rowflow_v2_model.inl) that each CTA copies to shared memory:
//   mma.sync B fragments in lane order [k-step][n8 tile][lane] (uint2), k = (row * taps + tap) * cin + ci:
//     RF2_FRAG1 conv #1 (9 k-steps x 2 tiles), RF2_FRAG2 conv #2 (9 x 4), RF2_FRAG3 conv #3 (18 x 4), RF2_FRAG4 3x3 (18 x 1)
//   then fp32 (fp16-representable) scalars at RF2_F32, indexed in floats: feature weight [16][3][3] and bias, head weight [16]
//   and bias, the conv biases.
constexpr int RF2_T = 110, RF2_ROWS = 16;
constexpr int RF2_FRAG1 = 0, RF2_FRAG2 = RF2_FRAG1 + 9 * 2 * 256, RF2_FRAG3 = RF2_FRAG2 + 9 * 4 * 256, RF2_FRAG4 = RF2_FRAG3 + 18 * 4 * 256;
constexpr int RF2_F32 = RF2_FRAG4 + 18 * 256;
constexpr int RF2_FW = 0, RF2_FB = 144, RF2_HW = 160, RF2_B1 = 176, RF2_B2 = 192, RF2_B3 = 224, RF2_HB = 256, RF2_B4 = 257;
constexpr int RF2_PARAM_BYTES = RF2_F32 + 264 * 4;
// x fp32 [B][3][h][w] -> delta fp32 [B][1][h][w] (fp16 values)
int rf2_forward(cudaStream_t st, const void* params, const float* x, int B, int h, int w, float* delta);

}  // namespace nb200
