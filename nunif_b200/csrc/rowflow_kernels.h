// Non-GEMM kernels of the learned stereo warp sbs.row_flow_v3 (rowflow_kernels.cu); wiring in rowflow_model.inl.
#pragma once
#include "common.cuh"

namespace nb200 {

// x fp32 [B][3][h][w] -> tokens fp16 [B][Hp][Wt][32]: replicate-pad to (Hp, Wt*8), pixel_unshuffle (1, 8) (channel = c*8 + sw),
// channels 24..31 zero
int rf_prep(cudaStream_t st, const float* x, int B, int h, int w, int Hp, int Wt, __half* out);
// pixel_shuffle (1, 8) + crop to (h, w) + replication pad 1 + conv3x3 (8 -> 1): tokens [B][Hp][Wt][64] -> delta fp32 [B][1][h][w]
int rf_last_conv(cudaStream_t st, const __half* x, int B, int Hp, int Wt, int h, int w, const float* wt72, float bias, float* delta);

}  // namespace nb200
