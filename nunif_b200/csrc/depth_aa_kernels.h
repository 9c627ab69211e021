// Non-GEMM kernels of the learned depth anti-aliasing filter iw3.depth_aa (depth_aa.cu); wiring in depth_aa_model.cu.
#pragma once
#include "common.cuh"

namespace nb200 {

// whole-tensor min / max of n floats -> mm[0], mm[1] (DepthAA.infer, iw3/models/depth_aa.py:49)
int aa_minmax(cudaStream_t st, const float* x, long long n, float* mm);
// replicate-pad (ph1, pw1 leading) + optional (x - min) / (max - min) with nan_to_num + pixel_unshuffle(2) + proj_in (1x1 conv 4 -> 32):
// x fp32 [B][1][H][W] -> tokens fp16 [B][Hh][Wh][32]
int aa_prep(cudaStream_t st, const float* x, const float* mm, int B, int H, int W, int ph1, int pw1, int Hh, int Wh, const float* w_in,
            const float* b_in, __half* out);
// proj_out (1x1 conv 32 -> 4) + pixel_shuffle(2) + crop + residual (+ clamp, or de-normalisation by mm): -> fp32 [B][1][H][W]
int aa_out(cudaStream_t st, const __half* tok, const float* x, const float* mm, int B, int H, int W, int ph1, int pw1, int Hh, int Wh,
           const float* w_out, const float* b_out, int clamp, float* out);

}  // namespace nb200
