// Non-GEMM kernels of the window-attention block WABlock (window_mha.cu) that sbs.row_flow_v3, sbs.mlbw and iw3.depth_aa share;
// wiring in wa_block.cu.
#pragma once
#include "common.cuh"

namespace nb200 {

// WindowMHA2d core (nunif/modules/attention.py:118-161) over ws x ws windows of the [B][H][W] token grid, `heads` heads of
// C / heads channels, additive (N x N) bias, N = ws * ws.  pad_y / pad_x = ws / 2 where the block is shifted in that direction: the grid
// is zero padded BEFORE the qkv projection, so padded tokens carry q | k | v = the projection bias, and the padding is cropped
// after the attention.  qkv fp16 [M][3C] (q | k | v), qkv_bias fp32 [3C] (not read without padding), out fp16 [M][C].
// Window / head layouts: 3x3 and 4x4 with 2 heads of 32, 4x4 with 4 heads of 32, 8x8 with 2 heads of 16.
int window_mha(cudaStream_t st, const __half* qkv, const float* qkv_bias, const float* bias, __half* out, int B, int H, int W, int C,
               int ws, int heads, int pad_y, int pad_x);
// replication pad 1 of a [B][H][W][C] fp16 tensor (C % 8 == 0)
int reppad1(cudaStream_t st, const __half* x, int B, int H, int W, int C, __half* out);

}  // namespace nb200
