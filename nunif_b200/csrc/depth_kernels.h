// Kernels of the Depth-Anything-V2 path that are not GEMMs (depth_kernels.cu); model wiring in depth_model.cu.
#pragma once
#include "common.cuh"

namespace nb200 {

// x fp32 [B][3][H][W] (normalised) -> A fp16 [B*ph*pw][kpad], k = (c*14 + ky)*14 + kx (Conv2d weight order), zero padded
int da_patch_im2col(cudaStream_t st, const float* x, int B, int H, int W, __half* A, int kpad);
// X32[b][0] = cls + pos[0]; X32[b][1+n] = T[b*P+n] + pos[1+n]   (T fp16 = patch GEMM output incl. bias)
int da_assemble_tokens(cudaStream_t st, const __half* T, const float* cls, const float* pos, float* X32, int B, int P, int dim);
// X32 += delta (fp16, may be null); out = LayerNorm(X32) * w + b (eps 1e-6) as fp16.  rows x dim, dim in {256, 384, 768, 1024}
int da_add_layernorm(cudaStream_t st, float* X32, const __half* delta, const float* w, const float* b, __half* out, long long rows,
                     int dim);
// softmax(q k^T / sqrt(64)) v over all N tokens of each image; qkv [B*N][3*dim] (q | k | v, head-major 64-wide), out [B*N][dim]
// bias_log2e (optional): additive score bias [heads][N][ldb] fp32 already multiplied by log2(e), ldb >= cdiv(N,64)*64
int da_attention(cudaStream_t st, const __half* qkv, __half* out, int B, int N, int heads, const float* bias_log2e = nullptr, int ldb = 0);
// y = relu(x); if s: s = x0 + x   (NHWC fp16, n elements, n % 8 == 0)
int da_relu_add(cudaStream_t st, const __half* x, const __half* x0, __half* y, __half* s, long long n);
// bilinear, align_corners=True, NHWC fp16 [B][h][w][C] -> [B][H][W][C], C % 8 == 0
int da_upsample_bilinear(cudaStream_t st, const __half* x, int B, int h, int w, int C, __half* out, int H, int W);
// depth-to-space r=4: T [B*h*w][16*c] with n = (dy*4+dx)*c + co -> out [B][4h][4w][cpad] (channels >= c zeroed)
int da_depth_to_space4(cudaStream_t st, const __half* T, int B, int h, int w, int c, __half* out, int cpad);
// im2col for a 3x3 stride-2 pad-1 conv: x [B][h][w][C] -> A [B*ho*wo][9*C], k = (ky*3+kx)*C + c
int da_im2col_s2(cudaStream_t st, const __half* x, int B, int h, int w, int C, __half* A);
// depth[b][y][x] = relu(dot(wv[0..C), x[b][y][x][:]) + bias)   (conv1x1 C->1 + ReLU), fp32 out
int da_head_final(cudaStream_t st, const __half* x, long long npix, int C, const float* wv, float bias, float* depth);

}  // namespace nb200
