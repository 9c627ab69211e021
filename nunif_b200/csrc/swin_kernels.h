#pragma once
#include "common.cuh"

namespace nb200 {
int stem_conv3x3(cudaStream_t st, const __half* x, const float* wt, const float* bias, __half* out, int n, int Hi, int Wi,
                 int cout_pad, int ldo);
constexpr int BIAS_FRAG_FLOATS = 6 * 3 * 6 * 32 * 4;  // per Swin block, see swin_attention_mma.cu
int build_bias_frag(cudaStream_t st, const float* table_121x6, float* frag);
// qkv: three dense planes q | k | v, each [B][H][W][C], `plane` elements apart
int window_attention(cudaStream_t st, const __half* qkv, const float* bias_frag, __half* out, int B, int H, int W, int C,
                     int shift, size_t plane);
// fused block head (swin_attention_mma.cu): att = window attention of x . Wqkv^T + bqkv (everything of
// shifted_window_attention but the proj Linear); Wqkv [3C][C] fp16 in the reference's row order, bias_frag from build_bias_frag
int swin_attn_fused(cudaStream_t st, const __half* x, const __half* wqkv, const float* bqkv, const float* bias_frag, __half* att,
                    int B, int H, int W, int C, int shift);
// fused block tail (swin_block.cu): x1 = x + att . Wp^T + bp (att == nullptr: x1 = x); x <- x1 + gelu(x1 W1^T + b1) W2^T + b2
// y != nullptr (needs att): x is not written; y [T][cs] = x . Wy^T + by instead (Wy [cs][C]; cs = 48 at C = 192, 16 at C = 96)
int swin_mlp_fused(cudaStream_t st, __half* x, const __half* att, long long T, int C, const __half* wp, const float* bp,
                   const __half* w1, const float* b1, const __half* w2, const float* b2, __half* y, int cs, const __half* wy,
                   const float* by);
// z: fp16 [n][3][S][S] for down == 1, fp32 for down in {2, 4}
int to_image(cudaStream_t st, const __half* y, void* z, int n, int Hs, int Ws, int cs, int r, int down);
}  // namespace nb200
