// Kernels of the ZoeD_N path that are neither GEMMs nor shared with Depth-Anything (zoe_kernels.cu); model wiring in
// zoe_model.inl.  Restated architecture + parity anchor: oracle/zoedepth.py.
#pragma once
#include "common.cuh"

namespace nb200 {

// x fp32 [B][3][H][W] (normalised) -> A fp16 [B*ph*pw][768], k = (c*16 + ky)*16 + kx (Conv2d weight order)
int zoe_patch_im2col(cudaStream_t st, const float* x, int B, int H, int W, __half* A);
// X32[b][0] = cls; X32[b][1+n] = T[b*P+n]   (BEiT has no absolute position table; T fp16 = patch GEMM output incl. bias)
int zoe_assemble_tokens(cudaStream_t st, const __half* T, const float* cls, float* X32, int B, int P, int dim);
// X32 += delta (may be null); out = fp16(X32)   (the forward-hook activations of blocks 5/11/17/23: no norm)
int zoe_add_cast(cudaStream_t st, float* X32, const __half* delta, __half* out, long long n);
// bias[h][q][k] (ld = ldb floats, pre-multiplied by log2 e) = table[index(q, k)][h] for a ph x pw token grid + class token;
// table fp32 [(2ph-1)(2pw-1) + 3][heads] (already resampled to this grid), MiDaS beit.py gen_relative_position_index
int zoe_expand_rel_bias(cudaStream_t st, const float* table, int ph, int pw, int heads, float* bias, int ldb);
// ProjectReadout input: A[b*P+n][0..dim) = F[b][1+n][:], A[..][dim..2dim) = F[b][0][:]    (F fp16 [B][1+P][dim])
int zoe_readout_concat(cudaStream_t st, const __half* F, int B, int P, int dim, __half* A);
// y = e + bilinear(align_corners=True)(prev [B][h][w][C] -> [B][H][W][C]), fp16 NHWC, C % 8 == 0
int zoe_add_upsampled(cudaStream_t st, const __half* e, const __half* prev, int B, int h, int w, int C, int H, int W, __half* y);
// out fp32 = softplus(x fp16), n elements  (SeedBinRegressorUnnormed: the seed bin centres)
int zoe_softplus(cudaStream_t st, const __half* x, float* out, long long n);
// AttractorLayerUnnormed: c = bilinear(align_corners)(prev_bin [B][h][w][64] fp32 -> H x W); a_j = softplus(apre[pix][j]), j < na
// (apre fp16, row stride lda); out[pix][k] = c_k + mean_j inv_attractor(a_j - c_k), inv_attractor(dx) = dx / (1 + 300 dx^2)
int zoe_attractor(cudaStream_t st, const __half* apre, int lda, int na, const float* prev_bin, int B, int h, int w, int H, int W,
                  float* out);
// SeedBinRegressor (normed, ZoeD_Any_K): s fp16 [npix][64] = ReLU'd seed logits -> out fp32 [npix][64] = the bin centres in
// [0, 1] units, (centres - min) / (max - min), centres = midpoints of the edges min + cumsum((max - min) * w / sum(w)), w = s + 1e-3
int zoe_seed_normed(cudaStream_t st, const __half* s, long long npix, float min_depth, float max_depth, float* out);
// AttractorLayer (normed): c = bilinear(align_corners)(prev_bin [B][h][w][64] -> H x W); a_j = apre[pix][2j] + 1e-3 (apre fp16 ReLU'd,
// row stride lda >= 2 na); out[pix][k] = c_k + mean_j inv_attractor(a_j - c_k).  sorted (may be null): (max - min) out + min, sorted
// ascending over the 64 bins and clipped to [min, max] (what the last level hands to the log-binomial mixture)
int zoe_attractor_normed(cudaStream_t st, const __half* apre, int lda, int na, const float* prev_bin, int B, int h, int w, int H, int W,
                         float min_depth, float max_depth, float* out, float* sorted);
// ConditionalLogBinomial input: A[pix][0..128) = bilinear(align_corners)(emb [B][h][w][128] -> H x W), [128..160) = act, [160] = rel,
// [161..192) = 0 (the packed weight uses the same channel order);  act fp16 [B][H][W][32], rel fp32 [B][H][W]
int zoe_clb_concat(cudaStream_t st, const __half* act, const float* rel, const __half* emb, int B, int h, int w, int H, int W, __half* A);
// g fp16 [pix][ldg >= 80] (GELU'd hidden) -> 4 outputs (w2 fp32 [4][80], b2 [4]) -> softplus -> p, temperature -> log-binomial
// softmax over 64 bins -> sum_k prob_k * bilinear(align_corners)(bins [B][h][w][64] fp32)_k -> depth fp32 [B][H][W]
int zoe_clb_final(cudaStream_t st, const __half* g, int ldg, const float* w2, const float* b2, const float* bins, int B, int h, int w, int H,
                  int W, float* depth);

}  // namespace nb200
