// TransNetV2 (nunif/utils/transnetv2.py), the shot-boundary network of iw3's --scene-detect.  Packed by transnet_model.cu,
// small kernels in transnet.cu; every convolution runs on the wgmma implicit GEMM (gemm.h: CG_CONV3 and CG_TCONV3).
#pragma once
#include "common.cuh"

namespace nb200 {

constexpr int TN_H = 27, TN_W = 48;   // the network's input frame size
constexpr int TN_CIN = 32;            // input channels padded for the GEMM (K per tap must be a multiple of 32)
constexpr int TN_FEAT = 448;          // 64 + 128 + 256 channel means of the three stack outputs (FrameSimilarity input)
constexpr int TN_BAND = 101;          // lookup_window of FrameSimilarity / ColorHistograms
constexpr int TN_SIM = 128;           // similarity_dim / output_dim of both similarity branches
constexpr int TN_ROW = 4864;          // fc1 input: [histogram 128 | frame similarity 128 | stack-3 output 3 x 6 x 256]
constexpr int TN_HIDDEN = 1024;

struct TnBlock {
    size_t sw = 0;               // fp16 [8F][9][cin]: the four (1,3,3) convs of the block stacked along N, K = (ky, kx, c)
    size_t tw[4] = {}, tb[4] = {};   // per branch d = 1, 2, 4, 8: fp16 [F][3][2F] with the BatchNorm folded in, fp32 bias [F]
    int cin = 0, F = 0;
};

struct TnW {
    TnBlock blk[3][2];
    size_t proj_w = 0, proj_b = 0;     // fp32 frame_sim_layer.projection [128][448], [128]
    size_t sim_w = 0, sim_b = 0;       // fp32 frame_sim_layer.fc [128][101], [128]
    size_t hist_w = 0, hist_b = 0;     // fp32 color_hist_layer.fc [128][101], [128]
    size_t fc1_w = 0, fc1_b = 0;       // fp16 [1024][4864], fp32 [1024]
    size_t cls = 0;                    // fp32 cls_layer1.weight [1024], cls_layer2.weight [1024], the two biases
};

// x [n][3][27][48] fp32 -> x16 [n][27][48][32] fp16 (channels 3..31 zero)
int tn_prep(cudaStream_t st, const float* x, int n, __half* x16);
// relu(y2) + y1, AvgPool (1,2,2) with floor: y1, y2 [n][H][W][C] -> out frame f at out + f * out_stride, [H/2][W/2][C];
// the spatial mean of each pooled channel (fp32) goes to mean[f * TN_FEAT + mean_off + c]
int tn_stack_tail(cudaStream_t st, const __half* y1, const __half* y2, int n, int H, int W, int C, __half* out, long long out_stride,
                  float* mean, int mean_off);
// exact 512-bin colour histograms of x [n][3][27][48]: counts [n][512] int32
int tn_hist(cudaStream_t st, const float* x, int n, int* counts);
// L2-normalised projection of the channel means: emb [n][128] fp32
int tn_project(cudaStream_t st, const float* feat, int n, const float* w, const float* b, float* emb);
// both 101-wide similarity bands of every frame of B windows of T frames (bands [2][n][101]: histogram, frame similarity),
// each through its Linear(101 -> 128) + ReLU into columns [0, 128) / [128, 256) of row [n][4864]
int tn_bands(cudaStream_t st, const int* counts, const float* emb, int B, int T, const float* hist_w, const float* hist_b,
             const float* sim_w, const float* sim_b, float* bands, __half* row);
// cls_layer1 / cls_layer2 on hidden [n][1024] fp16 -> one_hot [n], many_hot [n] fp32
int tn_heads(cudaStream_t st, const __half* hidden, int n, const float* cls, float* one_hot, float* many_hot);

}  // namespace nb200
