// ATen's antialiased bilinear resize (_upsample_bilinear2d_aa, aten/src/ATen/native/cpu/UpSampleKernel.cpp) on the
// device: the taps and weights of one output index along one axis, and the separable sample (horizontal pass over each
// source row, then the vertical pass, in fp32).  align_corners only changes the scale the caller passes:
// (in - 1) / (out - 1) for True, in / out for False.  Shared by nb200_depth_resize_aa and the forward warp
// (warp_forward.cu), nb200_resize_bilinear_aa and the depth-model preprocess (frame_ops.cu), and the depth export
// (depth_io.cu).
#pragma once
#include "common.cuh"

namespace nb200 {

__device__ __forceinline__ float aa_tri(float x) {
    x = fabsf(x);
    return x < 1.f ? 1.f - x : 0.f;
}

// The source taps [min, min + size) of one output index, around centre = scale * (i + 0.5) with support max(scale, 1).
// Tap j weighs aa_tri((j + min - centre + 0.5) * inv), inv = 1 / scale when downsampling, else 1, before the weights
// are divided by their sum.
struct AaTaps {
    int min, size;
    float center, inv;
};

__device__ __forceinline__ AaTaps aa_taps(float scale, int i, int in_size) {
    const float support = scale >= 1.f ? scale : 1.f;
    AaTaps t;
    t.inv = scale >= 1.f ? 1.f / scale : 1.f;
    // the centre is a rounded fp32 product in ATen; without _rn nvcc fuses it into the tap offset of aa_weight (fma),
    // which shifts every weight by up to 1e-5
    t.center = __fmul_rn(scale, (float)i + 0.5f);
    t.min = max((int)(t.center - support + 0.5f), 0);
    t.size = min((int)(t.center + support + 0.5f), in_size) - t.min;
    return t;
}

__device__ __forceinline__ float aa_weight(const AaTaps& t, int j) {
    return aa_tri(((float)(j + t.min) - t.center + 0.5f) * t.inv);
}

__device__ __forceinline__ float aa_weight_sum(const AaTaps& t) {
    float s = 0.f;
    for (int j = 0; j < t.size; ++j) s += aa_weight(t, j);
    return s;
}

// One output sample.  load(y, x) returns source pixel (y, x); sum_y / sum_x are aa_weight_sum of ty / tx.
template <class Load>
__device__ __forceinline__ float aa_sample(const AaTaps& ty, const AaTaps& tx, float sum_y, float sum_x, Load load) {
    float acc = 0.f;
    for (int i = 0; i < ty.size; ++i) {
        float hs = 0.f;
        for (int j = 0; j < tx.size; ++j) hs += load(ty.min + i, tx.min + j) * (aa_weight(tx, j) / sum_x);
        acc += hs * (aa_weight(ty, i) / sum_y);
    }
    return acc;
}

}  // namespace nb200
