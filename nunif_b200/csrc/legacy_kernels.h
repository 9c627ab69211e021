#pragma once
#include "common.cuh"

namespace nb200 {
// 3-channel output head of upconv_7 (mode 1: ConvTranspose 4x4 s2 p3, cin 256) / vgg_7 (mode 0: conv 3x3 valid, cin 128):
// x [n][Hi][Wi][cin] fp16 -> planar z [n][3][Ho][Wo] fp16 = clamp(conv + bias, 0, 1).  wt: packed by legacy_model.cu.
int head_conv(cudaStream_t st, int mode, int cin, const __half* x, const float* wt, const float* bias, __half* out, int n, int Hi,
              int Wi);
}  // namespace nb200
