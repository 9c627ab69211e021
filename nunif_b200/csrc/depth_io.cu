// Depth export and import of iw3 (--export, --export-disparity, --export-depth-fit, an iw3_export.yml input):
//   * export: iw3/utils.py:1323-1328 (images) / :1378-1382 (video) then BaseDepthModel.save_normalized_depth
//     (iw3/base_depth_model.py:203-204): the optional disparity mapper, the optional antialiased bilinear fit to the
//     frame size, clamp(0, 1) and (0xffff * d).to(torch.uint16) - one kernel that writes the 16-bit map the host encodes;
//   * import: BaseDepthModel.load_depth (:225-232) on what TF.pil_to_tensor gives for a depth image (uint16 or int32 or
//     float32 with one channel, or uint8 with 1..4 channels), read interleaved as the decoder leaves it.
// The mapper runs on the source pixels, before the resize, as in the reference: it is evaluated per tap of the resize,
// which needs no workspace.  Measured against a separate source pass (profiles/bench_depth_export.py, H100 80GB HBM3,
// 700 W, ms per frame including the copy of the map to the host): div_6 is equal within the spread either way; the
// softplus blend mul_1+mul_2=0.5 costs 0.06-0.2 ms more fused (1080p fit 0.66 vs 0.66, 1080p from a 2x source 0.84 vs
// 0.76, 4K fit 2.38 vs 2.26, 4K from a 2x source 3.05 vs 2.86), against 2.3-3.1 ms for the whole 4K export.
#include "common.cuh"
#include "aa_resize.cuh"
#include "mapper.cuh"
#include "../../include/nunif_b200.h"

namespace nb200 {

// clamp, one fp32 multiply (not contracted into anything), truncation toward zero like torch's float -> uint16 cast
__device__ __forceinline__ uint16_t depth_to_u16(float d) {
    return (uint16_t)__fmul_rn(65535.f, clamp01(d));
}

__global__ void __launch_bounds__(128) depth_export_u16_kernel(const float* __restrict__ depth, int h, int w, int H, int W,
                                                               const nb200_mapper mapper, int fit, float scale_y,
                                                               float scale_x, uint16_t* __restrict__ out) {
    const int X = blockIdx.x * blockDim.x + threadIdx.x, y = blockIdx.y, b = blockIdx.z;
    if (X >= W) return;
    const float* src = depth + (size_t)b * h * w;
    float d;
    if (fit) {
        const AaTaps ty = aa_taps(scale_y, y, h), tx = aa_taps(scale_x, X, w);
        d = aa_sample(ty, tx, aa_weight_sum(ty), aa_weight_sum(tx),
                      [&](int yy, int xx) { return mapper_eval(mapper, __ldg(src + (size_t)yy * w + xx)); });
    } else {
        d = mapper_eval(mapper, __ldg(src + (size_t)y * w + X));
    }
    out[((size_t)b * H + y) * W + X] = depth_to_u16(d);
}

// integer maps are divided by 0xffff (8-bit maps too) and clamped; float maps are already depth
template <typename T>
__device__ __forceinline__ float import_channel(T v) {
    return clamp01(__fdiv_rn((float)v, 65535.f));
}
template <>
__device__ __forceinline__ float import_channel<float>(float v) {
    return v;
}

// One pixel of C interleaved channels: each converted by import_channel, then the channel mean
// (alpha included) as torch.mean evaluates it on the CPU - the sum in channel order, then one division - and the
// min/max rescale d * (hi - lo) + lo as two rounded ops.
template <typename T>
__global__ void __launch_bounds__(256) depth_import_kernel(const T* __restrict__ src, int C, size_t n, float range, float lo,
                                                           int has_range, float* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= n) return;
    const T* s = src + i * C;
    float d = import_channel(s[0]);
    if (C > 1) {
        for (int c = 1; c < C; ++c) d = __fadd_rn(d, import_channel(s[c]));
        d = __fdiv_rn(d, (float)C);
    }
    if (has_range) d = __fadd_rn(__fmul_rn(d, range), lo);
    out[i] = d;
}

}  // namespace nb200

using namespace nb200;

extern "C" int nb200_depth_export_u16(const float* depth, int B, int h, int w, const nb200_mapper* mapper_host, int fit,
                                      int H, int W, int align_corners, uint16_t* out, void* stream) {
    NB_CHECK(depth && out, "null pointer");
    NB_CHECK(B > 0 && B <= 65535 && h > 0 && w > 0, "bad shape");
    nb200_mapper mapper = {};
    if (mapper_host) {
        NB_CHECK(!*mapper_invalid(*mapper_host), mapper_invalid(*mapper_host));
        mapper = *mapper_host;
    }
    float sy = 0.f, sx = 0.f;
    if (fit) {
        NB_CHECK(H > 0 && H <= 65535 && W > 0, "bad fit size");
        // area_pixel_compute_scale: (in - 1) / (out - 1) with align_corners (F.interpolate, images), in / out without
        // (TF.resize, video)
        if (align_corners) {
            sy = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f;
            sx = W > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
        } else {
            sy = (float)h / (float)H;
            sx = (float)w / (float)W;
        }
    } else {
        NB_CHECK(h <= 65535, "bad shape");
        H = h;
        W = w;
    }
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope ps(st, PC_OTHER, (double)B * h * w * 4 + (double)B * H * W * 2);
    depth_export_u16_kernel<<<dim3(cdiv(W, 128), H, B), 128, 0, st>>>(depth, h, w, H, W, mapper, fit ? 1 : 0, sy, sx, out);
    NB_LAUNCHED();
    return 0;
}

extern "C" int nb200_depth_import(const void* src, int dtype, int C, int B, int H, int W, double lo, double hi, int has_range,
                                  float* out, void* stream) {
    NB_CHECK(src && out, "null pointer");
    NB_CHECK(dtype >= NB200_DEPTH_U8 && dtype <= NB200_DEPTH_F32, "unknown dtype");
    NB_CHECK(dtype == NB200_DEPTH_U8 ? C >= 1 && C <= 4 : C == 1, "expected uint8 with 1..4 channels, or one channel");
    NB_CHECK(B > 0 && H > 0 && W > 0, "bad shape");
    const size_t n = (size_t)B * H * W;
    // Python's max - min is a double; torch rounds the scalar to fp32 for the fp32 tensor
    const float range = (float)(hi - lo), lo32 = (float)lo;
    const int elem = dtype == NB200_DEPTH_U8 ? 1 : dtype == NB200_DEPTH_U16 ? 2 : 4;
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope ps(st, PC_OTHER, (double)n * (C * elem + 4));
    const unsigned blocks = (unsigned)cdiv64((int64_t)n, 256);
    switch (dtype) {
    case NB200_DEPTH_U8: depth_import_kernel<uint8_t><<<blocks, 256, 0, st>>>((const uint8_t*)src, C, n, range, lo32, has_range, out); break;
    case NB200_DEPTH_U16: depth_import_kernel<uint16_t><<<blocks, 256, 0, st>>>((const uint16_t*)src, C, n, range, lo32, has_range, out); break;
    case NB200_DEPTH_I32: depth_import_kernel<int32_t><<<blocks, 256, 0, st>>>((const int32_t*)src, C, n, range, lo32, has_range, out); break;
    default: depth_import_kernel<float><<<blocks, 256, 0, st>>>((const float*)src, C, n, range, lo32, has_range, out); break;
    }
    NB_LAUNCHED();
    return 0;
}
