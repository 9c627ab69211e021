// iw3's NULL depth model, the weight-free stand-in for stereo benchmarks (iw3/null_depth_model.py:17-21 NullDepth.forward):
// F.interpolate(x, (R, R), mode="bilinear") followed by x.mean(dim=1, keepdim=True), in one pass.  One thread per output
// pixel reads the four bilinear taps of the three channels, interpolates each channel and takes the channel mean in
// registers, so the 3 x R x R resized image never exists in memory.
//
// The arithmetic is ATen's two CUDA kernels, so the result equals torch's composition on the same GPU:
//   * upsample_bilinear2d_out_frame (UpSampleBilinear2d.cu) with align_corners=False and an output size: scale (float)in / R
//     computed on the host, bil_tap / bil_mix (common.cuh).  A frame that is already R x R is copied, not interpolated, as
//     there.
//   * the mean over dim 1 (mean_kernel_impl, ReduceMomentKernel.cu, through Reduce.cuh): one thread reduces the three
//     channels of its output into separate accumulators that start at 0 (the fourth of thread_reduce_impl's unrolled
//     accumulators stays 0), combines them left to right and multiplies by MeanOps' factor, (float)(B R R) / (float)(3 B R R).
#include "common.cuh"
#include "../../include/nunif_b200.h"
#include <climits>

namespace nb200 {

namespace {

constexpr int kThreads = 256;

__global__ void __launch_bounds__(kThreads) null_depth_kernel(const float* __restrict__ x, int H, int W, int R, float sy, float sx,
                                                              float factor, float* __restrict__ out) {
    const int i = blockIdx.x * kThreads + threadIdx.x, b = blockIdx.y;
    if (i >= R * R) return;
    const size_t plane = (size_t)H * W;
    const float* p = x + (size_t)b * 3 * plane;
    float v[3];
    if (H == R && W == R) {
#pragma unroll
        for (int c = 0; c < 3; ++c) v[c] = __ldg(p + c * plane + i);
    } else {
        const int oy = i / R, ox = i - oy * R;
        const BilTap ty = bil_tap(sy, oy, H), tx = bil_tap(sx, ox, W);
        const size_t r0 = (size_t)ty.i0 * W, r1 = (size_t)ty.i1 * W;
#pragma unroll
        for (int c = 0; c < 3; ++c) {
            const float* q = p + c * plane;
            v[c] = bil_mix(ty, tx, __ldg(q + r0 + tx.i0), __ldg(q + r0 + tx.i1), __ldg(q + r1 + tx.i0), __ldg(q + r1 + tx.i1));
        }
    }
    const float s = __fadd_rn(__fadd_rn(__fadd_rn(__fadd_rn(0.f, v[0]), __fadd_rn(0.f, v[1])), __fadd_rn(0.f, v[2])), 0.f);
    out[(size_t)b * R * R + i] = __fmul_rn(s, factor);
}

}  // namespace

}  // namespace nb200

using namespace nb200;

extern "C" int nb200_null_depth(const float* x, int B, int H, int W, int R, float* out, void* stream) {
    NB_CHECK(x && out, "null pointer");
    NB_CHECK(B > 0 && H > 0 && W > 0 && R > 0, "bad shape");
    NB_CHECK(B <= 65535, "B must be at most 65535");
    NB_CHECK((int64_t)R * R <= INT_MAX - kThreads, "R too large");
    NB_CHECK((const void*)x != (const void*)out, "out must not alias x");
    const int64_t n_out = (int64_t)B * R * R;
    const float factor = (float)n_out / (float)(3 * n_out);     // MeanOps factor: num_output_elements / numel in fp32
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope ps(st, PC_OTHER, (double)n_out * 13 * 4, (double)n_out * 12 * 4, (double)n_out * 4);
    null_depth_kernel<<<dim3(cdiv(R * R, kThreads), B), kThreads, 0, st>>>(x, H, W, R, (float)H / (float)R, (float)W / (float)R,
                                                                          factor, out);
    NB_LAUNCHED();
    return 0;
}
