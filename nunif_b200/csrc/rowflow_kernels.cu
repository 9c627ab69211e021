// Kernels of `sbs.row_flow_v3` (iw3/models/row_flow_v3.py:14-68), the learned row-flow stereo warp that is iw3's CLI
// default method: its input and output stages.  The network works on a (1, 8) pixel-unshuffled grid of 64-channel tokens
// with two tiny window-attention blocks (4x4 and 3x3 windows, 2 heads of 32), which run in window_mha.cu and on the wgmma
// GEMM; per frame it is ~1 GFLOP, so these are bandwidth/latency kernels.
#include "rowflow_kernels.h"

namespace nb200 {

__global__ void __launch_bounds__(256) rf_prep_kernel(const float* __restrict__ x, __half* __restrict__ out, int B, int h, int w,
                                                       int Hp, int Wt) {
    if (threadIdx.x == 0) NB_PDL_TRIGGER();
    const long long total = (long long)B * Hp * Wt * 4;       // 4 x 16-byte vectors per token (3 channels + zero pad)
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c = (int)(i & 3);
    long long t = i >> 2;
    const int xt = (int)(t % Wt);
    t /= Wt;
    const int y = (int)(t % Hp), b = (int)(t / Hp);
    __align__(16) __half v[8];
    if (c < 3) {
        const float* src = x + (((size_t)b * 3 + c) * h + min(y, h - 1)) * w;      // replication_pad2d_naive (0, pad1, 0, pad2)
#pragma unroll
        for (int s = 0; s < 8; ++s) v[s] = __float2half_rn(__ldg(src + min(xt * 8 + s, w - 1)));
    } else {
#pragma unroll
        for (int s = 0; s < 8; ++s) v[s] = __float2half_rn(0.f);
    }
    *reinterpret_cast<uint4*>(out + i * 8) = *reinterpret_cast<const uint4*>(v);
}

__global__ void __launch_bounds__(256) rf_last_conv_kernel(const __half* __restrict__ x, float* __restrict__ delta, int B, int Hp, int Wt,
                                                            int h, int w, const float* __restrict__ wt72, float bias) {
    __shared__ float sw[72];   // [oc][ky][kx]
    if (threadIdx.x < 72) sw[threadIdx.x] = wt72[threadIdx.x];
    __syncthreads();
    const long long total = (long long)B * h * w;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int X = (int)(i % w), Y = (int)((i / w) % h), b = (int)(i / ((long long)w * h));
    float acc = bias;
#pragma unroll
    for (int ky = 0; ky < 3; ++ky) {
        const int yy = min(max(Y + ky - 1, 0), h - 1);                       // crop to (h, w), then ReplicationPad2d(1)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
            const int xx = min(max(X + kx - 1, 0), w - 1);
            // pixel_shuffle (1, 8): S[oc][yy][xx] = token(yy, xx / 8)[oc * 8 + xx % 8]
            const __half* tp = x + (((size_t)b * Hp + yy) * Wt + (xx >> 3)) * 64 + (xx & 7);
#pragma unroll
            for (int oc = 0; oc < 8; ++oc) acc = fmaf(__half2float(tp[oc * 8]), sw[oc * 9 + ky * 3 + kx], acc);
        }
    }
    delta[i] = round_f16(acc);   // the reference's conv output is fp16 under autocast, then .float()
}

int rf_prep(cudaStream_t st, const float* x, int B, int h, int w, int Hp, int Wt, __half* out) {
    if (rec_on(REC_STEREO)) rec_launch("rfprep", {{"B", B}, {"h", h}, {"w", w}, {"Hp", Hp}, {"Wt", Wt}});
    const long long total = (long long)B * Hp * Wt * 4;
    rf_prep_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(x, out, B, h, w, Hp, Wt);
    NB_LAUNCHED();
    return 0;
}

int rf_last_conv(cudaStream_t st, const __half* x, int B, int Hp, int Wt, int h, int w, const float* wt72, float bias, float* delta) {
    if (rec_on(REC_STEREO)) rec_launch("rflast", {{"B", B}, {"Hp", Hp}, {"Wt", Wt}, {"h", h}, {"w", w}});
    const long long total = (long long)B * h * w;
    rf_last_conv_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(x, delta, B, Hp, Wt, h, w, wt72, bias);
    NB_LAUNCHED();
    return 0;
}

}  // namespace nb200
