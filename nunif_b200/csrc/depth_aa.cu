// Kernels of `iw3.depth_aa` (iw3/models/depth_aa.py:11-87), the learned anti-aliasing filter Depth-Anything's output goes
// through when `depth_aa=True` (iw3/depth_anything_model.py:153-154): its input and output stages.  The network works on a
// pixel_unshuffle(2) grid of 32-channel tokens with three 8x8 window-attention blocks (2 heads of 16; the first and the last
// shifted by zero padding), which run in window_mha.cu and on the wgmma GEMM; ~0.3 GFLOP per 392x686 map: latency kernels.
#include "depth_aa_kernels.h"

namespace nb200 {

namespace {

constexpr int C = 32;

__global__ void __launch_bounds__(1024) aa_minmax_kernel(const float* __restrict__ x, long long n, float* __restrict__ mm) {
    __shared__ float smn[32], smx[32];
    float mn = INFINITY, mx = -INFINITY;
    for (long long i = threadIdx.x; i < n; i += blockDim.x) {
        const float v = __ldg(x + i);
        mn = fminf(mn, v);
        mx = fmaxf(mx, v);
    }
    for (int o = 16; o; o >>= 1) {
        mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    }
    if ((threadIdx.x & 31) == 0) { smn[threadIdx.x >> 5] = mn; smx[threadIdx.x >> 5] = mx; }
    __syncthreads();
    if (threadIdx.x < 32) {
        mn = smn[threadIdx.x];
        mx = smx[threadIdx.x];
        for (int o = 16; o; o >>= 1) {
            mn = fminf(mn, __shfl_xor_sync(0xffffffffu, mn, o));
            mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
        }
        if (threadIdx.x == 0) { mm[0] = mn; mm[1] = mx; }
    }
}

// torch.nan_to_num of (v - mn) / (mx - mn)
__device__ __forceinline__ float aa_norm(float v, float mn, float scale) {
    float y = __fdiv_rn(__fsub_rn(v, mn), scale);
    if (isnan(y)) y = 0.f;
    else if (isinf(y)) y = y > 0.f ? 3.4028234663852886e38f : -3.4028234663852886e38f;
    return y;
}

__global__ void __launch_bounds__(256) aa_prep_kernel(const float* __restrict__ x, const float* __restrict__ mm, int B, int H, int W,
                                                       int ph1, int pw1, int Hh, int Wh, const float* __restrict__ w_in,
                                                       const float* __restrict__ b_in, __half* __restrict__ out) {
    __shared__ float sw[C * 4], sb[C];
    if (threadIdx.x == 0) NB_PDL_TRIGGER();
    if (threadIdx.x < C * 4) sw[threadIdx.x] = w_in[threadIdx.x];
    if (threadIdx.x < C) sb[threadIdx.x] = b_in[threadIdx.x];
    __syncthreads();
    const long long total = (long long)B * Hh * Wh;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int tx = (int)(i % Wh), ty = (int)((i / Wh) % Hh), b = (int)(i / ((long long)Wh * Hh));
    const bool norm = mm != nullptr;
    const float mn = norm ? mm[0] : 0.f, scale = norm ? __fsub_rn(mm[1], mm[0]) : 1.f;
    float v[4];
#pragma unroll
    for (int dy = 0; dy < 2; ++dy)
#pragma unroll
        for (int dx = 0; dx < 2; ++dx) {
            const int yy = min(max(2 * ty + dy - ph1, 0), H - 1), xx = min(max(2 * tx + dx - pw1, 0), W - 1);   // replication_pad2d_naive
            const float s = __ldg(x + ((size_t)b * H + yy) * W + xx);
            v[dy * 2 + dx] = norm ? aa_norm(s, mn, scale) : s;                                                  // pixel_unshuffle: c = dy * 2 + dx
        }
    __align__(16) __half2 o[C / 2];
#pragma unroll
    for (int n = 0; n < C; n += 2) {
        float a0 = sb[n], a1 = sb[n + 1];
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            a0 = fmaf(sw[n * 4 + c], v[c], a0);
            a1 = fmaf(sw[(n + 1) * 4 + c], v[c], a1);
        }
        o[n / 2] = __floats2half2_rn(a0, a1);
    }
    uint4* dst = reinterpret_cast<uint4*>(out + i * C);
#pragma unroll
    for (int k = 0; k < C / 8; ++k) dst[k] = reinterpret_cast<const uint4*>(o)[k];
}

__global__ void __launch_bounds__(256) aa_out_kernel(const __half* __restrict__ tok, const float* __restrict__ x, const float* __restrict__ mm,
                                                      int B, int H, int W, int ph1, int pw1, int Hh, int Wh, const float* __restrict__ w_out,
                                                      const float* __restrict__ b_out, int clamp, float* __restrict__ out) {
    __shared__ float sw[4 * C], sb[4];
    if (threadIdx.x < 4 * C) sw[threadIdx.x] = w_out[threadIdx.x];
    if (threadIdx.x < 4) sb[threadIdx.x] = b_out[threadIdx.x];
    __syncthreads();
    const long long total = (long long)B * H * W;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int X = (int)(i % W), Y = (int)((i / W) % H), b = (int)(i / ((long long)W * H));
    const int py = Y + ph1, px = X + pw1;                       // F.pad with negative padding = crop (depth_aa.py:77)
    const int sub = (py & 1) * 2 + (px & 1);                    // pixel_shuffle(2): channel dy * 2 + dx
    const __half* tp = tok + (((size_t)b * Hh + (py >> 1)) * Wh + (px >> 1)) * C;
    float acc = sb[sub];
#pragma unroll
    for (int v = 0; v < C / 8; ++v) {
        const uint4 raw = __ldg(reinterpret_cast<const uint4*>(tp) + v);
        const __half2* hh = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const float2 f = __half22float2(hh[k]);
            acc = fmaf(sw[sub * C + v * 8 + 2 * k], f.x, acc);
            acc = fmaf(sw[sub * C + v * 8 + 2 * k + 1], f.y, acc);
        }
    }
    const float s = __ldg(x + i);
    float r;
    if (mm) {
        const float mn = mm[0], scale = __fsub_rn(mm[1], mm[0]);
        r = __fadd_rn(__fmul_rn(__fadd_rn(aa_norm(s, mn, scale), acc), scale), mn);      // infer: (src + f(src)) * scale + min
    } else {
        r = s + acc;
        if (clamp) r = fminf(fmaxf(r, 0.f), 1.f);
    }
    out[i] = r;
}

}  // namespace

int aa_minmax(cudaStream_t st, const float* x, long long n, float* mm) {
    if (rec_on(REC_STEREO)) rec_launch("aaminmax", {{"n", n}});
    aa_minmax_kernel<<<1, 1024, 0, st>>>(x, n, mm);
    NB_LAUNCHED();
    return 0;
}
int aa_prep(cudaStream_t st, const float* x, const float* mm, int B, int H, int W, int ph1, int pw1, int Hh, int Wh, const float* w_in,
            const float* b_in, __half* out) {
    if (rec_on(REC_STEREO))
        rec_launch("aaprep", {{"B", B}, {"H", H}, {"W", W}, {"ph1", ph1}, {"pw1", pw1}, {"Hh", Hh}, {"Wh", Wh}, {"norm", mm ? 1 : 0}});
    const long long total = (long long)B * Hh * Wh;
    aa_prep_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(x, mm, B, H, W, ph1, pw1, Hh, Wh, w_in, b_in, out);
    NB_LAUNCHED();
    return 0;
}
int aa_out(cudaStream_t st, const __half* tok, const float* x, const float* mm, int B, int H, int W, int ph1, int pw1, int Hh, int Wh,
           const float* w_out, const float* b_out, int clamp, float* out) {
    if (rec_on(REC_STEREO))
        rec_launch("aaout", {{"B", B}, {"H", H}, {"W", W}, {"ph1", ph1}, {"pw1", pw1}, {"Hh", Hh}, {"Wh", Wh}, {"norm", mm ? 1 : 0},
                             {"clamp", clamp}});
    const long long total = (long long)B * H * W;
    aa_out_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(tok, x, mm, B, H, W, ph1, pw1, Hh, Wh, w_out, b_out, clamp, out);
    NB_LAUNCHED();
    return 0;
}

}  // namespace nb200
