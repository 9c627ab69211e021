// Kernels of `sbs.mlbw` (iw3/models/mlbw.py:36-127), the multi-layer learned stereo warp (methods mlbw_l2 / mlbw_l4 [s]): its input
// and output stages.  Like row_flow_v3 the network works on a (1, 8) pixel-unshuffled token grid, through window-attention
// blocks (window_mha.cu and the wgmma GEMM); it predicts L horizontal flow layers and L blending weights per pixel.
#include "mlbw_kernels.h"

namespace nb200 {

namespace {

__global__ void __launch_bounds__(256) mlbw_prep_kernel(const float* __restrict__ x, __half* __restrict__ out, int B, int H, int W, int ph1,
                                                         int pw1, int Hp, int Wt, int C1, const float* __restrict__ w_in,
                                                         const float* __restrict__ b_in) {
    extern __shared__ float sw[];            // [C1][3][9] + [C1]
    if (threadIdx.x == 0) NB_PDL_TRIGGER();
    for (int i = threadIdx.x; i < C1 * 27; i += blockDim.x) sw[i] = w_in[i];
    for (int i = threadIdx.x; i < C1; i += blockDim.x) sw[C1 * 27 + i] = b_in[i];
    __syncthreads();
    const long long total = (long long)B * Hp * Wt * C1;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c = (int)(i % C1);
    long long t = i / C1;
    const int xt = (int)(t % Wt);
    t /= Wt;
    const int y = (int)(t % Hp), b = (int)(t / Hp);
    const int sy = min(max(y - ph1, 0), H - 1);                       // replication_pad2d (pw1, pw2, ph1, ph2)
    float acc[8];
#pragma unroll
    for (int s = 0; s < 8; ++s) acc[s] = sw[C1 * 27 + c];
#pragma unroll
    for (int ci = 0; ci < 3; ++ci) {
        const float* row = x + (((size_t)b * 3 + ci) * H + sy) * W;
        float v[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) v[k] = __ldg(row + min(max(xt * 8 + k - 4 - pw1, 0), W - 1));    // both pads are replications: one clamp
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const float wv = sw[(c * 3 + ci) * 9 + tap];
#pragma unroll
            for (int s = 0; s < 8; ++s) acc[s] = fmaf(wv, v[s + tap], acc[s]);
        }
    }
    __align__(16) __half2 o[4];
#pragma unroll
    for (int s = 0; s < 4; ++s) {
        const float a0 = acc[2 * s] > 0.f ? acc[2 * s] : 0.2f * acc[2 * s], a1 = acc[2 * s + 1] > 0.f ? acc[2 * s + 1] : 0.2f * acc[2 * s + 1];
        o[s] = __floats2half2_rn(a0, a1);
    }
    *reinterpret_cast<uint4*>(out + (((size_t)b * Hp + y) * Wt + xt) * (8 * C1) + c * 8) = *reinterpret_cast<const uint4*>(o);
}

template <int L>
__global__ void __launch_bounds__(256) mlbw_out_kernel(const __half* __restrict__ t, const __half* __restrict__ t0, int B, int H, int W, int ph1,
                                                        int pw1, int Hp, int Wt, int C1, const float* __restrict__ w_out,
                                                        const float* __restrict__ b_out, float* __restrict__ delta, float* __restrict__ lw) {
    extern __shared__ float sw[];            // [2L][C1][9] + [2L]
    for (int i = threadIdx.x; i < 2 * L * C1 * 9 + 2 * L; i += blockDim.x) sw[i] = i < 2 * L * C1 * 9 ? w_out[i] : b_out[i - 2 * L * C1 * 9];
    __syncthreads();
    const long long total = (long long)B * H * W;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int X = (int)(i % W), Y = (int)((i / W) % H), b = (int)(i / ((long long)W * H));
    const int py = Y + ph1, px = X + pw1, Wp = Wt * 8;               // F.pad with negative padding = crop
    float acc[2 * L];
#pragma unroll
    for (int o = 0; o < 2 * L; ++o) acc[o] = sw[2 * L * C1 * 9 + o];
    const size_t rowtok = ((size_t)b * Hp + py) * Wt;
#pragma unroll 1
    for (int tap = 0; tap < 9; ++tap) {
        const int qx = min(max(px + tap - 4, 0), Wp - 1);              // ReplicationPad2d (4, 4, 0, 0)
        const size_t base = (rowtok + (qx >> 3)) * (size_t)(8 * C1) + (qx & 7);
        for (int c = 0; c < C1; ++c) {
            // pixel_shuffle (1, 8): S[c][y][x] = token(y, x / 8)[c * 8 + x % 8]; x + x1 is rounded to fp16 like the reference's tensor
            const float v = __half2float(__float2half_rn(__half2float(t[base + c * 8]) + __half2float(t0[base + c * 8])));
#pragma unroll
            for (int o = 0; o < 2 * L; ++o) acc[o] = fmaf(sw[(o * C1 + c) * 9 + tap], v, acc[o]);
        }
    }
    float lg[L], mx = -1e30f;
#pragma unroll
    for (int l = 0; l < L; ++l) {
        delta[((size_t)b * L + l) * H * W + (size_t)Y * W + X] = __half2float(__float2half_rn(acc[l]));   // conv output is fp16 under autocast
        lg[l] = __half2float(__float2half_rn(acc[L + l]));
        mx = fmaxf(mx, lg[l]);
    }
    float sum = 0.f;
#pragma unroll
    for (int l = 0; l < L; ++l) { lg[l] = __expf(lg[l] - mx); sum += lg[l]; }
    const float inv = 1.f / sum;
#pragma unroll
    for (int l = 0; l < L; ++l) lw[((size_t)b * L + l) * H * W + (size_t)Y * W + X] = lg[l] * inv;
}

}  // namespace

int mlbw_prep(cudaStream_t st, const float* x, int B, int H, int W, int ph1, int pw1, int Hp, int Wt, int C1, const float* w_in,
              const float* b_in, __half* out) {
    const long long total = (long long)B * Hp * Wt * C1;
    mlbw_prep_kernel<<<(unsigned)cdiv64(total, 256), 256, (size_t)(C1 * 28) * 4, st>>>(x, out, B, H, W, ph1, pw1, Hp, Wt, C1, w_in, b_in);
    NB_LAUNCHED();
    return 0;
}

int mlbw_out(cudaStream_t st, const __half* t, const __half* t0, int B, int H, int W, int ph1, int pw1, int Hp, int Wt, int C1, int L,
             const float* w_out, const float* b_out, float* delta, float* lw) {
    const long long total = (long long)B * H * W;
    const size_t smem = (size_t)(2 * L * C1 * 9 + 2 * L) * 4;
    if (L == 2) mlbw_out_kernel<2><<<(unsigned)cdiv64(total, 256), 256, smem, st>>>(t, t0, B, H, W, ph1, pw1, Hp, Wt, C1, w_out, b_out, delta, lw);
    else if (L == 4) mlbw_out_kernel<4><<<(unsigned)cdiv64(total, 256), 256, smem, st>>>(t, t0, B, H, W, ph1, pw1, Hp, Wt, C1, w_out, b_out, delta, lw);
    else return fail("mlbw_out: num_layers must be 2 or 4");
    NB_LAUNCHED();
    return 0;
}

}  // namespace nb200
