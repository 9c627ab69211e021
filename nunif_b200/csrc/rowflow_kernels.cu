// Kernels of `sbs.row_flow_v3` (iw3/models/row_flow_v3.py:14-68), the learned row-flow stereo warp that is iw3's CLI
// default method: everything except its Linears / 1x1 / 3x3 convs, which run on the wgmma GEMM.  The network works on
// a (1, 8) pixel-unshuffled grid of 64-channel tokens with two tiny window-attention blocks (4x4 and 3x3 windows,
// 2 heads of 32); per frame it is ~1 GFLOP, so these are bandwidth/latency kernels.
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

// One thread per (window, head, query); K and V of the window are staged in shared memory.
template <int WS>
__global__ void __launch_bounds__(128) rf_window_attention_kernel(const __half* __restrict__ qkv, const float* __restrict__ bias,
                                                                   __half* __restrict__ out, int Hp, int Wt, long long nwin) {
    constexpr int N = WS * WS, TPW = 2 * N, WPB = 128 / TPW;
    __shared__ __align__(16) __half sK[WPB][N][64];
    __shared__ __align__(16) __half sV[WPB][N][64];
    __shared__ float sBias[N * N];
    if (threadIdx.x == 0) NB_PDL_TRIGGER();
    for (int i = threadIdx.x; i < N * N; i += blockDim.x) sBias[i] = bias[i];
    const int wl = threadIdx.x / TPW, r = threadIdx.x % TPW;
    const long long win = (long long)blockIdx.x * WPB + wl;
    const bool active = wl < WPB && win < nwin;
    const int wpr = Wt / WS, wpc = Hp / WS;
    long long tok0 = 0;
    if (active) {
        const int wx = (int)(win % wpr), wy = (int)((win / wpr) % wpc), b = (int)(win / ((long long)wpr * wpc));
        tok0 = ((long long)b * Hp + wy * WS) * Wt + wx * WS;
        // stage K | V rows of this window: N tokens x 2 x 8 vectors of 16 B
        for (int i = r; i < N * 16; i += TPW) {
            const int j = i >> 4, v = i & 15;
            const long long tok = tok0 + (long long)(j / WS) * Wt + (j % WS);
            const uint4 val = __ldg(reinterpret_cast<const uint4*>(qkv + tok * 192 + 64) + v);
            if (v < 8) *reinterpret_cast<uint4*>(&sK[wl][j][v * 8]) = val;
            else *reinterpret_cast<uint4*>(&sV[wl][j][(v - 8) * 8]) = val;
        }
    }
    __syncthreads();
    if (!active) return;
    const int head = r / N, qi = r % N;
    const long long tokq = tok0 + (long long)(qi / WS) * Wt + (qi % WS);
    float q[32];
    {
        const uint4* qp = reinterpret_cast<const uint4*>(qkv + tokq * 192 + head * 32);
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            const uint4 raw = __ldg(qp + v);
            const __half2* hh = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float2 f = __half22float2(hh[k]);
                q[v * 8 + 2 * k] = f.x;
                q[v * 8 + 2 * k + 1] = f.y;
            }
        }
    }
    float s[N], mx = -1e30f;
#pragma unroll
    for (int j = 0; j < N; ++j) {
        const __half2* kp = reinterpret_cast<const __half2*>(&sK[wl][j][head * 32]);
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const float2 f = __half22float2(kp[k]);
            acc = fmaf(q[2 * k], f.x, acc);
            acc = fmaf(q[2 * k + 1], f.y, acc);
        }
        s[j] = acc * 0.17677669529663687f + sBias[qi * N + j];       // 1/sqrt(32); attn_mask is additive (F.scaled_dot_product_attention)
        mx = fmaxf(mx, s[j]);
    }
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < N; ++j) { s[j] = __expf(s[j] - mx); sum += s[j]; }
    const float inv = 1.f / sum;
    float o[32];
#pragma unroll
    for (int k = 0; k < 32; ++k) o[k] = 0.f;
#pragma unroll
    for (int j = 0; j < N; ++j) {
        const __half2* vp = reinterpret_cast<const __half2*>(&sV[wl][j][head * 32]);
        const float pj = s[j] * inv;
#pragma unroll
        for (int k = 0; k < 16; ++k) {
            const float2 f = __half22float2(vp[k]);
            o[2 * k] = fmaf(pj, f.x, o[2 * k]);
            o[2 * k + 1] = fmaf(pj, f.y, o[2 * k + 1]);
        }
    }
    __half* op = out + tokq * 64 + head * 32;
#pragma unroll
    for (int v = 0; v < 4; ++v) {
        __align__(16) __half2 hv[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) hv[k] = __floats2half2_rn(o[v * 8 + 2 * k], o[v * 8 + 2 * k + 1]);
        *reinterpret_cast<uint4*>(op + v * 8) = *reinterpret_cast<const uint4*>(hv);
    }
}

__global__ void __launch_bounds__(256) rf_reppad_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, int B, int H, int W) {
    if (threadIdx.x == 0) NB_PDL_TRIGGER();
    const long long total = (long long)B * (H + 2) * (W + 2) * 8;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int v = (int)(i & 7);
    long long t = i >> 3;
    const int X = (int)(t % (W + 2));
    t /= W + 2;
    const int Y = (int)(t % (H + 2)), b = (int)(t / (H + 2));
    const int sy = min(max(Y - 1, 0), H - 1), sx = min(max(X - 1, 0), W - 1);
    out[i] = __ldg(x + (((size_t)b * H + sy) * W + sx) * 8 + v);
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
    delta[i] = __half2float(__float2half_rn(acc));   // the reference's conv output is fp16 under autocast, then .float()
}

int rf_prep(cudaStream_t st, const float* x, int B, int h, int w, int Hp, int Wt, __half* out) {
    const long long total = (long long)B * Hp * Wt * 4;
    rf_prep_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(x, out, B, h, w, Hp, Wt);
    NB_LAUNCHED();
    return 0;
}

int rf_window_attention(cudaStream_t st, const __half* qkv, const float* bias, __half* out, int B, int Hp, int Wt, int ws) {
    NB_CHECK(Hp % ws == 0 && Wt % ws == 0, "token grid must be a multiple of the window");
    const long long nwin = (long long)B * (Hp / ws) * (Wt / ws);
    if (ws == 4) rf_window_attention_kernel<4><<<(unsigned)cdiv64(nwin, 4), 128, 0, st>>>(qkv, bias, out, Hp, Wt, nwin);
    else if (ws == 3) rf_window_attention_kernel<3><<<(unsigned)cdiv64(nwin, 7), 128, 0, st>>>(qkv, bias, out, Hp, Wt, nwin);
    else return fail("rf_window_attention: window must be 3 or 4");
    NB_LAUNCHED();
    return 0;
}

int rf_reppad(cudaStream_t st, const __half* x, int B, int H, int W, __half* out) {
    const long long total = (long long)B * (H + 2) * (W + 2) * 8;
    rf_reppad_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(out), B, H, W);
    NB_LAUNCHED();
    return 0;
}

int rf_last_conv(cudaStream_t st, const __half* x, int B, int Hp, int Wt, int h, int w, const float* wt72, float bias, float* delta) {
    const long long total = (long long)B * h * w;
    rf_last_conv_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(x, delta, B, Hp, Wt, h, w, wt72, bias);
    NB_LAUNCHED();
    return 0;
}

}  // namespace nb200
