// Kernels of `iw3.depth_aa` (iw3/models/depth_aa.py:11-87), the learned anti-aliasing filter Depth-Anything's output goes
// through when `depth_aa=True` (iw3/depth_anything_model.py:153-154): everything except its Linears / 1x1 / 3x3 convs, which run
// on the wgmma GEMM.  The network works on a pixel_unshuffle(2) grid of 32-channel tokens with three 8x8 window-attention
// blocks (2 heads of 16; the first and the last shifted by zero padding); ~0.3 GFLOP per 392x686 map: latency kernels.
#include "depth_aa_kernels.h"

namespace nb200 {

namespace {

constexpr int C = 32, WSZ = 8, NT = 64;

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

// One CTA per window, one thread per (head, query); K and V of the window staged in shared memory.
__global__ void __launch_bounds__(128) aa_window_attention_kernel(const __half* __restrict__ qkv, const float* __restrict__ qkv_bias,
                                                                   const float* __restrict__ bias, __half* __restrict__ out, int Hh, int Wh,
                                                                   int pad, int nwx, int nwy) {
    __shared__ __align__(16) __half sK[NT][C];
    __shared__ __align__(16) __half sV[NT][C];
    __shared__ float sBias[NT * NT];
    if (threadIdx.x == 0) NB_PDL_TRIGGER();
    for (int i = threadIdx.x; i < NT * NT; i += blockDim.x) sBias[i] = bias[i];
    const int wx = blockIdx.x % nwx, wy = (blockIdx.x / nwx) % nwy, b = blockIdx.x / (nwx * nwy);
    const int y0 = wy * WSZ - pad, x0 = wx * WSZ - pad;     // window origin in the un-padded token grid
    // stage K | V: 64 tokens x 2 x 4 vectors of 16 B; tokens of the zero padding carry the projection bias
    for (int i = threadIdx.x; i < NT * 8; i += blockDim.x) {
        const int j = i >> 3, v = i & 7;
        const int y = y0 + j / WSZ, x = x0 + j % WSZ;
        uint4 val;
        if (y >= 0 && y < Hh && x >= 0 && x < Wh) {
            val = __ldg(reinterpret_cast<const uint4*>(qkv + (((size_t)b * Hh + y) * Wh + x) * 96 + C) + v);
        } else {
            __align__(16) __half2 h[4];
#pragma unroll
            for (int k = 0; k < 4; ++k) h[k] = __floats2half2_rn(qkv_bias[C + v * 8 + 2 * k], qkv_bias[C + v * 8 + 2 * k + 1]);
            val = *reinterpret_cast<const uint4*>(h);
        }
        if (v < 4) *reinterpret_cast<uint4*>(&sK[j][v * 8]) = val;
        else *reinterpret_cast<uint4*>(&sV[j][(v - 4) * 8]) = val;
    }
    __syncthreads();
    const int head = threadIdx.x / NT, qi = threadIdx.x % NT;
    const int qy = y0 + qi / WSZ, qx = x0 + qi % WSZ;
    if (qy < 0 || qy >= Hh || qx < 0 || qx >= Wh) return;       // cropped away after the attention (attention.py:158-160)
    const size_t tokq = ((size_t)b * Hh + qy) * Wh + qx;
    float q[16];
    {
        const uint4* qp = reinterpret_cast<const uint4*>(qkv + tokq * 96 + head * 16);
#pragma unroll
        for (int v = 0; v < 2; ++v) {
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
    float s[NT], mx = -1e30f;
#pragma unroll
    for (int j = 0; j < NT; ++j) {
        const __half2* kp = reinterpret_cast<const __half2*>(&sK[j][head * 16]);
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float2 f = __half22float2(kp[k]);
            acc = fmaf(q[2 * k], f.x, acc);
            acc = fmaf(q[2 * k + 1], f.y, acc);
        }
        s[j] = acc * 0.25f + sBias[qi * NT + j];                 // 1/sqrt(16); attn_mask is additive (F.scaled_dot_product_attention)
        mx = fmaxf(mx, s[j]);
    }
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < NT; ++j) { s[j] = __expf(s[j] - mx); sum += s[j]; }
    const float inv = 1.f / sum;
    float o[16];
#pragma unroll
    for (int k = 0; k < 16; ++k) o[k] = 0.f;
#pragma unroll
    for (int j = 0; j < NT; ++j) {
        const __half2* vp = reinterpret_cast<const __half2*>(&sV[j][head * 16]);
        const float pj = s[j] * inv;
#pragma unroll
        for (int k = 0; k < 8; ++k) {
            const float2 f = __half22float2(vp[k]);
            o[2 * k] = fmaf(pj, f.x, o[2 * k]);
            o[2 * k + 1] = fmaf(pj, f.y, o[2 * k + 1]);
        }
    }
    __half* op = out + tokq * C + head * 16;
#pragma unroll
    for (int v = 0; v < 2; ++v) {
        __align__(16) __half2 hv[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) hv[k] = __floats2half2_rn(o[v * 8 + 2 * k], o[v * 8 + 2 * k + 1]);
        *reinterpret_cast<uint4*>(op + v * 8) = *reinterpret_cast<const uint4*>(hv);
    }
}

__global__ void __launch_bounds__(256) aa_reppad_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, int B, int H, int W, int V) {
    if (threadIdx.x == 0) NB_PDL_TRIGGER();
    const long long total = (long long)B * (H + 2) * (W + 2) * V;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int v = (int)(i % V);
    long long t = i / V;
    const int X = (int)(t % (W + 2));
    t /= W + 2;
    const int Y = (int)(t % (H + 2)), b = (int)(t / (H + 2));
    const int sy = min(max(Y - 1, 0), H - 1), sx = min(max(X - 1, 0), W - 1);
    out[i] = __ldg(x + (((size_t)b * H + sy) * W + sx) * V + v);
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
    aa_minmax_kernel<<<1, 1024, 0, st>>>(x, n, mm);
    NB_LAUNCHED();
    return 0;
}
int aa_prep(cudaStream_t st, const float* x, const float* mm, int B, int H, int W, int ph1, int pw1, int Hh, int Wh, const float* w_in,
            const float* b_in, __half* out) {
    const long long total = (long long)B * Hh * Wh;
    aa_prep_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(x, mm, B, H, W, ph1, pw1, Hh, Wh, w_in, b_in, out);
    NB_LAUNCHED();
    return 0;
}
int aa_window_attention(cudaStream_t st, const __half* qkv, const float* qkv_bias, const float* bias, __half* out, int B, int Hh, int Wh,
                        int shift) {
    NB_CHECK(Hh % WSZ == 0 && Wh % WSZ == 0, "token grid must be a multiple of the 8x8 window");
    const int pad = shift ? WSZ / 2 : 0;
    const int nwx = (Wh + 2 * pad) / WSZ, nwy = (Hh + 2 * pad) / WSZ;
    aa_window_attention_kernel<<<(unsigned)(B * nwx * nwy), 128, 0, st>>>(qkv, qkv_bias, bias, out, Hh, Wh, pad, nwx, nwy);
    NB_LAUNCHED();
    return 0;
}
int aa_reppad(cudaStream_t st, const __half* x, int B, int H, int W, int Cc, __half* out) {
    NB_CHECK(Cc % 8 == 0, "channels must be a multiple of 8");
    const long long total = (long long)B * (H + 2) * (W + 2) * (Cc / 8);
    aa_reppad_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(out), B, H, W,
                                                                   Cc / 8);
    NB_LAUNCHED();
    return 0;
}
int aa_out(cudaStream_t st, const __half* tok, const float* x, const float* mm, int B, int H, int W, int ph1, int pw1, int Hh, int Wh,
           const float* w_out, const float* b_out, int clamp, float* out) {
    const long long total = (long long)B * H * W;
    aa_out_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(tok, x, mm, B, H, W, ph1, pw1, Hh, Wh, w_out, b_out, clamp, out);
    NB_LAUNCHED();
    return 0;
}

}  // namespace nb200
