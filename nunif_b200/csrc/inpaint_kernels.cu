// iw3 forward_inpaint: the kernels of inpaint.light_inpaint_v1 (iw3/models/light_inpaint_v1.py) and its mask preparation
// (iw3/dilation.py, iw3/forward_inpaint.py:18-40) that are not convolutions.  The convolutions and Linears run on the wgmma
// implicit GEMM (gemm.cu); the sequence is in inpaint_model.cu.
#include "inpaint_kernels.h"
#include "ptx.cuh"
#include <cmath>

namespace nb200 {

extern int g_tune[16];  // gemm.cu; [7] != 0 selects the SIMT token-mixing kernel (tests)

// ---- mask preparation -----------------------------------------------------------------------------------------------------
__device__ __forceinline__ float mask_in(const float* m, size_t i, int binarize) {
    const float v = m[i];
    return binarize ? (v > 0.f ? 1.f : 0.f) : v;
}

// closing, first half: 2x max_pool2d(3, 1, 1) == the max over the 5x5 neighbourhood clipped to the image (the -inf padding
// never wins, and every in-image point of the 5x5 square is reachable through an in-image 3x3 step)
__global__ void __launch_bounds__(256) mask_dilate5_kernel(const float* __restrict__ m, int B, int H, int W, int binarize,
                                                           float* __restrict__ d) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)B * H * W) return;
    const int x = (int)(i % W), y = (int)((i / W) % H);
    const size_t base = i - (size_t)y * W - x;
    float v = -INFINITY;
    for (int yy = max(y - 2, 0); yy <= min(y + 2, H - 1); ++yy)
        for (int xx = max(x - 2, 0); xx <= min(x + 2, W - 1); ++xx) v = fmaxf(v, mask_in(m, base + (size_t)yy * W + xx, binarize));
    d[i] = v;
}

// one block per row: closing's 5x5 erosion + OR with the input (dilation.py:145-152) into shared memory, then the row runs
// of dilate_outer / dilate_inner (dilation.py:67-98): out[x] = any(c[x - n_left .. x + n_right] != 0)
__global__ void __launch_bounds__(256) mask_row_kernel(const float* __restrict__ m, const float* __restrict__ d, int H, int W,
                                                       int binarize, int closing, int n_left, int n_right, float* __restrict__ out) {
    extern __shared__ float row[];
    const int y = blockIdx.x % H;
    const size_t img = (size_t)(blockIdx.x / H) * H * W;
    for (int x = threadIdx.x; x < W; x += blockDim.x) {
        const float v0 = mask_in(m, img + (size_t)y * W + x, binarize);
        float c = v0;
        if (closing) {
            float e = INFINITY;
            for (int yy = max(y - 2, 0); yy <= min(y + 2, H - 1); ++yy)
                for (int xx = max(x - 2, 0); xx <= min(x + 2, W - 1); ++xx) e = fminf(e, d[img + (size_t)yy * W + xx]);
            c = fminf(fmaxf(e + v0, 0.f), 1.f);
        }
        row[x] = c;
    }
    __syncthreads();
    const bool dil = n_left > 0 || n_right > 0;
    for (int x = threadIdx.x; x < W; x += blockDim.x) {
        float v = row[x];
        if (dil) {
            bool any = false;
            for (int j = max(x - n_left, 0); j <= min(x + n_right, W - 1) && !any; ++j) any = row[j] != 0.f;
            v = any ? 1.f : 0.f;
        }
        out[img + (size_t)y * W + x] = v;
    }
}

int inpaint_mask(cudaStream_t st, const float* mask, int B, int H, int W, int binarize, int closing, int n_left, int n_right,
                 float* tmp, float* out) {
    const size_t n = (size_t)B * H * W;
    ProfScope ps(st, PC_DILATE, n * 8.0, n * 4.0, n * 4.0);
    if (closing) {
        mask_dilate5_kernel<<<(unsigned)cdiv64(n, 256), 256, 0, st>>>(mask, B, H, W, binarize, tmp);
        NB_LAUNCHED();
    }
    const size_t smem = (size_t)W * 4;
    if (ensure_dyn_smem((const void*)mask_row_kernel, smem)) return 1;
    mask_row_kernel<<<(unsigned)(B * H), 256, smem, st>>>(mask, tmp, H, W, binarize, closing, n_left, n_right, out);
    NB_LAUNCHED();
    return 0;
}

// SeparableGaussianFilter2d(1, 15, padding=7) (gaussian_filter.py:8-19,51-74): replicate padding, horizontal then vertical pass
struct Gauss15 { float w[15]; };

static Gauss15 gauss15() {
    // get_gaussian_kernel1d in fp32: linspace(-7, 7) / sigma, exp(-0.5 x^2), normalised by the sum
    Gauss15 k;
    const float sigma = (float)(15 * 0.15 + 0.35);
    float s = 0.f;
    for (int i = 0; i < 15; ++i) {
        const float x = (float)(i - 7) / sigma;
        k.w[i] = expf(-0.5f * (x * x));
        s += k.w[i];
    }
    for (int i = 0; i < 15; ++i) k.w[i] /= s;
    return k;
}

__global__ void __launch_bounds__(256) blur_h_kernel(const float* __restrict__ m, int B, int H, int W, int mirror, Gauss15 k,
                                                     float* __restrict__ t) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)B * H * W) return;
    const int x = (int)(i % W);   // network coordinates
    const size_t row = i - x;
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 15; ++j) {
        const int xx = min(max(x + j - 7, 0), W - 1);
        s = fmaf(k.w[j], m[row + (mirror ? W - 1 - xx : xx)], s);
    }
    t[i] = s;
}

__global__ void __launch_bounds__(256) blur_v_kernel(const float* __restrict__ t, const float* __restrict__ m, int B, int H, int W,
                                                     int mirror, Gauss15 k, float* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)B * H * W) return;
    const int x = (int)(i % W), y = (int)((i / W) % H);
    const size_t img = i - (size_t)y * W - x;
    float s = 0.f;
#pragma unroll
    for (int j = 0; j < 15; ++j) s = fmaf(k.w[j], t[img + (size_t)min(max(y + j - 7, 0), H - 1) * W + x], s);
    const float m0 = m[img + (size_t)y * W + (mirror ? W - 1 - x : x)];
    out[i] = fminf(fmaxf(s + m0, 0.f), 1.f);
}

int inpaint_blur(cudaStream_t st, const float* mask, int B, int H, int W, int mirror, float* tmp, float* out) {
    const size_t n = (size_t)B * H * W;
    ProfScope ps(st, PC_DILATE, n * 16.0, n * 8.0, n * 8.0);
    const Gauss15 k = gauss15();
    blur_h_kernel<<<(unsigned)cdiv64(n, 256), 256, 0, st>>>(mask, B, H, W, mirror, k, tmp);
    NB_LAUNCHED();
    blur_v_kernel<<<(unsigned)cdiv64(n, 256), 256, 0, st>>>(tmp, mask, B, H, W, mirror, k, out);
    NB_LAUNCHED();
    return 0;
}

// ---- stem (light_inpaint_v1.py:113-118, 132-146) ------------------------------------------------------------------------------
// one thread per /4 token; the 48 x 96 weights (fp16 precision, as the reference's autocast conv) are broadcast from smem
__global__ void __launch_bounds__(128) inpaint_stem_kernel(const float* __restrict__ x, const float* __restrict__ hole,
                                                           const float* __restrict__ blur, int B, int H, int W, int H4, int W4,
                                                           int mirror, const float* __restrict__ w, const float* __restrict__ b,
                                                           const float* __restrict__ mask_bias, __half* __restrict__ out) {
    __shared__ float sw[48 * 96];
    __shared__ float sb[96];
    for (int i = threadIdx.x; i < 48 * 96; i += blockDim.x) sw[i] = w[i];
    for (int i = threadIdx.x; i < 96; i += blockDim.x) sb[i] = b[i];
    __syncthreads();
    const size_t tok = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (tok >= (size_t)B * H4 * W4) return;
    const int tx = (int)(tok % W4), ty = (int)((tok / W4) % H4), bi = (int)(tok / ((size_t)W4 * H4));
    const size_t plane = (size_t)H * W;
    float in[48];
    float amax = 0.f;
#pragma unroll
    for (int dy = 0; dy < 4; ++dy)
#pragma unroll
        for (int dx = 0; dx < 4; ++dx) {
            const int yn = min(4 * ty + dy, H - 1), xn = min(4 * tx + dx, W - 1);   // replicate pad right / bottom
            const int xi = mirror ? W - 1 - xn : xn;
            const size_t p = (size_t)yn * W + xi;
            const float keep = 1.f - hole[bi * plane + p];
            amax = fmaxf(amax, blur[bi * plane + (size_t)yn * W + xn]);
#pragma unroll
            for (int c = 0; c < 3; ++c) {
                const float v = x[((size_t)bi * 3 + c) * plane + p] * keep;
                in[c * 16 + dy * 4 + dx] = round_f16((v - 0.5f) / 0.5f);
            }
        }
    uint4* dst = reinterpret_cast<uint4*>(out + tok * 96);
    if (amax > 0.99f) {
#pragma unroll 1
        for (int q = 0; q < 12; ++q) {
            __align__(16) __half h[8];
#pragma unroll
            for (int e = 0; e < 8; ++e) h[e] = __float2half_rn(mask_bias[q * 8 + e]);
            dst[q] = *reinterpret_cast<const uint4*>(h);
        }
        return;
    }
#pragma unroll 1
    for (int q = 0; q < 12; ++q) {
        float acc[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[e] = sb[q * 8 + e];
#pragma unroll
        for (int k = 0; k < 48; ++k) {
            const float4 w0 = *reinterpret_cast<const float4*>(&sw[k * 96 + q * 8]);
            const float4 w1 = *reinterpret_cast<const float4*>(&sw[k * 96 + q * 8 + 4]);
            acc[0] = fmaf(w0.x, in[k], acc[0]); acc[1] = fmaf(w0.y, in[k], acc[1]);
            acc[2] = fmaf(w0.z, in[k], acc[2]); acc[3] = fmaf(w0.w, in[k], acc[3]);
            acc[4] = fmaf(w1.x, in[k], acc[4]); acc[5] = fmaf(w1.y, in[k], acc[5]);
            acc[6] = fmaf(w1.z, in[k], acc[6]); acc[7] = fmaf(w1.w, in[k], acc[7]);
        }
        __align__(16) __half h[8];
#pragma unroll
        for (int e = 0; e < 8; ++e) h[e] = __float2half_rn(acc[e] >= 0.f ? acc[e] : 0.2f * acc[e]);
        dst[q] = *reinterpret_cast<const uint4*>(h);
    }
}

int inpaint_stem(cudaStream_t st, const float* x, const float* hole, const float* blur, int B, int H, int W, int Hp, int Wp,
                 int mirror, const float* w, const float* b, const float* mask_bias, __half* out) {
    const size_t tokens = (size_t)B * (Hp / 4) * (Wp / 4);
    ProfScope ps(st, PC_STEM, 2.0 * tokens * 48 * 96, (double)B * H * W * 20, tokens * 192.0);
    inpaint_stem_kernel<<<(unsigned)cdiv64(tokens, 128), 128, 0, st>>>(x, hole, blur, B, H, W, Hp / 4, Wp / 4, mirror, w, b,
                                                                        mask_bias, out);
    NB_LAUNCHED();
    return 0;
}

// ---- LN1 + zero ring + doubled shortcut ---------------------------------------------------------------------------------------
template <int C>
__global__ void __launch_bounds__(256) ln_pad_kernel(__half* __restrict__ x, const float* __restrict__ g, __half* __restrict__ t,
                                                     int B, int H, int W, int p) {
    constexpr int C2 = C / 2, PER = (C2 + 31) / 32;   // half2 per token, per lane (C = 96: 48 half2, lanes 0..15 take two)
    const int Hq = H + 2 * p, Wq = W + 2 * p;
    const size_t q = (size_t)blockIdx.x * 8 + (threadIdx.x >> 5);
    const int lane = threadIdx.x & 31;
    if (q >= (size_t)B * Hq * Wq) return;
    const int xq = (int)(q % Wq), yq = (int)((q / Wq) % Hq), bi = (int)(q / ((size_t)Wq * Hq));
    __half2* tq = reinterpret_cast<__half2*>(t + q * C);
    const int y = yq - p, xx = xq - p;
    if (y < 0 || y >= H || xx < 0 || xx >= W) {
#pragma unroll
        for (int i = 0; i < PER; ++i)
            if (lane + 32 * i < C2) tq[lane + 32 * i] = __floats2half2_rn(0.f, 0.f);
        return;
    }
    __half2* xp = reinterpret_cast<__half2*>(x + (((size_t)bi * H + y) * W + xx) * C);
    float2 v[PER];
    float s = 0.f;
#pragma unroll
    for (int i = 0; i < PER; ++i) {
        v[i] = lane + 32 * i < C2 ? __half22float2(xp[lane + 32 * i]) : make_float2(0.f, 0.f);
        s += v[i].x + v[i].y;
    }
    s = warp_sum(s);
    const float mean = s / C;
    float s2 = 0.f;
#pragma unroll
    for (int i = 0; i < PER; ++i) {
        if (lane + 32 * i >= C2) continue;
        const float a = v[i].x - mean, b = v[i].y - mean;
        s2 += a * a + b * b;
    }
    s2 = warp_sum(s2);
    const float rstd = rsqrtf(s2 / C + 1e-5f);
#pragma unroll
    for (int i = 0; i < PER; ++i) {
        if (lane + 32 * i >= C2) continue;
        const int c = 2 * (lane + 32 * i);
        tq[lane + 32 * i] = __floats2half2_rn((v[i].x - mean) * rstd * g[c], (v[i].y - mean) * rstd * g[c + 1]);
        xp[lane + 32 * i] = __floats2half2_rn(2.f * v[i].x, 2.f * v[i].y);
    }
}

int inpaint_ln_pad(cudaStream_t st, __half* x, const float* g, __half* t, int B, int H, int W, int C, int p) {
    const size_t n = (size_t)B * (H + 2 * p) * (W + 2 * p);
    ProfScope ps(st, PC_OTHER, (double)B * H * W * C * 6.0, (double)B * H * W * C * 2.0, (double)B * H * W * C * 2.0 + n * C * 2.0);
    const unsigned grid = (unsigned)cdiv64(n, 8);
    if (C == 96) ln_pad_kernel<96><<<grid, 256, 0, st>>>(x, g, t, B, H, W, p);
    else if (C == 192) ln_pad_kernel<192><<<grid, 256, 0, st>>>(x, g, t, B, H, W, p);
    else return fail("inpaint_ln_pad: C must be 96 or 192");
    NB_LAUNCHED();
    return 0;
}

// ---- token mixing (attention.py:643-660: LN2, proj_spatial, u * v) --------------------------------------------------------------
// One CTA per (window, 64 of the 2C channels), N / 32 warps.  LN2 statistics of the window's N tokens (over all 2C channels of v),
// then the normalised 64-channel slice of v goes to smem as the B operand [m][64] (16-byte chunks XOR-swizzled by row), and
// every warp computes 32 rows n of  Ws[n][:] . v[:][64]  with mma.sync m16n8k16 (Ws fragments straight from L2: the same
// N x N matrix serves every window).  The epilogue adds bs[n] and multiplies by u in place.
template <int N>
struct MixSmem {
    __half v[N * 64];
    float mean[N], rstd[N];
};

__device__ __forceinline__ size_t mix_pixel(int wi, int n, int ws, int Hq, int Wq) {
    const int nwx = Wq / ws, nwy = Hq / ws;
    const int bi = wi / (nwx * nwy), r = wi - bi * nwx * nwy;
    const int wy = r / nwx, wx = r - wy * nwx;
    return ((size_t)bi * Hq + wy * ws + n / ws) * Wq + wx * ws + n % ws;
}

template <int N>
__device__ __forceinline__ void mix_load(MixSmem<N>& s, const __half* __restrict__ u, int Hq, int Wq, int C, const float* __restrict__ g2) {
    constexpr int WS = N == 256 ? 16 : 8;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31, nw = N / 32;
    const int C4 = 4 * C, c0 = blockIdx.y * 64;
    for (int n = warp; n < N; n += nw) {
        const __half2* vp = reinterpret_cast<const __half2*>(u + mix_pixel(blockIdx.x, n, WS, Hq, Wq) * C4 + 2 * C);
        float sum = 0.f;
        for (int i = lane; i < C; i += 32) {   // 2C channels = C half2
            const float2 f = __half22float2(vp[i]);
            sum += f.x + f.y;
        }
        sum = warp_sum(sum);
        const float mean = sum / (2 * C);
        float s2 = 0.f;
        for (int i = lane; i < C; i += 32) {
            const float2 f = __half22float2(vp[i]);
            s2 += (f.x - mean) * (f.x - mean) + (f.y - mean) * (f.y - mean);
        }
        s2 = warp_sum(s2);
        if (lane == 0) {
            s.mean[n] = mean;
            s.rstd[n] = rsqrtf(s2 / (2 * C) + 1e-5f);
        }
    }
    __syncthreads();
    for (int i = threadIdx.x; i < N * 8; i += blockDim.x) {
        const int m = i >> 3, q = i & 7;
        const uint4 raw = *reinterpret_cast<const uint4*>(u + mix_pixel(blockIdx.x, m, WS, Hq, Wq) * C4 + 2 * C + c0 + 8 * q);
        const __half* h = reinterpret_cast<const __half*>(&raw);
        __align__(16) __half o[8];
        const float mean = s.mean[m], rstd = s.rstd[m];
#pragma unroll
        for (int e = 0; e < 8; ++e) o[e] = __float2half_rn((__half2float(h[e]) - mean) * rstd * g2[c0 + 8 * q + e]);
        *reinterpret_cast<uint4*>(&s.v[m * 64 + ((q ^ (m & 7)) << 3)]) = *reinterpret_cast<const uint4*>(o);
    }
    __syncthreads();
}

template <int N>
__global__ void __launch_bounds__(N) token_mix_mma_kernel(__half* __restrict__ u, int Hq, int Wq, int C,
                                                          const uint4* __restrict__ wfrag, const float* __restrict__ bs,
                                                          const float* __restrict__ g2) {
    constexpr int WS = N == 256 ? 16 : 8;
    __shared__ __align__(16) MixSmem<N> s;
    mix_load<N>(s, u, Hq, Wq, C, g2);
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    float acc[2][8][4];
#pragma unroll
    for (int a = 0; a < 2; ++a)
#pragma unroll
        for (int b = 0; b < 8; ++b)
#pragma unroll
            for (int c = 0; c < 4; ++c) acc[a][b][c] = 0.f;
    const uint32_t sv = smem_u32(s.v);
#pragma unroll 2
    for (int kt = 0; kt < N / 16; ++kt) {
        uint4 af[2];
#pragma unroll
        for (int mt = 0; mt < 2; ++mt) af[mt] = __ldg(&wfrag[((size_t)(warp * 2 + mt) * (N / 16) + kt) * 32 + lane]);
        const int row = kt * 16 + (lane & 15);
#pragma unroll
        for (int np = 0; np < 4; ++np) {
            const int chunk = (np * 2 + (lane >> 4)) ^ (row & 7);
            uint32_t b[4];
            ldmatrix_x4_trans(b, sv + (uint32_t)(row * 64 + chunk * 8) * 2);
#pragma unroll
            for (int mt = 0; mt < 2; ++mt) {
                const uint32_t a[4] = {af[mt].x, af[mt].y, af[mt].z, af[mt].w};
                mma16816(acc[mt][2 * np], a, b[0], b[1]);
                mma16816(acc[mt][2 * np + 1], a, b[2], b[3]);
            }
        }
    }
    const int g = lane >> 2, t4 = lane & 3, c0 = blockIdx.y * 64, C4 = 4 * C;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int n = warp * 32 + mt * 16 + g + 8 * h;
            const float bn = bs[n];
            __half2* up = reinterpret_cast<__half2*>(u + mix_pixel(blockIdx.x, n, WS, Hq, Wq) * C4 + c0);
#pragma unroll
            for (int nt = 0; nt < 8; ++nt) {
                const int c = nt * 8 + 2 * t4;
                const float2 uu = __half22float2(up[c / 2]);
                up[c / 2] = __floats2half2_rn(uu.x * (acc[mt][nt][2 * h] + bn), uu.y * (acc[mt][nt][2 * h + 1] + bn));
            }
        }
}

// SIMT cross-check (g_tune[7]): one thread per row n, fp32 weights
template <int N>
__global__ void __launch_bounds__(N) token_mix_simt_kernel(__half* __restrict__ u, int Hq, int Wq, int C, const float* __restrict__ wf,
                                                           const float* __restrict__ bs, const float* __restrict__ g2) {
    constexpr int WS = N == 256 ? 16 : 8;
    __shared__ __align__(16) MixSmem<N> s;
    mix_load<N>(s, u, Hq, Wq, C, g2);
    const int n = threadIdx.x, c0 = blockIdx.y * 64;
    float acc[64];
#pragma unroll
    for (int c = 0; c < 64; ++c) acc[c] = 0.f;
#pragma unroll 1
    for (int m = 0; m < N; ++m) {
        const float w = wf[(size_t)n * N + m];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const uint4 raw = *reinterpret_cast<const uint4*>(&s.v[m * 64 + ((q ^ (m & 7)) << 3)]);
            const __half* h = reinterpret_cast<const __half*>(&raw);
#pragma unroll
            for (int e = 0; e < 8; ++e) acc[q * 8 + e] = fmaf(w, __half2float(h[e]), acc[q * 8 + e]);
        }
    }
    __half2* up = reinterpret_cast<__half2*>(u + mix_pixel(blockIdx.x, n, WS, Hq, Wq) * 4 * C + c0);
    const float bn = bs[n];
#pragma unroll
    for (int c = 0; c < 64; c += 2) {
        const float2 uu = __half22float2(up[c / 2]);
        up[c / 2] = __floats2half2_rn(uu.x * (acc[c] + bn), uu.y * (acc[c + 1] + bn));
    }
}

int inpaint_token_mix(cudaStream_t st, __half* u, int B, int Hq, int Wq, int C, int ws, const __half* wfrag, const float* wf,
                      const float* bs, const float* g2) {
    NB_CHECK(Hq % ws == 0 && Wq % ws == 0 && (2 * C) % 64 == 0, "token mixing: the grid must tile into windows");
    const int N = ws * ws;
    const long long windows = (long long)B * (Hq / ws) * (Wq / ws);
    NB_CHECK(windows < (1LL << 31), "token mixing: too many windows");
    const dim3 grid((unsigned)windows, 2 * C / 64);
    const double tok = (double)windows * N;
    ProfScope ps(st, PC_ATTN, 2.0 * tok * N * 2 * C, tok * 4 * C * 2.0, tok * 2 * C * 2.0);
    const bool simt = g_tune[7] != 0;
    if (N == 256) {
        if (simt) token_mix_simt_kernel<256><<<grid, 256, 0, st>>>(u, Hq, Wq, C, wf, bs, g2);
        else token_mix_mma_kernel<256><<<grid, 256, 0, st>>>(u, Hq, Wq, C, reinterpret_cast<const uint4*>(wfrag), bs, g2);
    } else if (N == 64) {
        if (simt) token_mix_simt_kernel<64><<<grid, 64, 0, st>>>(u, Hq, Wq, C, wf, bs, g2);
        else token_mix_mma_kernel<64><<<grid, 64, 0, st>>>(u, Hq, Wq, C, reinterpret_cast<const uint4*>(wfrag), bs, g2);
    } else {
        return fail("token mixing: window must be 8 or 16");
    }
    NB_LAUNCHED();
    return 0;
}

// ---- replicate pad (+ GLU) -------------------------------------------------------------------------------------------------------
__global__ void __launch_bounds__(256) inpaint_pad_kernel(const __half* __restrict__ x, int B, int H, int W, int cs, int co, int glu,
                                                          __half* __restrict__ out) {
    const int groups = co / 8;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (size_t)B * (H + 2) * (W + 2) * groups) return;
    const int q = (int)(i % groups);
    const size_t pix = i / groups;
    const int xp = (int)(pix % (W + 2)), yp = (int)((pix / (W + 2)) % (H + 2)), bi = (int)(pix / ((size_t)(W + 2) * (H + 2)));
    const int y = min(max(yp - 1, 0), H - 1), xx = min(max(xp - 1, 0), W - 1);
    const __half* src = x + (((size_t)bi * H + y) * W + xx) * cs;
    uint4 r;
    if (!glu) {
        r = *reinterpret_cast<const uint4*>(src + 8 * q);
    } else {
        const int half = cs / 2;
        __align__(16) __half o[8];
        if (8 * q >= half) {
#pragma unroll
            for (int e = 0; e < 8; ++e) o[e] = __float2half_rn(0.f);
        } else {
            const uint4 ra = *reinterpret_cast<const uint4*>(src + 8 * q), rb = *reinterpret_cast<const uint4*>(src + half + 8 * q);
            const __half* a = reinterpret_cast<const __half*>(&ra);
            const __half* b = reinterpret_cast<const __half*>(&rb);
#pragma unroll
            for (int e = 0; e < 8; ++e) o[e] = __float2half_rn(__half2float(a[e]) / (1.f + __expf(-__half2float(b[e]))));
        }
        r = *reinterpret_cast<const uint4*>(o);
    }
    *reinterpret_cast<uint4*>(out + pix * co + 8 * q) = r;
}

int inpaint_pad(cudaStream_t st, const __half* x, int B, int H, int W, int cs, int co, int glu, __half* out) {
    NB_CHECK(co % 8 == 0 && cs % 8 == 0 && (glu ? (cs / 2) % 8 == 0 && co >= cs / 2 : co == cs), "inpaint_pad: bad channels");
    const size_t n = (size_t)B * (H + 2) * (W + 2) * (co / 8);
    ProfScope ps(st, PC_OTHER, n * 16.0 + (double)B * H * W * cs * 2, (double)B * H * W * cs * 2, n * 16.0);
    inpaint_pad_kernel<<<(unsigned)cdiv64(n, 256), 256, 0, st>>>(x, B, H, W, cs, co, glu, out);
    NB_LAUNCHED();
    return 0;
}

// ---- tail (light_inpaint_v1.py:125-126,137-154) -------------------------------------------------------------------------------------
// y: the to_image conv output [B][H4][W4][48]; pixel_shuffle(4) puts channel c*16 + dy*4 + dx of token (ty, tx) at (4ty+dy, 4tx+dx)
__global__ void __launch_bounds__(256) inpaint_tail_kernel(const __half* __restrict__ y, const float* __restrict__ x,
                                                           const float* __restrict__ hole, const float* __restrict__ blur, int B,
                                                           int H, int W, int H4, int W4, int mirror, float* __restrict__ out) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    const size_t plane = (size_t)H * W;
    if (i >= (size_t)B * plane) return;
    const int xi = (int)(i % W), yy = (int)((i / W) % H), bi = (int)(i / plane);
    const size_t p = i - (size_t)bi * plane;
    const int xn = mirror ? W - 1 - xi : xi;
    const float m = blur[(size_t)bi * plane + (size_t)yy * W + xn];
    const float keep = 1.f - hole[i];
    const __half* yt = y + (((size_t)bi * H4 + yy / 4) * W4 + xn / 4) * 48 + (yy % 4) * 4 + (xn % 4);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        const float src = x[((size_t)bi * 3 + c) * plane + p] * keep;
        const float net = __half2float(yt[c * 16]);
        out[((size_t)bi * 3 + c) * plane + p] = clamp01(src * (1.f - m) + net * m);
    }
}

int inpaint_tail(cudaStream_t st, const __half* y, const float* x, const float* hole, const float* blur, int B, int H, int W,
                 int Hp, int Wp, int mirror, float* out) {
    const size_t n = (size_t)B * H * W;
    ProfScope ps(st, PC_TOIMG, n * 34.0, n * 22.0, n * 12.0);
    inpaint_tail_kernel<<<(unsigned)cdiv64(n, 256), 256, 0, st>>>(y, x, hole, blur, B, H, W, Hp / 4, Wp / 4, mirror, out);
    NB_LAUNCHED();
    return 0;
}

}  // namespace nb200
