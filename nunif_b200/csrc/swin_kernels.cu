// Non-GEMM kernels of the SwinUNet path (NHWC fp16 activations).
//   stem_conv3x3_kernel     first 3x3 valid conv from the (3->8 padded) tile batch, LeakyReLU(0.1)
//                           (swin_unet.py:133-134, cunet.py:14-15 conv.0); K=27 is too thin for tensor cores
//   to_image_kernel         pixel_shuffle + clamp (+ bicubic-antialias /2,/4 + clamp) -> planar fp16 z
//                           (swin_unet.py:108-115, :366-379)
#include "common.cuh"
#include "swin_kernels.h"
#include "ptx.cuh"

namespace nb200 {

// ---------------------------------------------------------------------------------------------
// stem conv: x [n][Hi][Wi][8] fp16 -> out [n][Hi-2][Wi-2][ldo] fp16, channels >= cout written as 0
// weights: wt [27][COUT_PAD] fp32 (k = (ky*3+kx)*3 + ci), bias [COUT_PAD] fp32 (zero padded)
// ---------------------------------------------------------------------------------------------
template <int COUT_PAD>
__global__ void __launch_bounds__(128) stem_conv3x3_kernel(const __half* __restrict__ x, const float* __restrict__ wt,
                                                           const float* __restrict__ bias, __half* __restrict__ out,
                                                           int n, int Hi, int Wi, int ldo) {
    __shared__ __align__(16) float sw[27 * COUT_PAD];
    __shared__ __align__(16) float sb[COUT_PAD];
    for (int i = threadIdx.x; i < 27 * COUT_PAD; i += blockDim.x) sw[i] = wt[i];
    for (int i = threadIdx.x; i < COUT_PAD; i += blockDim.x) sb[i] = bias[i];
    __syncthreads();
    const int Ho = Hi - 2, Wo = Wi - 2;
    const size_t total = (size_t)n * Ho * Wo;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int ox = (int)(i % Wo), oy = (int)((i / Wo) % Ho), b = (int)(i / ((size_t)Wo * Ho));
    float in[27];
#pragma unroll
    for (int ky = 0; ky < 3; ++ky)
#pragma unroll
        for (int kx = 0; kx < 3; ++kx) {
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(x + (((size_t)b * Hi + oy + ky) * Wi + ox + kx) * 8));
            const __half2* h = reinterpret_cast<const __half2*>(&v);
            const float2 a = __half22float2(h[0]), c = __half22float2(h[1]);
            in[(ky * 3 + kx) * 3 + 0] = a.x;
            in[(ky * 3 + kx) * 3 + 1] = a.y;
            in[(ky * 3 + kx) * 3 + 2] = c.x;
        }
    __half* o = out + i * ldo;
#pragma unroll 1
    for (int c0 = 0; c0 < COUT_PAD; c0 += 8) {
        float acc[8];
#pragma unroll
        for (int j = 0; j < 8; ++j) acc[j] = sb[c0 + j];
#pragma unroll
        for (int k = 0; k < 27; ++k) {
            const float4 w0 = *reinterpret_cast<const float4*>(&sw[k * COUT_PAD + c0]);
            const float4 w1 = *reinterpret_cast<const float4*>(&sw[k * COUT_PAD + c0 + 4]);
            acc[0] += in[k] * w0.x; acc[1] += in[k] * w0.y; acc[2] += in[k] * w0.z; acc[3] += in[k] * w0.w;
            acc[4] += in[k] * w1.x; acc[5] += in[k] * w1.y; acc[6] += in[k] * w1.z; acc[7] += in[k] * w1.w;
        }
        __align__(16) __half2 hv[4];
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            float a0 = acc[2 * j], a1 = acc[2 * j + 1];
            a0 = a0 > 0.f ? a0 : 0.1f * a0;
            a1 = a1 > 0.f ? a1 : 0.1f * a1;
            hv[j] = __floats2half2_rn(a0, a1);
        }
        *reinterpret_cast<uint4*>(o + c0) = *reinterpret_cast<const uint4*>(hv);
    }
}

// Tensor-core version (production path): K = 9 taps x 4 (3 channels + a zero) = 36 -> 3 k16 steps of mma.sync.m16n8k16.
// One block = 2 output rows x 64 columns (8 warps x 16 pixels); the 4 x 66 input window is staged in shared memory
// (16 B per NHWC8 pixel, so every A-fragment register is one 4-byte load: tap = ks*4 + t4/2 (+2), channel pair = (t4&1)*2),
// B fragments are pre-packed at load time (model.cu pack_stem) and copied with 16-byte loads; the warp's 16 x COUT tile is
// staged through shared memory so that global stores are 16 bytes per lane.  ~10 instructions per pixel instead of ~2200:
// the SIMT kernel above reached 32 % of the fp32 FMA peak (153 us per 16-tile batch), this one is bound by its
// 0.15 GB of output.
template <int COUT_PAD>
__global__ void __launch_bounds__(256) stem_conv_mma_kernel(const __half* __restrict__ x, const float* __restrict__ wt,
                                                            const float* __restrict__ bias, __half* __restrict__ out, int Hi, int Wi,
                                                            int ldo) {
    if (threadIdx.x == 0) NB_PDL_TRIGGER();
    constexpr int NT = COUT_PAD / 8, WC = 66;
    __shared__ __align__(16) __half sB[3 * NT * 128];
    __shared__ __align__(16) __half sX[4 * WC * 8];
    __shared__ __align__(16) __half sO[8][16][COUT_PAD + 8];
    __shared__ float sBias[COUT_PAD];
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
    const int Ho = Hi - 2, Wo = Wi - 2;
    const int j0 = blockIdx.x * 64, oy0 = blockIdx.y * 2, b = blockIdx.z;
    {
        const uint4* frag = reinterpret_cast<const uint4*>(wt + 27 * COUT_PAD);
        for (int i = tid; i < 3 * NT * 16; i += 256) reinterpret_cast<uint4*>(sB)[i] = __ldg(frag + i);
        if (tid < COUT_PAD) sBias[tid] = bias[tid];
    }
    const __half* xb = x + (size_t)b * Hi * Wi * 8;
    for (int i = tid; i < 4 * WC; i += 256) {
        const int col = i % WC, r = i / WC;
        const int iy = oy0 + r, ix = j0 + col;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (iy < Hi && ix < Wi) v = __ldg(reinterpret_cast<const uint4*>(xb + ((size_t)iy * Wi + ix) * 8));
        reinterpret_cast<uint4*>(sX)[i] = v;
    }
    __syncthreads();
    const int lrow = warp >> 2, lj = (warp & 3) * 16, oy = oy0 + lrow;
    if (oy >= Ho || j0 + lj >= Wo) return;
    float acc[NT][4];
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) acc[nt][0] = acc[nt][1] = acc[nt][2] = acc[nt][3] = 0.f;
#pragma unroll
    for (int ks = 0; ks < 3; ++ks) {
        // k = 2*t4 (+8): tap = ks*4 + (t4 >> 1) (+2), channels (t4 & 1)*2, +1
        const int tapa = ks * 4 + (t4 >> 1), tapb = tapa + 2, ch = (t4 & 1) * 2;
        uint32_t a[4] = {0u, 0u, 0u, 0u};
        if (tapa < 9) {
            const __half* p = sX + ((lrow + tapa / 3) * WC + lj + g + tapa % 3) * 8 + ch;
            a[0] = *reinterpret_cast<const uint32_t*>(p);
            a[1] = *reinterpret_cast<const uint32_t*>(p + 64);     // pixel + 8
        }
        if (tapb < 9) {
            const __half* p = sX + ((lrow + tapb / 3) * WC + lj + g + tapb % 3) * 8 + ch;
            a[2] = *reinterpret_cast<const uint32_t*>(p);
            a[3] = *reinterpret_cast<const uint32_t*>(p + 64);
        }
        const __half* wb = sB + ks * NT * 128 + g * 16 + 2 * t4;
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            mma16816(acc[nt], a, *reinterpret_cast<const uint32_t*>(wb + nt * 128), *reinterpret_cast<const uint32_t*>(wb + nt * 128 + 8));
        }
    }
    // bias + LeakyReLU(0.1) -> fp16, staged per warp, then 16-byte stores (one output pixel row = COUT_PAD*2 bytes)
#pragma unroll
    for (int nt = 0; nt < NT; ++nt) {
        const float b0 = sBias[nt * 8 + 2 * t4], b1 = sBias[nt * 8 + 2 * t4 + 1];
        float v0 = acc[nt][0] + b0, v1 = acc[nt][1] + b1, v2 = acc[nt][2] + b0, v3 = acc[nt][3] + b1;
        v0 = v0 > 0.f ? v0 : 0.1f * v0; v1 = v1 > 0.f ? v1 : 0.1f * v1;
        v2 = v2 > 0.f ? v2 : 0.1f * v2; v3 = v3 > 0.f ? v3 : 0.1f * v3;
        *reinterpret_cast<__half2*>(&sO[warp][g][nt * 8 + 2 * t4]) = __floats2half2_rn(v0, v1);
        *reinterpret_cast<__half2*>(&sO[warp][g + 8][nt * 8 + 2 * t4]) = __floats2half2_rn(v2, v3);
    }
    __syncwarp();
    constexpr int VPR = COUT_PAD / 8;                          // 16-byte vectors per pixel
    for (int i = lane; i < 16 * VPR; i += 32) {
        const int r = i / VPR, v = i - r * VPR;
        const int ox = j0 + lj + r;
        if (ox < Wo)
            *reinterpret_cast<uint4*>(out + (((size_t)b * Ho + oy) * Wo + ox) * ldo + v * 8) = *reinterpret_cast<const uint4*>(&sO[warp][r][v * 8]);
    }
}

extern int g_tune[16];  // gemm.cu; [7] != 0 selects the SIMT stem / tail kernels (tests)

int stem_conv3x3(cudaStream_t st, const __half* x, const float* wt, const float* bias, __half* out, int n, int Hi, int Wi,
                 int cout_pad, int ldo) {
    NB_CHECK(ldo >= cout_pad && ldo % 8 == 0, "bad output stride");
    const bool mma = g_tune[7] == 0 && n <= 65535 && (cout_pad == 64 || cout_pad == 32);
    if (rec_on(REC_CONV))
        rec_launch("stem", {{"n", n}, {"Hi", Hi}, {"Wi", Wi}, {"cout_pad", cout_pad}, {"ldo", ldo}, {"path", mma ? 0 : 1}});
    if (mma) {
        const int Ho = Hi - 2, Wo = Wi - 2;
        ProfScope ps(st, PC_STEM, (double)n * Hi * Wi * 16 + (double)n * Ho * Wo * ldo * 2, (double)n * Hi * Wi * 16, (double)n * Ho * Wo * cout_pad * 2);
        const dim3 grid(cdiv(Wo, 64), cdiv(Ho, 2), n);
        if (cout_pad == 64) stem_conv_mma_kernel<64><<<grid, 256, 0, st>>>(x, wt, bias, out, Hi, Wi, ldo);
        else stem_conv_mma_kernel<32><<<grid, 256, 0, st>>>(x, wt, bias, out, Hi, Wi, ldo);
        NB_LAUNCHED();
        return 0;
    }
    const size_t total = (size_t)n * (Hi - 2) * (Wi - 2);
    const unsigned blocks = (unsigned)cdiv64(total, 128);
    ProfScope ps(st, PC_STEM, (double)n * Hi * Wi * 16 + (double)total * ldo * 2);
    if (cout_pad == 64) stem_conv3x3_kernel<64><<<blocks, 128, 0, st>>>(x, wt, bias, out, n, Hi, Wi, ldo);
    else if (cout_pad == 32) stem_conv3x3_kernel<32><<<blocks, 128, 0, st>>>(x, wt, bias, out, n, Hi, Wi, ldo);
    else return fail("stem_conv3x3: unsupported channel count");
    NB_LAUNCHED();
    return 0;
}

// ---------------------------------------------------------------------------------------------
// ToImage tail: y [n][Hs][Ws][cs] fp16 with channel = c*r*r + dy*r + dx (F.pixel_shuffle) ->
// z planar fp16 [n][3][S][S], S = Hs*r/down.  down>1: clamp, bicubic antialias (A=-0.5) resize, clamp.
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ float shuffled_px(const __half* __restrict__ yb, int Ws, int cs, int r, int c, int Y, int X) {
    const int ty = Y / r, dy = Y - ty * r, tx = X / r, dx = X - tx * r;
    return __half2float(yb[((size_t)ty * Ws + tx) * cs + c * r * r + dy * r + dx]);
}

// z: fp16 for down == 1 (what the reference's module returns under autocast), fp32 for the downscaled models (the reference
// resizes `z.float()` and returns fp32, swin_unet.py:366-379)
__global__ void __launch_bounds__(256) to_image_kernel(const __half* __restrict__ y, void* __restrict__ z, int n, int Hs,
                                                       int Ws, int cs, int r, int down) {
    const int S_full = Hs * r, S = S_full / down;
    const size_t total = (size_t)n * 3 * S * S;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int X = (int)(i % S), Y = (int)((i / S) % S), c = (int)((i / ((size_t)S * S)) % 3), b = (int)(i / ((size_t)3 * S * S));
    const __half* yb = y + (size_t)b * Hs * Ws * cs;
    float v;
    if (down == 1) {
        v = clamp01(shuffled_px(yb, Ws, cs, r, c, Y, X));
    } else {
        // ATen upsample_bicubic2d_aa, align_corners=False: scale = down, support = 2*scale
        const float scale = (float)down, support = 2.f * scale, inv = 1.f / scale;
        const float cy = scale * (Y + 0.5f), cx = scale * (X + 0.5f);
        const int ymin = max((int)(cy - support + 0.5f), 0), ysz = min((int)(cy + support + 0.5f), S_full) - ymin;
        const int xmin = max((int)(cx - support + 0.5f), 0), xsz = min((int)(cx + support + 0.5f), S_full) - xmin;
        float wy[17], wx[17], ty = 0.f, tx = 0.f;
        for (int k = 0; k < ysz; ++k) { wy[k] = cubic_aa((k + ymin - cy + 0.5f) * inv); ty += wy[k]; }
        for (int k = 0; k < xsz; ++k) { wx[k] = cubic_aa((k + xmin - cx + 0.5f) * inv); tx += wx[k]; }
        float acc = 0.f;
        for (int a = 0; a < ysz; ++a) {
            float row = 0.f;
            for (int k = 0; k < xsz; ++k) row += clamp01(shuffled_px(yb, Ws, cs, r, c, ymin + a, xmin + k)) * (wx[k] / tx);
            acc += row * (wy[a] / ty);
        }
        v = clamp01(acc);
    }
    if (down == 1) reinterpret_cast<__half*>(z)[i] = __float2half_rn(v);
    else reinterpret_cast<float*>(z)[i] = v;
}

// r=4, down=1 fast path: one thread per token reads its 48 contiguous channels (6 x 16 B) and writes, for each
// colour plane, four rows of four horizontally adjacent pixels (8-byte stores, coalesced across the warp).
__global__ void __launch_bounds__(256) to_image_r4_kernel(const __half* __restrict__ y, __half* __restrict__ z, int n, int Hs, int Ws) {
    const size_t total = (size_t)n * Hs * Ws;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int tx = (int)(i % Ws), ty = (int)((i / Ws) % Hs), b = (int)(i / ((size_t)Ws * Hs));
    const uint4* src = reinterpret_cast<const uint4*>(y + i * 48);
    const int S = Hs * 4;
    const __half2 zero = __float2half2_rn(0.f), one = __float2half2_rn(1.f);
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        // channel index = c*16 + dy*4 + dx (F.pixel_shuffle): two uint4 per colour plane
        uint4 v0 = __ldg(src + 2 * c), v1 = __ldg(src + 2 * c + 1);
        __half2* h0 = reinterpret_cast<__half2*>(&v0);
        __half2* h1 = reinterpret_cast<__half2*>(&v1);
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            h0[k] = __hmin2(__hmax2(h0[k], zero), one);  // clamp(z, 0, 1), swin_unet.py:286
            h1[k] = __hmin2(__hmax2(h1[k], zero), one);
        }
        __half* dst = z + (((size_t)b * 3 + c) * S + (size_t)ty * 4) * S + (size_t)tx * 4;
        *reinterpret_cast<uint2*>(dst) = make_uint2(v0.x, v0.y);
        *reinterpret_cast<uint2*>(dst + S) = make_uint2(v0.z, v0.w);
        *reinterpret_cast<uint2*>(dst + 2 * (size_t)S) = make_uint2(v1.x, v1.y);
        *reinterpret_cast<uint2*>(dst + 3 * (size_t)S) = make_uint2(v1.z, v1.w);
    }
}

// r = 4, down in {2, 4} (SwinUNetDownscaled, swin_unet.py:366-379): separable form of the kernel above.
// One block = a TO x TO output tile of one colour plane: the clamped 4x pixels it needs are gathered once into shared
// memory (8-byte loads: the 4 dx of a token row are contiguous), then a horizontal and a vertical pass with per-row /
// per-column tap tables (ATen upsample_bicubic2d_aa weights incl. border renormalisation): 2*4*down FMAs per output
// instead of (4*down)^2 taps with index arithmetic each.  Same summation order as ATen (horizontal first).
template <int DOWN>
__global__ void __launch_bounds__(256) to_image_down_kernel(const __half* __restrict__ y, float* __restrict__ z, int Hs, int Ws) {
    constexpr int NT = 4 * DOWN, TO = 64 / DOWN, IN = TO * DOWN + NT;   // taps, output tile, staged input side
    __shared__ float sP[IN][IN + 1];
    __shared__ float sH[IN][TO + 1];
    __shared__ float sWy[TO][NT], sWx[TO][NT];
    __shared__ int sMinY[TO], sMinX[TO], sSzY[TO], sSzX[TO];
    const int S_full = Hs * 4, S = S_full / DOWN;
    const int X0 = blockIdx.x * TO, Y0 = blockIdx.y * TO, c = blockIdx.z % 3, b = blockIdx.z / 3;
    const int tid = threadIdx.x;
    if (tid < 2 * TO) {
        const bool isx = tid >= TO;
        const int o = (isx ? X0 : Y0) + (isx ? tid - TO : tid);
        const float scale = (float)DOWN, support = 2.f * scale, inv = 1.f / scale;
        const float ctr = scale * ((float)min(o, S - 1) + 0.5f);
        const int mn = max((int)(ctr - support + 0.5f), 0), sz = min((int)(ctr + support + 0.5f), S_full) - mn;
        float w[NT], t = 0.f;
#pragma unroll
        for (int k = 0; k < NT; ++k) {
            w[k] = k < sz ? cubic_aa(((float)(k + mn) - ctr + 0.5f) * inv) : 0.f;
            t += w[k];
        }
        const int i = isx ? tid - TO : tid;
#pragma unroll
        for (int k = 0; k < NT; ++k) (isx ? sWx : sWy)[i][k] = w[k] / t;
        (isx ? sMinX : sMinY)[i] = mn;
        (isx ? sSzX : sSzY)[i] = sz;
    }
    __syncthreads();
    const int ry0 = sMinY[0], rx0 = sMinX[0];
    const int rx0a = rx0 & ~3;                                         // token-aligned start column
    const __half* yb = y + (size_t)b * Hs * Ws * 48 + c * 16;
    // gather: rows ry0 .. ry0+IN-1, columns rx0a .. in groups of 4 (one token row segment = 8 bytes)
    constexpr int G = (IN + 3) / 4 + 1;
    for (int i = tid; i < IN * G; i += 256) {
        const int r = i / G, gq = i - r * G;
        const int py = min(ry0 + r, S_full - 1), px = rx0a + 4 * gq;
        uint2 raw = make_uint2(0, 0);
        if (px < S_full) raw = __ldg(reinterpret_cast<const uint2*>(yb + ((size_t)(py >> 2) * Ws + (px >> 2)) * 48 + (py & 3) * 4));
        const __half2* h = reinterpret_cast<const __half2*>(&raw);
        const float2 f0 = __half22float2(h[0]), f1 = __half22float2(h[1]);
        const float v[4] = {f0.x, f0.y, f1.x, f1.y};
#pragma unroll
        for (int k = 0; k < 4; ++k) {
            const int col = px + k - rx0;
            if (col >= 0 && col < IN) sP[r][col] = clamp01(v[k]);      // clamp(z, 0, 1) before the resize (:369)
        }
    }
    __syncthreads();
    for (int i = tid; i < IN * TO; i += 256) {
        const int r = i / TO, ox = i - r * TO;
        const int base = sMinX[ox] - rx0, sz = sSzX[ox];
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < NT; ++k)
            if (k < sz) acc += sP[r][base + k] * sWx[ox][k];
        sH[r][ox] = acc;
    }
    __syncthreads();
    for (int i = tid; i < TO * TO; i += 256) {
        const int oy = i / TO, ox = i - oy * TO;
        if (Y0 + oy >= S || X0 + ox >= S) continue;
        const int base = sMinY[oy] - ry0, sz = sSzY[oy];
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < NT; ++k)
            if (k < sz) acc += sH[base + k][ox] * sWy[oy][k];
        z[(((size_t)b * 3 + c) * S + Y0 + oy) * S + X0 + ox] = clamp01(acc);
    }
}

int to_image(cudaStream_t st, const __half* y, void* z, int n, int Hs, int Ws, int cs, int r, int down) {
    if (rec_on(REC_CONV)) rec_launch("toimg", {{"n", n}, {"Hs", Hs}, {"Ws", Ws}, {"cs", cs}, {"r", r}, {"down", down}});
    NB_CHECK(down == 1 || down == 2 || down == 4, "downscale must be 1, 2 or 4");
    NB_CHECK(Hs == Ws && (Hs * r) % down == 0, "bad ToImage geometry");
    const size_t total = (size_t)n * 3 * (Hs * r / down) * (Ws * r / down);
    ProfScope ps(st, PC_TOIMG, (double)n * Hs * Ws * cs * 2 + (double)total * 2);
    if (r == 4 && down == 1 && cs == 48) {
        const size_t tokens = (size_t)n * Hs * Ws;
        to_image_r4_kernel<<<(unsigned)cdiv64(tokens, 256), 256, 0, st>>>(y, (__half*)z, n, Hs, Ws);
    } else if (r == 4 && cs == 48 && down == 2) {
        const int S = Hs * 2;
        to_image_down_kernel<2><<<dim3(cdiv(S, 32), cdiv(S, 32), n * 3), 256, 0, st>>>(y, (float*)z, Hs, Ws);
    } else if (r == 4 && cs == 48 && down == 4) {
        const int S = Hs;
        to_image_down_kernel<4><<<dim3(cdiv(S, 16), cdiv(S, 16), n * 3), 256, 0, st>>>(y, (float*)z, Hs, Ws);
    } else {
        to_image_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(y, z, n, Hs, Ws, cs, r, down);
    }
    NB_LAUNCHED();
    return 0;
}

}  // namespace nb200

using namespace nb200;

extern "C" int nb200_to_image_f16(const void* y, int n, int Hs, int Ws, int cs, int r, int down, void* z, void* stream) {
    NB_CHECK(y && z, "null pointer");
    NB_CHECK(n > 0 && Hs > 0 && r > 0 && cs >= 3 * r * r, "bad ToImage shape");
    return to_image((cudaStream_t)stream, (const __half*)y, z, n, Hs, Ws, cs, r, down);
}
