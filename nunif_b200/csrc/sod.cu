// iw3.sod_v1 saliency network and the convergence estimate built on it (iw3/models/sod_v1.py, nunif/utils/u2netp.py,
// iw3/convergence_estimator.py).
//
//   * sod_prep_kernel: both bilinear resizes to 192 x 192 (ATen upsample_bilinear2d arithmetic), depth ** 0.5, depth ** 2
//     and the NHWC fp16 pack of the 6 network channels (padded to 16).
//   * sod_conv_kernel: every REBNCONV as an implicit GEMM on mma.sync m16n8k16 - one CTA = 8 x 16 output pixels x all output
//     channels, K = 9 taps x 16-channel chunks staged in shared memory with the dilated zero halo.  The epilogue adds the
//     folded bias, applies ReLU and the RSU residual and writes into a channel slice of a wider buffer, so every
//     torch.cat of the reference is free (the decoder half is written by the upsample, the skip half by the encoder conv).
//   * sod_pool_kernel / sod_upsample_kernel: MaxPool2d(2, ceil_mode) at even sizes and _upsample_like (bilinear,
//     align_corners=False) on fp16, with the same channel-slice addressing.
//   * sod_side_kernel + sod_head_kernel: the six 64 -> 1 side convs, their upsample to 192, the 1x1 outconv and the sigmoid.
//   * sod_position_kernel: ConvergenceEstimator.depth_position_from_ratio, one CTA per image (mask, the two torch.quantile
//     values by radix select, the branch, the clamp).  sod_ema_kernel: the EMA recurrence over the batch.
#include "sod_kernels.h"
#include "ptx.cuh"
#include "../../include/nunif_b200.h"
#include <cmath>

namespace nb200 {

// rgb [B][3][H][W], depth [B][1][h][w] -> x [B][192][192][16] fp16 (r, g, b, d, sqrt(d), d*d, 0 ...), depth192 fp32
__global__ void __launch_bounds__(256) sod_prep_kernel(const float* __restrict__ rgb, int H, int W, const float* __restrict__ depth,
                                                       int h, int w, __half* __restrict__ x, float* __restrict__ depth192) {
    const int S = SOD_SIZE;
    const int i = blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (i >= S * S) return;
    const int oy = i / S, ox = i % S;
    float v[8];
    {
        const BilTap ty = bil_tap((float)H / (float)S, oy, H), tx = bil_tap((float)W / (float)S, ox, W);
        for (int c = 0; c < 3; ++c) {
            const float* p = rgb + ((size_t)b * 3 + c) * H * W;
            v[c] = bil_mix(ty, tx, __ldg(p + (size_t)ty.i0 * W + tx.i0), __ldg(p + (size_t)ty.i0 * W + tx.i1),
                           __ldg(p + (size_t)ty.i1 * W + tx.i0), __ldg(p + (size_t)ty.i1 * W + tx.i1));
        }
    }
    {
        const BilTap ty = bil_tap((float)h / (float)S, oy, h), tx = bil_tap((float)w / (float)S, ox, w);
        const float* p = depth + (size_t)b * h * w;
        const float d = bil_mix(ty, tx, __ldg(p + (size_t)ty.i0 * w + tx.i0), __ldg(p + (size_t)ty.i0 * w + tx.i1),
                                __ldg(p + (size_t)ty.i1 * w + tx.i0), __ldg(p + (size_t)ty.i1 * w + tx.i1));
        depth192[(size_t)b * S * S + i] = d;
        v[3] = d;
        v[4] = __fsqrt_rn(d);       // depth ** 0.5 is ATen's sqrt kernel
        v[5] = __fmul_rn(d, d);     // depth ** 2 is base * base
    }
    v[6] = v[7] = 0.f;
    __align__(16) __half hv[16];
    for (int c = 0; c < 8; ++c) hv[c] = __float2half_rn(v[c]);
    for (int c = 8; c < 16; ++c) hv[c] = __float2half_rn(0.f);
    uint4* o = reinterpret_cast<uint4*>(x + ((size_t)b * S * S + i) * 16);
    o[0] = reinterpret_cast<const uint4*>(hv)[0];
    o[1] = reinterpret_cast<const uint4*>(hv)[1];
}

// ---------------------------------------------------------------------------------------------
// REBNCONV: out = relu(conv3x3_dil(in) + bias) [+ res], fp16 in / out, fp32 accumulation
// ---------------------------------------------------------------------------------------------
struct SodConvArgs {
    const __half* in; int in_ld, in_off, cin;   // reads channels [in_off, in_off + cin) of an NHWC buffer with stride in_ld
    const __half* wt; const float* bias;        // wt [cout][9][cin]
    __half* out; int out_ld, out_off;
    const __half* res; int res_ld, res_off;     // optional residual (added after the ReLU)
    int H, W, dil;
};

constexpr int SC_TH = 8, SC_TW = 16, SC_PX = 24, SC_WROW = 152;   // tile rows / cols; smem halves per pixel / per weight row

template <int COUT>
__global__ void __launch_bounds__(128) sod_conv_kernel(SodConvArgs a) {
    constexpr int NT = COUT / 8;
    extern __shared__ __align__(16) __half sc_smem[];
    const int d = a.dil, tw = SC_TW + 2 * d, th = SC_TH + 2 * d;
    __half* s_in = sc_smem;                          // [th][tw][SC_PX]
    __half* s_w = sc_smem + th * tw * SC_PX;         // [COUT][SC_WROW]: [9][16] of the chunk
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t = lane & 3;
    const int x0 = blockIdx.x * SC_TW, y0 = blockIdx.y * SC_TH, b = blockIdx.z;
    const __half* in = a.in + (size_t)b * a.H * a.W * a.in_ld + a.in_off;

    float acc[2][NT][4];
#pragma unroll
    for (int m = 0; m < 2; ++m)
#pragma unroll
        for (int n = 0; n < NT; ++n)
#pragma unroll
            for (int q = 0; q < 4; ++q) acc[m][n][q] = 0.f;

    for (int c0 = 0; c0 < a.cin; c0 += 16) {
        __syncthreads();
        for (int i = tid; i < th * tw * 2; i += 128) {
            const int px = i >> 1, hf = i & 1, r = px / tw, q = px % tw;
            const int gy = y0 - d + r, gx = x0 - d + q;
            uint4 v = make_uint4(0, 0, 0, 0);
            if (gy >= 0 && gy < a.H && gx >= 0 && gx < a.W)
                v = __ldg(reinterpret_cast<const uint4*>(in + ((size_t)gy * a.W + gx) * a.in_ld + c0 + hf * 8));
            *reinterpret_cast<uint4*>(s_in + px * SC_PX + hf * 8) = v;
        }
        for (int i = tid; i < COUT * 9 * 2; i += 128) {
            const int row = i / 18, k = i % 18, tap = k >> 1, hf = k & 1;
            *reinterpret_cast<uint4*>(s_w + row * SC_WROW + tap * 16 + hf * 8) =
                __ldg(reinterpret_cast<const uint4*>(a.wt + ((size_t)row * 9 + tap) * a.cin + c0 + hf * 8));
        }
        __syncthreads();
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const int dy = (tap / 3) * d, dx = (tap % 3) * d;
            uint32_t bf[NT][2];
#pragma unroll
            for (int n = 0; n < NT; ++n) {
                const __half* wp = s_w + (n * 8 + g) * SC_WROW + tap * 16 + 2 * t;
                bf[n][0] = *reinterpret_cast<const uint32_t*>(wp);
                bf[n][1] = *reinterpret_cast<const uint32_t*>(wp + 8);
            }
#pragma unroll
            for (int m = 0; m < 2; ++m) {
                const int r = warp * 2 + m + dy;
                const __half* ap = s_in + (r * tw + g + dx) * SC_PX + 2 * t;
                const uint32_t af[4] = {*reinterpret_cast<const uint32_t*>(ap), *reinterpret_cast<const uint32_t*>(ap + 8 * SC_PX),
                                        *reinterpret_cast<const uint32_t*>(ap + 8), *reinterpret_cast<const uint32_t*>(ap + 8 * SC_PX + 8)};
#pragma unroll
                for (int n = 0; n < NT; ++n) mma16816(acc[m][n], af, bf[n][0], bf[n][1]);
            }
        }
    }
    // epilogue: the conv output is rounded to fp16 before its fp16 bias is added (cuDNN under autocast), ReLU, residual
#pragma unroll
    for (int m = 0; m < 2; ++m) {
        const int y = y0 + warp * 2 + m;
        if (y >= a.H) continue;
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {
            const int x = x0 + g + hh * 8;
            if (x >= a.W) continue;
            const size_t px = ((size_t)b * a.H + y) * a.W + x;
#pragma unroll
            for (int n = 0; n < NT; ++n) {
                const int co = n * 8 + 2 * t;
                float v0 = fmaxf(round_f16(round_f16(acc[m][n][hh * 2]) + a.bias[co]), 0.f);
                float v1 = fmaxf(round_f16(round_f16(acc[m][n][hh * 2 + 1]) + a.bias[co + 1]), 0.f);
                if (a.res) {
                    const __half2 r = *reinterpret_cast<const __half2*>(a.res + px * a.res_ld + a.res_off + co);
                    v0 += __low2float(r);
                    v1 += __high2float(r);
                }
                *reinterpret_cast<__half2*>(a.out + px * a.out_ld + a.out_off + co) = __floats2half2_rn(v0, v1);
            }
        }
    }
}

// one REBNCONV launch over B images (the network's layers and nb200_sod_conv_f16)
int sod_conv(cudaStream_t st, const SodConvArgs& a, int cout, int B) {
    if (rec_on(REC_CONV))
        rec_launch("sodconv", {{"B", B}, {"H", a.H}, {"W", a.W}, {"cin", a.cin}, {"cout", cout}, {"dil", a.dil}, {"in_ld", a.in_ld},
                               {"in_off", a.in_off}, {"out_ld", a.out_ld}, {"out_off", a.out_off}, {"has_res", a.res ? 1 : 0},
                               {"res_ld", a.res_ld}});
    NB_CHECK(cout == 16 || cout == 64, "output channels must be 16 or 64");
    NB_CHECK(a.cin > 0 && a.cin % 16 == 0 && a.in_ld % 8 == 0 && a.in_off % 8 == 0 && a.in_off + a.cin <= a.in_ld,
             "input channels must be a multiple of 16 inside a 16-byte aligned slice");
    NB_CHECK(a.out_ld % 2 == 0 && a.out_off % 2 == 0 && a.out_off + cout <= a.out_ld, "bad output slice");
    NB_CHECK(!a.res || (a.res_ld % 2 == 0 && a.res_off % 2 == 0 && a.res_off + cout <= a.res_ld), "bad residual slice");
    NB_CHECK(a.dil >= 1 && a.H > 0 && a.W > 0 && B > 0 && B <= 65535, "bad geometry");
    const int d = a.dil;
    const size_t smem = ((size_t)(SC_TH + 2 * d) * (SC_TW + 2 * d) * SC_PX + (size_t)cout * SC_WROW) * sizeof(__half);
    const dim3 grid(cdiv(a.W, SC_TW), cdiv(a.H, SC_TH), B);
    ProfScope ps(st, PC_OTHER, 2.0 * B * a.H * a.W * cout * 9.0 * a.cin);
    if (cout == 64) {
        if (ensure_dyn_smem((const void*)sod_conv_kernel<64>, smem)) return 1;
        sod_conv_kernel<64><<<grid, 128, smem, st>>>(a);
    } else {
        if (ensure_dyn_smem((const void*)sod_conv_kernel<16>, smem)) return 1;
        sod_conv_kernel<16><<<grid, 128, smem, st>>>(a);
    }
    NB_LAUNCHED();
    return 0;
}

// MaxPool2d(2, stride 2, ceil_mode=True) at even H, W: in channels [in_off, in_off + C) -> out [H/2][W/2] slice
__global__ void __launch_bounds__(256) sod_pool_kernel(const __half* __restrict__ in, int in_ld, int in_off, int C, int H, int W,
                                                       __half* __restrict__ out, int out_ld, int out_off, long long total) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int G = C / 8, Ho = H / 2, Wo = W / 2;
    const int gq = (int)(i % G);
    long long px = i / G;
    const int x = (int)(px % Wo), y = (int)((px / Wo) % Ho), b = (int)(px / ((long long)Wo * Ho));
    const __half* p = in + (((size_t)b * H + 2 * y) * W + 2 * x) * in_ld + in_off + gq * 8;
    uint4 v[4] = {__ldg(reinterpret_cast<const uint4*>(p)), __ldg(reinterpret_cast<const uint4*>(p + in_ld)),
                  __ldg(reinterpret_cast<const uint4*>(p + (size_t)W * in_ld)), __ldg(reinterpret_cast<const uint4*>(p + (size_t)(W + 1) * in_ld))};
    uint4 r;
    const __half2* h0 = reinterpret_cast<const __half2*>(&v[0]);
    const __half2* h1 = reinterpret_cast<const __half2*>(&v[1]);
    const __half2* h2 = reinterpret_cast<const __half2*>(&v[2]);
    const __half2* h3 = reinterpret_cast<const __half2*>(&v[3]);
    __half2* hr = reinterpret_cast<__half2*>(&r);
#pragma unroll
    for (int k = 0; k < 4; ++k) hr[k] = __hmax2(__hmax2(h0[k], h1[k]), __hmax2(h2[k], h3[k]));
    *reinterpret_cast<uint4*>(out + (((size_t)b * Ho + y) * Wo + x) * out_ld + out_off + gq * 8) = r;
}

// _upsample_like: bilinear, align_corners=False, on fp16 (fp32 arithmetic, one rounding)
__global__ void __launch_bounds__(256) sod_upsample_kernel(const __half* __restrict__ in, int in_ld, int in_off, int C, int h, int w,
                                                           __half* __restrict__ out, int out_ld, int out_off, int H, int W,
                                                           long long total) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int G = C / 8;
    const int gq = (int)(i % G);
    long long px = i / G;
    const int x = (int)(px % W), y = (int)((px / W) % H), b = (int)(px / ((long long)W * H));
    const BilTap ty = bil_tap((float)h / (float)H, y, h), tx = bil_tap((float)w / (float)W, x, w);
    const __half* base = in + (size_t)b * h * w * in_ld + in_off + gq * 8;
    uint4 q00 = __ldg(reinterpret_cast<const uint4*>(base + ((size_t)ty.i0 * w + tx.i0) * in_ld));
    uint4 q01 = __ldg(reinterpret_cast<const uint4*>(base + ((size_t)ty.i0 * w + tx.i1) * in_ld));
    uint4 q10 = __ldg(reinterpret_cast<const uint4*>(base + ((size_t)ty.i1 * w + tx.i0) * in_ld));
    uint4 q11 = __ldg(reinterpret_cast<const uint4*>(base + ((size_t)ty.i1 * w + tx.i1) * in_ld));
    const __half* v00 = reinterpret_cast<const __half*>(&q00);
    const __half* v01 = reinterpret_cast<const __half*>(&q01);
    const __half* v10 = reinterpret_cast<const __half*>(&q10);
    const __half* v11 = reinterpret_cast<const __half*>(&q11);
    __align__(16) __half r[8];
#pragma unroll
    for (int k = 0; k < 8; ++k)
        r[k] = __float2half_rn(bil_mix(ty, tx, __half2float(v00[k]), __half2float(v01[k]), __half2float(v10[k]), __half2float(v11[k])));
    *reinterpret_cast<uint4*>(out + (((size_t)b * H + y) * W + x) * out_ld + out_off + gq * 8) = *reinterpret_cast<const uint4*>(r);
}

// side1..side6: Conv2d(64, 1, 3, padding=1) on hx1d, hx2d, hx3d, hx4d, hx5d, hx6 (dense 64-channel maps, level l at 192 >> l)
struct SodSideArgs {
    const __half* x[6];
    float* out[6];        // [B][s][s] fp32 holding fp16 values
    const float* w;       // [6][9][64] then [6] biases
};

__global__ void __launch_bounds__(256) sod_side_kernel(SodSideArgs a) {
    const int l = blockIdx.y, b = blockIdx.z, s = SOD_SIZE >> l;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= s * s) return;
    const int y = i / s, x = i % s;
    // pick the level's pointers with constant indices (a dynamic index would copy the parameter arrays to the stack)
    const __half* xl = a.x[0];
    float* ol = a.out[0];
#pragma unroll
    for (int k = 1; k < 6; ++k)
        if (k == l) { xl = a.x[k]; ol = a.out[k]; }
    const __half* in = xl + (size_t)b * s * s * 64;
    const float* wl = a.w + l * 9 * 64;
    float acc = 0.f;
    for (int tap = 0; tap < 9; ++tap) {
        const int yy = y + tap / 3 - 1, xx = x + tap % 3 - 1;
        if (yy < 0 || yy >= s || xx < 0 || xx >= s) continue;
        const uint4* p = reinterpret_cast<const uint4*>(in + ((size_t)yy * s + xx) * 64);
#pragma unroll
        for (int q = 0; q < 8; ++q) {
            const uint4 v = __ldg(p + q);
            const __half2* hv = reinterpret_cast<const __half2*>(&v);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float2 f = __half22float2(hv[k]);
                acc = fmaf(f.x, wl[tap * 64 + q * 8 + 2 * k], acc);
                acc = fmaf(f.y, wl[tap * 64 + q * 8 + 2 * k + 1], acc);
            }
        }
    }
    ol[(size_t)b * s * s + i] = round_f16(round_f16(acc) + a.w[6 * 9 * 64 + l]);
}

// d2..d6 upsampled to 192 (fp16), outconv (1x1, 6 -> 1) and the sigmoid, all rounded to fp16 as under autocast
__global__ void __launch_bounds__(256) sod_head_kernel(SodSideArgs a, const float* __restrict__ hw, float* __restrict__ sal) {
    const int S = SOD_SIZE, b = blockIdx.y;
    const int i = blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= S * S) return;
    const int y = i / S, x = i % S;
    float acc = __ldg(a.out[0] + (size_t)b * S * S + i) * hw[0];
#pragma unroll
    for (int l = 1; l < 6; ++l) {
        const int s = S >> l;
        const BilTap ty = bil_tap((float)s / (float)S, y, s), tx = bil_tap((float)s / (float)S, x, s);
        const float* p = a.out[l] + (size_t)b * s * s;
        const float d = round_f16(bil_mix(ty, tx, __ldg(p + ty.i0 * s + tx.i0), __ldg(p + ty.i0 * s + tx.i1),
                                        __ldg(p + ty.i1 * s + tx.i0), __ldg(p + ty.i1 * s + tx.i1)));
        acc = fmaf(d, hw[l], acc);
    }
    const float d0 = round_f16(round_f16(acc) + hw[6]);
    sal[(size_t)b * S * S + i] = round_f16(1.f / (1.f + expf(-d0)));
}

// ---------------------------------------------------------------------------------------------
// host: the U^2-Net-p forward
// ---------------------------------------------------------------------------------------------
struct HView { __half* p; int ld, off; };

struct SodRun {
    cudaStream_t st;
    const uint8_t* blob;
    const SodW* w;
    int B;
    size_t li = 0;   // next conv of w->convs
    // RSU scratch, sized for the 192 level and reused by every block
    __half* hin;     // [B][192][192][64]
    __half* cat[6];  // [B][192 >> k][192 >> k][32]: [0, 16) decoder / innermost, [16, 32) encoder skip
    __half* pool16;  // [B][96][96][16]
    __half* dec16;   // [B][192][192][16]

    int conv(HView in, int H, int W, HView out, const __half* res = nullptr, int res_ld = 0) {
        NB_CHECK(li < w->convs.size(), "layer list exhausted");
        const SodConv& L = w->convs[li++];
        SodConvArgs a;
        a.in = in.p; a.in_ld = in.ld; a.in_off = in.off; a.cin = L.cin_pad;
        a.wt = reinterpret_cast<const __half*>(blob + L.w); a.bias = reinterpret_cast<const float*>(blob + L.b);
        a.out = out.p; a.out_ld = out.ld; a.out_off = out.off;
        a.res = res; a.res_ld = res_ld; a.res_off = 0;
        a.H = H; a.W = W; a.dil = L.dil;
        return sod_conv(st, a, L.cout, B);
    }
    int pool(HView in, int C, int H, int W, HView out) {
        const long long total = (long long)B * (H / 2) * (W / 2) * (C / 8);
        sod_pool_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(in.p, in.ld, in.off, C, H, W, out.p, out.ld, out.off, total);
        NB_LAUNCHED();
        return 0;
    }
    int upsample(HView in, int C, int h, int wd, HView out, int H, int W) {
        const long long total = (long long)B * H * W * (C / 8);
        sod_upsample_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(in.p, in.ld, in.off, C, h, wd, out.p, out.ld, out.off, H, W,
                                                                          total);
        NB_LAUNCHED();
        return 0;
    }
    // RSU7/6/5/4 (n) or RSU4F (n = 0) at s x s: in -> out (64 channels) = rebnconv1d(...) + rebnconvin(in)
    int rsu(int n, HView in, int s, HView out) {
        const HView hin_v{hin, 64, 0};
        if (conv(in, s, s, hin_v)) return 1;
        if (n == 0) {
            // dilations 1, 2, 4, 8 / 4, 2, 1 at one resolution; hx_k lives in cat[k-1][16:32], hx4 / hx3d / hx2d in the left halves
            if (conv(hin_v, s, s, {cat[0], 32, 16})) return 1;
            if (conv({cat[0], 32, 16}, s, s, {cat[1], 32, 16})) return 1;
            if (conv({cat[1], 32, 16}, s, s, {cat[2], 32, 16})) return 1;
            if (conv({cat[2], 32, 16}, s, s, {cat[2], 32, 0})) return 1;
            if (conv({cat[2], 32, 0}, s, s, {cat[1], 32, 0})) return 1;
            if (conv({cat[1], 32, 0}, s, s, {cat[0], 32, 0})) return 1;
            return conv({cat[0], 32, 0}, s, s, out, hin, 64);
        }
        // encoder: hx1 at s, pool, hx2 at s/2, ... hx_{n-1} at s >> (n-2)
        if (conv(hin_v, s, s, {cat[0], 32, 16})) return 1;
        for (int k = 2; k < n; ++k) {
            const int sp = s >> (k - 2), sk = s >> (k - 1);
            if (pool({cat[k - 2], 32, 16}, 16, sp, sp, {pool16, 16, 0})) return 1;
            if (conv({pool16, 16, 0}, sk, sk, {cat[k - 1], 32, 16})) return 1;
        }
        const int si = s >> (n - 2);
        if (conv({cat[n - 2], 32, 16}, si, si, {cat[n - 2], 32, 0})) return 1;   // innermost, dilation 2
        // decoder: hx_kd = conv(cat(hx_{k+1}d up, hx_k)), upsampled into the left half of the level above
        for (int k = n - 1; k >= 2; --k) {
            const int sk = s >> (k - 1);
            if (conv({cat[k - 1], 32, 0}, sk, sk, {dec16, 16, 0})) return 1;
            if (upsample({dec16, 16, 0}, 16, sk, sk, {cat[k - 2], 32, 0}, 2 * sk, 2 * sk)) return 1;
        }
        return conv({cat[0], 32, 0}, s, s, out, hin, 64);
    }
};

int sod_forward(cudaStream_t st, const uint8_t* blob, const SodW& w, const float* rgb, int B, int H, int W, const float* depth,
                int h, int wd, float* saliency, float* depth192) {
    const int S = SOD_SIZE;
    const size_t px0 = (size_t)B * S * S;   // pixels of the 192 level; level l has px0 >> 2l
    SodRun r;
    r.st = st; r.blob = blob; r.w = &w; r.B = B;
    __half* x16;
    __half* scat[5];    // decoder stage inputs at levels 0..4: [up-sampled decoder 64 | encoder stage output 64]
    __half* pooled;     // pooled input of encoder stages 2..6
    __half* hxd[6];     // hx1d, hx2d, hx3d, hx4d, hx5d, hx6 (dense 64 channels)
    float* side;        // side1..6 outputs, level l at 192 >> l
    // the workspace is listed once: a pass over a null base sizes it, the second hands out the pointers
    auto plan = [&](uint8_t* base) {
        size_t off = 0;
        auto take = [&](size_t bytes) { off = (off + 255) & ~(size_t)255; uint8_t* p = base ? base + off : nullptr; off += bytes; return p; };
        auto th = [&](size_t halves) { return reinterpret_cast<__half*>(take(halves * 2)); };
        x16 = th(px0 * 16);
        r.hin = th(px0 * 64);
        r.pool16 = th((px0 >> 2) * 16);
        r.dec16 = th(px0 * 16);
        for (int k = 0; k < 6; ++k) r.cat[k] = th((px0 >> (2 * k)) * 32);
        for (int l = 0; l < 5; ++l) scat[l] = th((px0 >> (2 * l)) * 128);
        pooled = th((px0 >> 2) * 64);
        for (int l = 0; l < 6; ++l) hxd[l] = th((px0 >> (2 * l)) * 64);
        side = reinterpret_cast<float*>(take(px0 * 2 * 4));   // sum of px0 >> 2l over l < 2 * px0
        return off;
    };
    const size_t ws_bytes = plan(nullptr);
    size_t side_floats = 0;
    for (int l = 0; l < 6; ++l) side_floats += px0 >> (2 * l);
    uint8_t* ws = nullptr;
    NB_CUDA(cudaMallocAsync((void**)&ws, ws_bytes, st));
    plan(ws);

    int rc = 0;
    do {
        {
            ProfScope ps(st, PC_OTHER, 0.0, (double)B * (3.0 * H * W + (double)h * wd) * 4.0, (double)px0 * 36.0);
            sod_prep_kernel<<<dim3(cdiv(S * S, 256), B), 256, 0, st>>>(rgb, H, W, depth, h, wd, x16, depth192);
            NB_LAUNCHED();
        }
        // encoder: stage k output goes to the right half of the decoder input at its level
        if ((rc = r.rsu(7, {x16, 16, 0}, S, {scat[0], 128, 64}))) break;
        const int enc_n[4] = {6, 5, 4, 0};
        for (int l = 1; l <= 4; ++l) {
            const int s = S >> l;
            if ((rc = r.pool({scat[l - 1], 128, 64}, 64, 2 * s, 2 * s, {pooled, 64, 0}))) break;
            if ((rc = r.rsu(enc_n[l - 1], {pooled, 64, 0}, s, {scat[l], 128, 64}))) break;
        }
        if (rc) break;
        if ((rc = r.pool({scat[4], 128, 64}, 64, S >> 4, S >> 4, {pooled, 64, 0}))) break;
        if ((rc = r.rsu(0, {pooled, 64, 0}, S >> 5, {hxd[5], 64, 0}))) break;                       // hx6
        // decoder: stage5d, 4d, 3d, 2d, 1d
        const int dec_n[5] = {0, 4, 5, 6, 7};
        for (int j = 0; j < 5; ++j) {
            const int l = 4 - j, s = S >> l;
            if ((rc = r.upsample({hxd[l + 1], 64, 0}, 64, s / 2, s / 2, {scat[l], 128, 0}, s, s))) break;
            if ((rc = r.rsu(dec_n[j], {scat[l], 128, 0}, s, {hxd[l], 64, 0}))) break;
        }
        if (rc) break;
        NB_CHECK(r.li == w.convs.size(), "not every conv was run");
        SodSideArgs sa;
        float* sp = side;
        for (int l = 0; l < 6; ++l) { sa.x[l] = hxd[l]; sa.out[l] = sp; sp += px0 >> (2 * l); }
        sa.w = reinterpret_cast<const float*>(blob + w.side);
        {
            ProfScope ps(st, PC_OTHER, 2.0 * 576.0 * (double)side_floats);
            sod_side_kernel<<<dim3(cdiv(S * S, 256), 6, B), 256, 0, st>>>(sa);
            NB_LAUNCHED();
        }
        {
            ProfScope ps(st, PC_OTHER, 12.0 * (double)px0);
            sod_head_kernel<<<dim3(cdiv(S * S, 256), B), 256, 0, st>>>(sa, reinterpret_cast<const float*>(blob + w.head), saliency);
            NB_LAUNCHED();
        }
    } while (0);
    cudaFreeAsync(ws, st);
    return rc;
}

// ---------------------------------------------------------------------------------------------
// depth_position_from_ratio: one CTA per image
// ---------------------------------------------------------------------------------------------
constexpr int POS_THREADS = 1024;

// k-th smallest (0-based) of keys[0, n) by 4 radix passes of 8 bits
__device__ float select_kth(const uint32_t* keys, int n, int k, uint32_t* hist, uint32_t* sel) {
    uint32_t prefix = 0, mask = 0;
    for (int shift = 24; shift >= 0; shift -= 8) {
        for (int i = threadIdx.x; i < 256; i += POS_THREADS) hist[i] = 0;
        __syncthreads();
        for (int i = threadIdx.x; i < n; i += POS_THREADS) {
            const uint32_t key = keys[i];
            if ((key & mask) == prefix) atomicAdd(&hist[(key >> shift) & 255u], 1u);
        }
        __syncthreads();
        if (threadIdx.x == 0) {
            uint32_t cum = 0, dgt = 255;
            for (uint32_t q = 0; q < 256; ++q) {
                if (cum + hist[q] > (uint32_t)k) { dgt = q; break; }
                cum += hist[q];
            }
            sel[0] = dgt;
            sel[1] = cum;
        }
        __syncthreads();
        prefix |= sel[0] << shift;
        mask |= 255u << shift;
        k -= (int)sel[1];
        __syncthreads();
    }
    return order_key_inv(prefix);
}

// torch.quantile(d, q), linear interpolation: rank = q * (n - 1) in fp32, ATen's lerp (two FMA forms)
__device__ float quantile_sorted(const uint32_t* keys, int n, float q, uint32_t* hist, uint32_t* sel) {
    const float rank = __fmul_rn(q, (float)(n - 1));
    const int rb = (int)rank, ra = (int)ceilf(rank);
    const float wgt = __fsub_rn(rank, (float)rb);
    const float lo = select_kth(keys, n, rb, hist, sel);
    const float hi = ra == rb ? lo : select_kth(keys, n, ra, hist, sel);
    const float diff = __fsub_rn(hi, lo);
    return fabsf(wgt) < 0.5f ? fmaf(wgt, diff, lo) : fmaf(-diff, __fsub_rn(1.f, wgt), hi);
}

__global__ void __launch_bounds__(POS_THREADS) sod_position_kernel(const float* __restrict__ sal, const float* __restrict__ depth,
                                                                   int n, float pos_term, float* __restrict__ out) {
    extern __shared__ uint32_t pos_keys[];   // [n]
    __shared__ uint32_t hist[256], sel[2], cnt;
    const int b = blockIdx.x;
    if (threadIdx.x == 0) cnt = 0;
    __syncthreads();
    const float* s = sal + (size_t)b * n;
    const float* d = depth + (size_t)b * n;
    for (int i = threadIdx.x; i < n; i += POS_THREADS)
        if (__ldg(s + i) > 0.5f) pos_keys[atomicAdd(&cnt, 1u)] = order_key(__ldg(d + i));
    __syncthreads();
    const int m = (int)cnt;
    float r;
    if (m == 0) {
        r = 0.5f;
    } else {
        const float q01 = quantile_sorted(pos_keys, m, 0.1f, hist, sel);
        const float q09 = quantile_sorted(pos_keys, m, 0.9f, hist, sel);
        const float range = __fsub_rn(q09, q01);
        if (range < 1e-6f) {
            r = q01;
        } else {
            const float center = __fmul_rn(__fadd_rn(q01, q09), 0.5f);
            r = __fadd_rn(center, __fmul_rn(pos_term, __fmul_rn(range, 3.0f)));
        }
    }
    if (threadIdx.x == 0) out[b] = fminf(fmaxf(r, 0.f), 1.f);
}

// the EMA of ConvergenceEstimator.__call__ over the batch, in order; state = {ema, has_value}
struct SodResetBits { uint32_t w[32]; };

__global__ void sod_ema_kernel(float* __restrict__ state, const float* __restrict__ z, int B, SodResetBits reset, float decay,
                               float one_minus_decay, float* __restrict__ out) {
    float ema = state[0];
    bool has = state[1] != 0.f;
    for (int i = 0; i < B; ++i) {
        const float p = z[i];
        ema = has ? __fadd_rn(__fmul_rn(decay, ema), __fmul_rn(one_minus_decay, p)) : p;
        has = true;
        out[i] = ema;
        if ((reset.w[i >> 5] >> (i & 31)) & 1u) has = false;
    }
    state[0] = ema;
    state[1] = has ? 1.f : 0.f;
}

}  // namespace nb200

using namespace nb200;

extern "C" int nb200_sod_position(const float* saliency, const float* depth, int B, int n, double pos, float* out, void* stream) {
    NB_CHECK(saliency && depth && out, "null pointer");
    NB_CHECK(B > 0 && n > 0 && n <= 48 * 1024, "n must be in [1, 49152]");
    const size_t smem = (size_t)n * 4;
    if (ensure_dyn_smem((const void*)sod_position_kernel, smem)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope ps(st, PC_OTHER, 0.0, (double)B * n * 8.0, (double)B * 4.0);
    // (pos - 0.5) is a Python float; times the fp32 expanded_range it is rounded to fp32 first
    sod_position_kernel<<<B, POS_THREADS, smem, st>>>(saliency, depth, n, (float)(pos - 0.5), out);
    NB_LAUNCHED();
    return 0;
}

extern "C" int nb200_sod_conv_f16(const void* in, int in_ld, int in_off, int cin, const void* wt, const float* bias, int cout, int dil,
                                  void* out, int out_ld, int out_off, const void* res, int res_ld, int B, int H, int W, void* stream) {
    NB_CHECK(in && wt && bias && out, "null pointer");
    SodConvArgs a;
    a.in = (const __half*)in; a.in_ld = in_ld; a.in_off = in_off; a.cin = cin;
    a.wt = (const __half*)wt; a.bias = bias;
    a.out = (__half*)out; a.out_ld = out_ld; a.out_off = out_off;
    a.res = (const __half*)res; a.res_ld = res_ld; a.res_off = 0;
    a.H = H; a.W = W; a.dil = dil;
    return sod_conv((cudaStream_t)stream, a, cout, B);
}

extern "C" int nb200_sod_ema(float* state, const float* z, int B, const int* reset_host, double decay, float* out, void* stream) {
    NB_CHECK(state && z && out, "null pointer");
    NB_CHECK(B > 0 && B <= 1024, "batch must be in [1, 1024]");
    SodResetBits bits;
    memset(&bits, 0, sizeof(bits));
    if (reset_host)
        for (int i = 0; i < B; ++i)
            if (reset_host[i]) bits.w[i >> 5] |= 1u << (i & 31);
    // decay * ema and (1. - decay) * p: Python floats times fp32 tensors, each rounded to fp32
    sod_ema_kernel<<<1, 1, 0, (cudaStream_t)stream>>>(state, z, B, bits, (float)decay, (float)(1.0 - decay), out);
    NB_LAUNCHED();
    return 0;
}
