// Non-GEMM kernels of the CUNet path (NHWC fp16 activations):
//   SE block (nunif/modules/attention.py:38-44): deterministic global average pool,
//   the two 1x1 convs + ReLU + sigmoid on the pooled vector, channel scaling in place;
//   the 3-channel tail convolutions (cunet.py:43 conv_bottom 3x3, :41 deconv 4x4 s2 p3),
//   fused with the cascade's clamp / crop-add (cunet.py:149-163).
#include "common.cuh"
#include "cunet_kernels.h"
#include "ptx.cuh"

namespace nb200 {

// ---- SE: pool ------------------------------------------------------------------------------
// partial[b][chunk][c] = sum over the chunk's pixels; chunks are fixed-size => deterministic.
constexpr int SE_CHUNK = 2048;  // pixels per partial

template <int C>
__global__ void __launch_bounds__(256) se_pool_partial_kernel(const __half* __restrict__ x, float* __restrict__ partial, int HW,
                                                              int nchunks) {
    const int b = blockIdx.y, chunk = blockIdx.x;
    const int p0 = chunk * SE_CHUNK, p1 = min(p0 + SE_CHUNK, HW);
    constexpr int LANES = C / 8;             // threads covering one pixel (8 channels each)
    constexpr int ROWS = 256 / LANES;        // pixels processed per step
    const int lane = threadIdx.x % LANES, row = threadIdx.x / LANES;
    float acc[8] = {0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f, 0.f};
    const __half* xb = x + (size_t)b * HW * C;
    for (int p = p0 + row; p < p1; p += ROWS) {
        const uint4 v = __ldg(reinterpret_cast<const uint4*>(xb + (size_t)p * C + lane * 8));
        const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
        for (int j = 0; j < 4; ++j) {
            const float2 f = __half22float2(h[j]);
            acc[2 * j] += f.x;
            acc[2 * j + 1] += f.y;
        }
    }
    __shared__ float sm[ROWS][C];
#pragma unroll
    for (int j = 0; j < 8; ++j) sm[row][lane * 8 + j] = acc[j];
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += 256) {
        float s = 0.f;
        for (int r = 0; r < ROWS; ++r) s += sm[r][c];
        partial[((size_t)b * nchunks + chunk) * C + c] = s;
    }
}

// ---- SE: finalize pool + fc1 + relu + fc2 + sigmoid -> scale[b][c] ---------------------------
template <int C>
__global__ void se_fc_kernel(const float* __restrict__ partial, int nchunks, int HW, const float* __restrict__ w1,
                             const float* __restrict__ b1, const float* __restrict__ w2, const float* __restrict__ b2,
                             float* __restrict__ scale) {
    constexpr int R = C / 8;
    __shared__ float mean[C];
    __shared__ float hid[R];
    const int b = blockIdx.x;
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float s = 0.f;
        for (int k = 0; k < nchunks; ++k) s += partial[((size_t)b * nchunks + k) * C + c];
        mean[c] = s / (float)HW;
    }
    __syncthreads();
    for (int r = threadIdx.x; r < R; r += blockDim.x) {
        float s = b1[r];
        for (int c = 0; c < C; ++c) s += mean[c] * w1[r * C + c];
        hid[r] = fmaxf(s, 0.f);
    }
    __syncthreads();
    for (int c = threadIdx.x; c < C; c += blockDim.x) {
        float s = b2[c];
        for (int r = 0; r < R; ++r) s += hid[r] * w2[c * R + r];
        scale[(size_t)b * C + c] = 1.f / (1.f + __expf(-s));
    }
}

// ---- SE: x *= scale[b][c] ---------------------------------------------------------------------
__global__ void __launch_bounds__(256) se_scale_kernel(__half* __restrict__ x, const float* __restrict__ scale, int C, size_t HW,
                                                       size_t total_vec) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total_vec) return;
    const int vpp = C / 8;
    const size_t pix = i / vpp;
    const int c0 = (int)(i % vpp) * 8;
    const size_t b = pix / HW;
    uint4 v = reinterpret_cast<uint4*>(x)[i];
    __half2* h = reinterpret_cast<__half2*>(&v);
    const float* s = scale + b * C + c0;
#pragma unroll
    for (int j = 0; j < 4; ++j) {
        float2 f = __half22float2(h[j]);
        h[j] = __floats2half2_rn(f.x * s[2 * j], f.y * s[2 * j + 1]);
    }
    reinterpret_cast<uint4*>(x)[i] = v;
}

int se_block(cudaStream_t st, __half* x, int n, int H, int W, int C, const float* w1, const float* b1, const float* w2,
             const float* b2, float* partial, float* scale) {
    if (rec_on(REC_CONV)) rec_launch("se", {{"n", n}, {"H", H}, {"W", W}, {"C", C}});
    const int HW = H * W, nchunks = cdiv(HW, SE_CHUNK);
    ProfScope ps(st, PC_SE, (double)n * HW * C * 2 * 3);
    if (C == 64) {
        se_pool_partial_kernel<64><<<dim3(nchunks, n), 256, 0, st>>>(x, partial, HW, nchunks);
        NB_LAUNCHED();
        se_fc_kernel<64><<<n, 64, 0, st>>>(partial, nchunks, HW, w1, b1, w2, b2, scale);
    } else if (C == 128) {
        se_pool_partial_kernel<128><<<dim3(nchunks, n), 256, 0, st>>>(x, partial, HW, nchunks);
        NB_LAUNCHED();
        se_fc_kernel<128><<<n, 128, 0, st>>>(partial, nchunks, HW, w1, b1, w2, b2, scale);
    } else {
        return fail("se_block: unsupported channel count");
    }
    NB_LAUNCHED();
    const size_t total_vec = (size_t)n * HW * (C / 8);
    se_scale_kernel<<<(unsigned)cdiv64(total_vec, 256), 256, 0, st>>>(x, scale, C, (size_t)HW, total_vec);
    NB_LAUNCHED();
    return 0;
}

size_t se_partial_floats(int n, int H, int W, int C) { return (size_t)n * cdiv(H * W, SE_CHUNK) * C; }

// ---- 3-channel tails --------------------------------------------------------------------------
// MODE 0: conv 3x3 valid 64->3 ; MODE 1: ConvTranspose 4x4 s2 p3 64->3
// EPI 0: out = NHWC8 fp16 (3 ch + 5 zeros), optional clamp(0,1)   (z1 feeding unet2, cunet.py:150-153)
// EPI 1: out = planar fp16 z [n][3][Ho][Wo] = clamp(acc + z1[crop 20])  (cunet.py:154-163)
template <int MODE, int EPI>
__global__ void __launch_bounds__(128) tail_conv_kernel(const __half* __restrict__ x, const float* __restrict__ wt,
                                                        const float* __restrict__ bias, __half* __restrict__ out,
                                                        const __half* __restrict__ z1, int n, int Hi, int Wi, int Ho, int Wo,
                                                        int z1H, int z1W, int clip) {
    constexpr int TAPS = MODE == 0 ? 9 : 16;
    __shared__ __align__(16) float sw[TAPS * 64 * 3];  // [tap][ci][co]
    for (int i = threadIdx.x; i < TAPS * 64 * 3; i += blockDim.x) sw[i] = wt[i];
    __syncthreads();
    const size_t total = (size_t)n * Ho * Wo;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int ox = (int)(i % Wo), oy = (int)((i / Wo) % Ho), b = (int)(i / ((size_t)Wo * Ho));
    float acc[3] = {bias[0], bias[1], bias[2]};
    const __half* xb = x + (size_t)b * Hi * Wi * 64;
    if (MODE == 0) {
#pragma unroll 1
        for (int t = 0; t < 9; ++t) {
            const __half* px = xb + ((size_t)(oy + t / 3) * Wi + (ox + t % 3)) * 64;
            const float* w = sw + t * 192;
#pragma unroll
            for (int c8 = 0; c8 < 8; ++c8) {
                const uint4 v = __ldg(reinterpret_cast<const uint4*>(px) + c8);
                const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
                for (int j = 0; j < 4; ++j) {
                    const float2 f = __half22float2(h[j]);
                    const float* w0 = w + (c8 * 8 + 2 * j) * 3;
                    acc[0] += f.x * w0[0] + f.y * w0[3];
                    acc[1] += f.x * w0[1] + f.y * w0[4];
                    acc[2] += f.x * w0[2] + f.y * w0[5];
                }
            }
        }
    } else {
        // oy = 2*iy - 3 + ky  =>  ky parity = (oy+3)&1, iy = (oy + 3 - ky) / 2
        const int py = (oy + 3) & 1, pxp = (ox + 3) & 1;
#pragma unroll 1
        for (int a = 0; a < 2; ++a) {
            const int ky = py + 2 * a, iy = (oy + 3 - ky) >> 1;
            if (iy < 0 || iy >= Hi) continue;
#pragma unroll 1
            for (int c = 0; c < 2; ++c) {
                const int kx = pxp + 2 * c, ix = (ox + 3 - kx) >> 1;
                if (ix < 0 || ix >= Wi) continue;
                const __half* px = xb + ((size_t)iy * Wi + ix) * 64;
                const float* w = sw + (ky * 4 + kx) * 192;
#pragma unroll
                for (int c8 = 0; c8 < 8; ++c8) {
                    const uint4 v = __ldg(reinterpret_cast<const uint4*>(px) + c8);
                    const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
                    for (int j = 0; j < 4; ++j) {
                        const float2 f = __half22float2(h[j]);
                        const float* w0 = w + (c8 * 8 + 2 * j) * 3;
                        acc[0] += f.x * w0[0] + f.y * w0[3];
                        acc[1] += f.x * w0[1] + f.y * w0[4];
                        acc[2] += f.x * w0[2] + f.y * w0[5];
                    }
                }
            }
        }
    }
    if (EPI == 0) {
        __align__(16) __half o[8];
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            float v = acc[k];
            if (clip) v = clamp01(v);
            o[k] = __float2half_rn(v);
        }
#pragma unroll
        for (int k = 3; k < 8; ++k) o[k] = __float2half_rn(0.f);
        reinterpret_cast<uint4*>(out)[i] = *reinterpret_cast<const uint4*>(o);
    } else {
        const __half* zp = z1 + (((size_t)b * z1H + oy + 20) * z1W + ox + 20) * 8;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float v = acc[k] + __half2float(zp[k]);
            out[(((size_t)b * 3 + k) * Ho + oy) * Wo + ox] = __float2half_rn(clamp01(v));
        }
    }
}

// Tensor-core version of the tails (production path).  The 3 output channels are padded to the n=8 of
// mma.sync.m16n8k16; a warp owns 16 output pixels (for the ConvTranspose: 16 pixels of one column parity, so that all
// rows of the MMA share the same 2x2 subset of the 4x4 taps).  The block first stages its input window in shared memory
// (zero-filled outside the image; pixel stride 144 B so that fragment loads are bank-conflict free) - without that every
// tap re-reads its 128-byte pixel from L2 and the kernel is L2-bandwidth bound (0.8 ms per launch; same for the SIMT
// kernel above, kept as fallback / cross-check).  Weights are staged as fp16 B fragments (the reference runs these convs
// in fp16 under autocast as well).
//   MODE 0 (conv 3x3):        block = 2 output rows x 64 columns, window 4 x 66 pixels
//   MODE 1 (ConvT 4x4 s2 p3): block = 1 output row x 128 columns (64 per parity), window 2 x 66 pixels
constexpr int TC_PS = 72;        // halves per staged pixel (64 channels + 8 pad)
constexpr int TC_WC = 66;        // staged window columns
template <int MODE, int EPI>
__global__ void __launch_bounds__(256) tail_conv_mma_kernel(const __half* __restrict__ x, const float* __restrict__ wt,
                                                            const float* __restrict__ bias, __half* __restrict__ out,
                                                            const __half* __restrict__ z1, int Hi, int Wi, int Ho, int Wo,
                                                            int z1H, int z1W, int clip) {
    constexpr int TAPS = MODE == 0 ? 9 : 16;
    constexpr int WR = MODE == 0 ? 4 : 2;                        // staged window rows
    extern __shared__ __align__(16) unsigned char tc_smem[];
    __half* sB = reinterpret_cast<__half*>(tc_smem);             // [tap][kc][n (8)][16 halves]; rows n >= 3 are zero
    __half* sX = sB + TAPS * 512;                                // [WR][66][72]
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
    const int b = blockIdx.z;
    // block origin in output and input space
    const int j0 = blockIdx.x * 64;                              // first output column (MODE 1: first index within a parity)
    const int oy0 = MODE == 0 ? blockIdx.y * 2 : blockIdx.y;
    int iy0, ix0;
    if (MODE == 0) { iy0 = oy0; ix0 = j0; }
    else {
        // oy = 2*iy - 3 + ky: the two rows that feed output row oy are iy_lo, iy_lo + 1 with iy_lo = (oy + 3 - ky_hi) / 2
        const int ky_hi = ((oy0 + 3) & 1) + 2;
        iy0 = (oy0 + 3 - ky_hi) >> 1;                            // may be -1 at the top edge (zero-filled)
        ix0 = j0;                                                // columns j0 .. j0 + 65 (see tap table below)
    }
    {   // fp16 B fragments are stored right behind the fp32 [tap][ci][co] array (cunet_model.cu pack_tail)
        const uint4* frag = reinterpret_cast<const uint4*>(wt + TAPS * 192);
        for (int i = tid; i < TAPS * 64; i += 256) reinterpret_cast<uint4*>(sB)[i] = __ldg(frag + i);
    }
    const __half* xb = x + (size_t)b * Hi * Wi * 64;
    for (int i = tid; i < WR * TC_WC * 8; i += 256) {
        const int c8 = i & 7, col = (i >> 3) % TC_WC, r = (i >> 3) / TC_WC;
        const int iy = iy0 + r, ix = ix0 + col;
        uint4 v = make_uint4(0, 0, 0, 0);
        if (iy >= 0 && iy < Hi && ix >= 0 && ix < Wi) v = __ldg(reinterpret_cast<const uint4*>(xb + ((size_t)iy * Wi + ix) * 64) + c8);
        *reinterpret_cast<uint4*>(sX + (r * TC_WC + col) * TC_PS + c8 * 8) = v;
    }
    __syncthreads();
    // this warp's 16 pixels
    const int lrow = MODE == 0 ? warp >> 2 : 0;                  // local output row
    const int par = MODE == 1 ? warp >> 2 : 0;                   // column parity class
    const int lj = (warp & 3) * 16;                              // first local column index
    const int oy = oy0 + lrow;
    const int npx = MODE == 1 ? Wo / 2 : Wo;
    if (oy >= Ho || j0 + lj >= npx) return;
    float acc[4] = {0.f, 0.f, 0.f, 0.f};
    constexpr int NT = MODE == 0 ? 9 : 4;
#pragma unroll 1
    for (int tt = 0; tt < NT; ++tt) {
        int tap, dr, dc;
        if (MODE == 0) { tap = tt; dr = lrow + tt / 3; dc = tt % 3; }
        else {
            // ky has the parity of oy+3, kx that of ox+3 (cunet.py:41 ConvTranspose2d(64, 3, 4, 2, 3));
            // ix = (2j + par + 3 - kx) / 2 = j + (par + 3 - kx) / 2
            const int ky = ((oy + 3) & 1) + 2 * (tt >> 1), kx = ((par + 3) & 1) + 2 * (tt & 1);
            tap = ky * 4 + kx;
            dr = ((oy + 3 - ky) >> 1) - iy0;
            dc = (par + 3 - kx) >> 1;
        }
        const __half* p0 = sX + (dr * TC_WC + lj + g + dc) * TC_PS + 2 * t4;
        const __half* p1 = p0 + 8 * TC_PS;
        const __half* wb = sB + tap * 512 + g * 16 + 2 * t4;
#pragma unroll
        for (int kc = 0; kc < 4; ++kc) {
            const uint32_t a[4] = {*reinterpret_cast<const uint32_t*>(p0 + kc * 16), *reinterpret_cast<const uint32_t*>(p1 + kc * 16),
                                   *reinterpret_cast<const uint32_t*>(p0 + kc * 16 + 8), *reinterpret_cast<const uint32_t*>(p1 + kc * 16 + 8)};
            mma16816(acc, a, *reinterpret_cast<const uint32_t*>(wb + kc * 128), *reinterpret_cast<const uint32_t*>(wb + kc * 128 + 8));
        }
    }
    // accumulator layout: acc[0..1] = row g, channels 2*t4, 2*t4+1; acc[2..3] = row g+8.  Channels 0,1 live in t4 == 0,
    // channel 2 in t4 == 1; gather the three into the t4 == 0 lane of each row.
    const float c2a = __shfl_down_sync(0xffffffffu, acc[0], 1), c2b = __shfl_down_sync(0xffffffffu, acc[2], 1);
    if (t4 != 0) return;
    const float bv[3] = {bias[0], bias[1], bias[2]};
#pragma unroll
    for (int r = 0; r < 2; ++r) {
        const int j = j0 + lj + g + 8 * r;
        if (j >= npx) continue;
        const int ox = MODE == 1 ? 2 * j + par : j;
        float v[3] = {(r ? acc[2] : acc[0]) + bv[0], (r ? acc[3] : acc[1]) + bv[1], (r ? c2b : c2a) + bv[2]};
        const size_t pix = ((size_t)b * Ho + oy) * Wo + ox;
        if (EPI == 0) {
            __align__(16) __half o[8];
#pragma unroll
            for (int k = 0; k < 3; ++k) o[k] = __float2half_rn(clip ? clamp01(v[k]) : v[k]);
#pragma unroll
            for (int k = 3; k < 8; ++k) o[k] = __float2half_rn(0.f);
            reinterpret_cast<uint4*>(out)[pix] = *reinterpret_cast<const uint4*>(o);
        } else {
            const __half* zp = z1 + (((size_t)b * z1H + oy + 20) * z1W + ox + 20) * 8;
#pragma unroll
            for (int k = 0; k < 3; ++k)
                out[(((size_t)b * 3 + k) * Ho + oy) * Wo + ox] = __float2half_rn(clamp01(v[k] + __half2float(zp[k])));
        }
    }
}

template <int MODE, int EPI>
static int launch_tail_mma(cudaStream_t st, const __half* x, const float* wt, const float* bias, __half* out, const __half* z1, int n,
                           int Hi, int Wi, int Ho, int Wo, int z1H, int z1W, int clip) {
    constexpr int TAPS = MODE == 0 ? 9 : 16, WR = MODE == 0 ? 4 : 2;
    const size_t smem = (size_t)(TAPS * 512 + WR * TC_WC * TC_PS) * sizeof(__half);
    if (ensure_dyn_smem((const void*)tail_conv_mma_kernel<MODE, EPI>, smem)) return 1;
    const int npx = MODE == 1 ? Wo / 2 : Wo;
    const dim3 grid(cdiv(npx, 64), MODE == 0 ? cdiv(Ho, 2) : Ho, n);
    tail_conv_mma_kernel<MODE, EPI><<<grid, 256, smem, st>>>(x, wt, bias, out, z1, Hi, Wi, Ho, Wo, z1H, z1W, clip);
    return 0;
}

extern int g_tune[16];  // gemm.cu; [7] != 0 selects the SIMT tail kernel (tests)

int tail_conv(cudaStream_t st, int mode, int epi, const __half* x, const float* wt, const float* bias, __half* out,
              const __half* z1, int n, int Hi, int Wi, int z1H, int z1W, int clip) {
    const int Ho = mode == 0 ? Hi - 2 : 2 * Hi - 4, Wo = mode == 0 ? Wi - 2 : 2 * Wi - 4;
    const size_t total = (size_t)n * Ho * Wo;
    const unsigned blocks = (unsigned)cdiv64(total, 128);
    const bool mma = g_tune[7] == 0 && (mode == 0 || Wo % 2 == 0) && n <= 65535;
    if (rec_on(REC_CONV))
        rec_launch("tail", {{"mode", mode}, {"epi", epi}, {"n", n}, {"Hi", Hi}, {"Wi", Wi}, {"z1H", z1H}, {"z1W", z1W},
                            {"clip", clip}, {"path", mma ? 0 : 1}});
    ProfScope ps(st, PC_TAIL, (double)n * Hi * Wi * 128 + (double)total * 16);
    if (mma) {
        int rc;
        if (mode == 0 && epi == 0) rc = launch_tail_mma<0, 0>(st, x, wt, bias, out, z1, n, Hi, Wi, Ho, Wo, z1H, z1W, clip);
        else if (mode == 0 && epi == 1) rc = launch_tail_mma<0, 1>(st, x, wt, bias, out, z1, n, Hi, Wi, Ho, Wo, z1H, z1W, clip);
        else if (mode == 1 && epi == 0) rc = launch_tail_mma<1, 0>(st, x, wt, bias, out, z1, n, Hi, Wi, Ho, Wo, z1H, z1W, clip);
        else return fail("tail_conv: unsupported mode");
        if (rc) return rc;
        NB_LAUNCHED();
        return 0;
    }
    if (mode == 0 && epi == 0) tail_conv_kernel<0, 0><<<blocks, 128, 0, st>>>(x, wt, bias, out, z1, n, Hi, Wi, Ho, Wo, z1H, z1W, clip);
    else if (mode == 0 && epi == 1) tail_conv_kernel<0, 1><<<blocks, 128, 0, st>>>(x, wt, bias, out, z1, n, Hi, Wi, Ho, Wo, z1H, z1W, clip);
    else if (mode == 1 && epi == 0) tail_conv_kernel<1, 0><<<blocks, 128, 0, st>>>(x, wt, bias, out, z1, n, Hi, Wi, Ho, Wo, z1H, z1W, clip);
    else return fail("tail_conv: unsupported mode");
    NB_LAUNCHED();
    return 0;
}

}  // namespace nb200
