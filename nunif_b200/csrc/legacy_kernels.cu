// Output heads of the plain conv stacks waifu2x.upconv_7 / waifu2x.vgg_7 (waifu2x/models/upconv_7.py, vgg_7.py):
//   MODE 0: Conv2d(CIN, 3, 3) valid                  (vgg_7 net.12, CIN = 128)
//   MODE 1: ConvTranspose2d(CIN, 3, 4, stride 2, pad 3) (upconv_7 net.12, CIN = 256)
// each fused with bias + clamp(0, 1) (the eval-mode forward) and the store of the planar fp16 tile z [n][3][Ho][Wo] that the
// seam gather reads.  Input: NHWC fp16 with a dense channel dimension of CIN.
//
// These are separate kernels from CUNet's tail_conv_mma_kernel (cunet_kernels.cu), which stages all 64 input channels of its
// window at once: 256 channels that way would need ~134 KB of shared memory per CTA.  Here the CIN channels are streamed in
// 64-channel chunks (window + that chunk's weight fragments) through a two-stage cp.async pipeline, so the CTA's footprint
// does not grow with CIN, and the fp32 accumulators carry across chunks.
#include "common.cuh"
#include "legacy_kernels.h"
#include "ptx.cuh"

namespace nb200 {

extern int g_tune[16];  // gemm.cu; [7] != 0 selects the SIMT kernels (tests)

// ---- SIMT version (cross-check, g_tune[7]): one thread per output pixel, fp32 weights [tap][ci][co] read through L1 ------
template <int MODE, int CIN>
__global__ void __launch_bounds__(128) head_conv_kernel(const __half* __restrict__ x, const float* __restrict__ wt,
                                                        const float* __restrict__ bias, __half* __restrict__ out, int n, int Hi,
                                                        int Wi, int Ho, int Wo) {
    const size_t total = (size_t)n * Ho * Wo;
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int ox = (int)(i % Wo), oy = (int)((i / Wo) % Ho), b = (int)(i / ((size_t)Wo * Ho));
    float acc[3] = {bias[0], bias[1], bias[2]};
    const __half* xb = x + (size_t)b * Hi * Wi * CIN;
    auto tap = [&](const __half* px, const float* w) {
#pragma unroll 4
        for (int c8 = 0; c8 < CIN / 8; ++c8) {
            const uint4 v = __ldg(reinterpret_cast<const uint4*>(px) + c8);
            const __half2* h = reinterpret_cast<const __half2*>(&v);
#pragma unroll
            for (int j = 0; j < 4; ++j) {
                const float2 f = __half22float2(h[j]);
                const float* w0 = w + (c8 * 8 + 2 * j) * 3;
                acc[0] += f.x * __ldg(w0 + 0) + f.y * __ldg(w0 + 3);
                acc[1] += f.x * __ldg(w0 + 1) + f.y * __ldg(w0 + 4);
                acc[2] += f.x * __ldg(w0 + 2) + f.y * __ldg(w0 + 5);
            }
        }
    };
    if (MODE == 0) {
#pragma unroll 1
        for (int t = 0; t < 9; ++t) tap(xb + ((size_t)(oy + t / 3) * Wi + (ox + t % 3)) * CIN, wt + t * CIN * 3);
    } else {
        // oy = 2*iy - 3 + ky  =>  ky has the parity of oy + 3, iy = (oy + 3 - ky) / 2
        const int py = (oy + 3) & 1, pxp = (ox + 3) & 1;
#pragma unroll 1
        for (int a = 0; a < 2; ++a) {
            const int ky = py + 2 * a, iy = (oy + 3 - ky) >> 1;
            if (iy < 0 || iy >= Hi) continue;
#pragma unroll 1
            for (int c = 0; c < 2; ++c) {
                const int kx = pxp + 2 * c, ix = (ox + 3 - kx) >> 1;
                if (ix < 0 || ix >= Wi) continue;
                tap(xb + ((size_t)iy * Wi + ix) * CIN, wt + (ky * 4 + kx) * CIN * 3);
            }
        }
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) out[(((size_t)b * 3 + k) * Ho + oy) * Wo + ox] = __float2half_rn(clamp01(acc[k]));
}

// ---- tensor-core version (production path) ---------------------------------------------------------------------------
// mma.sync.m16n8k16 with the 3 output channels padded to n = 8; a warp owns 16 output pixels of one row (for MODE 1: of one
// column parity, so that all 16 rows of the MMA share the same 2x2 subset of the 4x4 taps).
//   MODE 0: CTA = 2 output rows x 64 columns, window 4 x 66 input pixels; warp w: row w / 4, columns (w % 4) * 16 ...
//   MODE 1: CTA = output rows 2m+1 and 2m+2 x 128 columns (64 per parity); both rows read the same two input rows m+1, m+2
//           (oy odd: ky in {0, 2}, iy = (oy + 3 - ky) / 2 = m+2, m+1; oy even: ky in {1, 3}, iy = m+2, m+1), so every A
//           fragment feeds two MMAs, one per output row.  Window 2 x 66; warp w: parity w / 4, columns (w % 4) * 16 ...
// Per 64-channel chunk a stage holds the window [WR][66][72 halves] (pixel stride 144 B: conflict-free fragment loads) and
// the chunk's B fragments [tap][kc (4)][n (8)][16].
constexpr int HD_PS = 72;   // halves per staged pixel (64 channels + 8 pad)
constexpr int HD_WC = 66;   // staged window columns

template <int MODE>
struct HeadCfg {
    static constexpr int TAPS = MODE == 0 ? 9 : 16;
    static constexpr int WR = MODE == 0 ? 4 : 2;
    static constexpr int W_HALVES = TAPS * 512;                 // B fragments of one chunk
    static constexpr int X_HALVES = WR * HD_WC * HD_PS;         // window of one chunk
    static constexpr int STAGE_HALVES = W_HALVES + X_HALVES;
    static constexpr size_t SMEM = (size_t)2 * STAGE_HALVES * sizeof(__half);
};

template <int MODE, int CIN>
__global__ void __launch_bounds__(256) head_conv_mma_kernel(const __half* __restrict__ x, const __half* __restrict__ frag,
                                                            const float* __restrict__ bias, __half* __restrict__ out, int Hi,
                                                            int Wi, int Ho, int Wo) {
    using Cfg = HeadCfg<MODE>;
    constexpr int NCH = CIN / 64;
    constexpr int ROWS = MODE == 0 ? 1 : 2;                      // output rows per warp
    extern __shared__ __align__(16) unsigned char hd_smem[];
    __half* stage0 = reinterpret_cast<__half*>(hd_smem);
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
    const int b = blockIdx.z;
    const int j0 = blockIdx.x * 64;                              // first output column (MODE 1: first index within a parity)
    const int oy0 = MODE == 0 ? blockIdx.y * 2 : 2 * blockIdx.y - 1;   // MODE 1: may be -1 (that row is not stored)
    const int iy0 = MODE == 0 ? oy0 : blockIdx.y;
    const __half* xb = x + (size_t)b * Hi * Wi * CIN;

    auto load_chunk = [&](int c, __half* st) {
        const uint4* fsrc = reinterpret_cast<const uint4*>(frag + (size_t)c * Cfg::W_HALVES);
        for (int i = tid; i < Cfg::W_HALVES / 8; i += 256) cp_async16(st + i * 8, fsrc + i, 16);
        __half* sx = st + Cfg::W_HALVES;
        for (int i = tid; i < Cfg::WR * HD_WC * 8; i += 256) {
            const int c8 = i & 7, col = (i >> 3) % HD_WC, r = (i >> 3) / HD_WC;
            const int iy = iy0 + r, ix = j0 + col;
            const bool in = iy >= 0 && iy < Hi && ix < Wi;      // outside the image: zero fill (src-size 0)
            const __half* src = in ? xb + ((size_t)iy * Wi + ix) * CIN + c * 64 + c8 * 8 : xb;
            cp_async16(sx + (r * HD_WC + col) * HD_PS + c8 * 8, src, in ? 16 : 0);
        }
        cp_async_commit();
    };

    const int lrow = MODE == 0 ? warp >> 2 : 0;
    const int par = MODE == 1 ? warp >> 2 : 0;
    const int lj = (warp & 3) * 16;
    const int npx = MODE == 1 ? Wo / 2 : Wo;
    float acc[ROWS][4];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) acc[r][0] = acc[r][1] = acc[r][2] = acc[r][3] = 0.f;

    load_chunk(0, stage0);
#pragma unroll 1
    for (int c = 0; c < NCH; ++c) {
        if (c + 1 < NCH) {
            load_chunk(c + 1, stage0 + ((c + 1) & 1) * Cfg::STAGE_HALVES);
            cp_async_wait<1>();
        } else {
            cp_async_wait<0>();
        }
        __syncthreads();
        const __half* sB = stage0 + (c & 1) * Cfg::STAGE_HALVES;
        const __half* sX = sB + Cfg::W_HALVES;
        if (MODE == 0) {
#pragma unroll 1
            for (int t = 0; t < 9; ++t) {
                const __half* p0 = sX + ((lrow + t / 3) * HD_WC + lj + g + t % 3) * HD_PS + 2 * t4;
                const __half* p1 = p0 + 8 * HD_PS;
                const __half* wb = sB + t * 512 + g * 16 + 2 * t4;
#pragma unroll
                for (int kc = 0; kc < 4; ++kc) {
                    const uint32_t a[4] = {*reinterpret_cast<const uint32_t*>(p0 + kc * 16), *reinterpret_cast<const uint32_t*>(p1 + kc * 16),
                                           *reinterpret_cast<const uint32_t*>(p0 + kc * 16 + 8), *reinterpret_cast<const uint32_t*>(p1 + kc * 16 + 8)};
                    mma16816(acc[0], a, *reinterpret_cast<const uint32_t*>(wb + kc * 128), *reinterpret_cast<const uint32_t*>(wb + kc * 128 + 8));
                }
            }
        } else {
            // input pixel (dr, dc) of the window; row r = 0 is the odd output row (ky = 2 - 2 dr), r = 1 the even one
            // (ky = 3 - 2 dr); kx has the parity of par + 3: ix = j + (par + 3 - kx) / 2, so kx = par + 3 - 2 (dc') with
            // dc' in {dc_lo, dc_lo + 1}
            const int kx_hi = ((par + 3) & 1) + 2;               // dc = (par + 3 - kx) / 2
#pragma unroll
            for (int dr = 0; dr < 2; ++dr)
#pragma unroll
                for (int q = 0; q < 2; ++q) {
                    const int kx = kx_hi - 2 * q, dc = (par + 3 - kx) >> 1;
                    const __half* p0 = sX + (dr * HD_WC + lj + g + dc) * HD_PS + 2 * t4;
                    const __half* p1 = p0 + 8 * HD_PS;
                    const __half* wb0 = sB + ((2 - 2 * dr) * 4 + kx) * 512 + g * 16 + 2 * t4;
                    const __half* wb1 = sB + ((3 - 2 * dr) * 4 + kx) * 512 + g * 16 + 2 * t4;
#pragma unroll
                    for (int kc = 0; kc < 4; ++kc) {
                        const uint32_t a[4] = {*reinterpret_cast<const uint32_t*>(p0 + kc * 16), *reinterpret_cast<const uint32_t*>(p1 + kc * 16),
                                               *reinterpret_cast<const uint32_t*>(p0 + kc * 16 + 8),
                                               *reinterpret_cast<const uint32_t*>(p1 + kc * 16 + 8)};
                        mma16816(acc[0], a, *reinterpret_cast<const uint32_t*>(wb0 + kc * 128), *reinterpret_cast<const uint32_t*>(wb0 + kc * 128 + 8));
                        mma16816(acc[ROWS - 1], a, *reinterpret_cast<const uint32_t*>(wb1 + kc * 128),
                                 *reinterpret_cast<const uint32_t*>(wb1 + kc * 128 + 8));
                    }
                }
        }
        __syncthreads();   // the next iteration's prefetch overwrites this stage
    }
    // accumulator layout: acc[0..1] = MMA row g, channels 2*t4, 2*t4+1; acc[2..3] = row g+8.  Channels 0, 1 live in t4 == 0,
    // channel 2 in t4 == 1: gather the three into the t4 == 0 lane.
    float c2[ROWS][2];
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
        c2[r][0] = __shfl_down_sync(0xffffffffu, acc[r][0], 1);
        c2[r][1] = __shfl_down_sync(0xffffffffu, acc[r][2], 1);
    }
    if (t4 != 0) return;
    const float bv[3] = {bias[0], bias[1], bias[2]};
#pragma unroll
    for (int r = 0; r < ROWS; ++r) {
        const int oy = oy0 + lrow + r;
        if (oy < 0 || oy >= Ho) continue;
#pragma unroll
        for (int h = 0; h < 2; ++h) {
            const int j = j0 + lj + g + 8 * h;
            if (j >= npx) continue;
            const int ox = MODE == 1 ? 2 * j + par : j;
            const float v[3] = {acc[r][2 * h] + bv[0], acc[r][2 * h + 1] + bv[1], c2[r][h] + bv[2]};
#pragma unroll
            for (int k = 0; k < 3; ++k) out[(((size_t)b * 3 + k) * Ho + oy) * Wo + ox] = __float2half_rn(clamp01(v[k]));
        }
    }
}

template <int MODE, int CIN>
static int launch_head(cudaStream_t st, bool mma, const __half* x, const float* wt, const float* bias, __half* out, int n, int Hi,
                       int Wi, int Ho, int Wo) {
    using Cfg = HeadCfg<MODE>;
    if (mma) {
        if (ensure_dyn_smem((const void*)head_conv_mma_kernel<MODE, CIN>, Cfg::SMEM)) return 1;
        const int npx = MODE == 1 ? Wo / 2 : Wo;
        const dim3 grid(cdiv(npx, 64), MODE == 0 ? cdiv(Ho, 2) : cdiv(Ho + 1, 2), n);
        // fp16 B fragments follow the fp32 [tap][ci][co] array (legacy_model.cu pack_head)
        const __half* frag = reinterpret_cast<const __half*>(wt + (size_t)Cfg::TAPS * CIN * 3);
        head_conv_mma_kernel<MODE, CIN><<<grid, 256, Cfg::SMEM, st>>>(x, frag, bias, out, Hi, Wi, Ho, Wo);
    } else {
        const size_t total = (size_t)n * Ho * Wo;
        head_conv_kernel<MODE, CIN><<<(unsigned)cdiv64(total, 128), 128, 0, st>>>(x, wt, bias, out, n, Hi, Wi, Ho, Wo);
    }
    NB_LAUNCHED();
    return 0;
}

int head_conv(cudaStream_t st, int mode, int cin, const __half* x, const float* wt, const float* bias, __half* out, int n, int Hi,
              int Wi) {
    const int Ho = mode == 0 ? Hi - 2 : 2 * Hi - 4, Wo = mode == 0 ? Wi - 2 : 2 * Wi - 4;
    NB_CHECK(Ho > 0 && Wo > 0, "head_conv: input too small");
    const bool mma = g_tune[7] == 0 && (mode == 0 || Wo % 2 == 0) && n <= 65535;
    if (rec_on(REC_CONV))
        rec_launch("head", {{"mode", mode}, {"cin", cin}, {"n", n}, {"Hi", Hi}, {"Wi", Wi}, {"path", mma ? 0 : 1}});
    const double rbytes = (double)n * Hi * Wi * cin * 2, wbytes = (double)n * Ho * Wo * 3 * 2;
    ProfScope ps(st, PC_TAIL, rbytes + wbytes, rbytes, wbytes);
    if (mode == 0 && cin == 128) return launch_head<0, 128>(st, mma, x, wt, bias, out, n, Hi, Wi, Ho, Wo);
    if (mode == 1 && cin == 256) return launch_head<1, 256>(st, mma, x, wt, bias, out, n, Hi, Wi, Ho, Wo);
    return fail("head_conv: unsupported (mode, input channels)");
}

}  // namespace nb200
