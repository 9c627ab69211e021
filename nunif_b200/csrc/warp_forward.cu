// Depth-ordered bilinear forward warp (splat) + hole handling, one CTA per image row.
//
// Replaces iw3/forward_warp.py:140-243 (depth_order_bilinear_forward_warp):
//   global argsort of B*H*W depths + 4 deterministic index_copy_ scatters + iterative
//   shift_fill / fix_layered_holes loops with a host sync per iteration.
//
// Restructuring (DESIGN.md "forward warp"):
//  * every index the reference touches stays inside its row (forward_warp.py:68-72),
//    so a row is an independent unit -> one CTA per (batch, row), state in shared memory.
//  * "scatter in ascending depth order, last writer wins" == "per destination cell the
//    writer with the largest depth wins".  Two writers with equal depth can never hit the
//    same destination cell of the same (floor|ceil) buffer (equal depth => equal shift =>
//    destinations differ by the source distance >= 1), so a shared-memory atomicMax
//    z-buffer on the order-preserving depth key reproduces the sort exactly.
//  * shift_fill (<=100 iterations of 1-px propagation) == "nearest valid cell within 100
//    to the left, else the value 100 cells to the left"; F.pad's zero at the edge is a
//    virtual valid cell holding 0.
//  * fix_layered_holes (<=100 iterations) == "mark where idx[q] > min(idx[q+1..q+100])";
//    the windowed minimum is built by 6 doubling steps in shared memory.
//  The right eye runs the same code on the mirrored row (the reference flips it,
//  forward_warp.py:39-41) with the index negated for the monotonicity test.
//  All fp32 arithmetic that feeds floor()/compare uses non-contracted _rn intrinsics so
//  results are bit-identical to the reference's op-by-op evaluation.
#include "common.cuh"
#include "aa_resize.cuh"
#include "../../include/nunif_b200.h"
#include <math.h>

namespace nb200 {

constexpr int FW_THREADS = 256;
constexpr int FW_MAX_TRIES = 100;  // forward_warp.py:18,45

struct FwParams {
    const float* c;      // [B][3][H][W]
    const float* depth;  // [B][1][h][w]
    float* left;
    float* right;
    float* left_mask;
    float* right_mask;
    int B, H, W, h, w, P, Wp;
    float shift_size;  // divergence*0.01*base*0.5
    float conv_term;   // shift_size*convergence
    const float* conv = nullptr;  // per-frame convergence [B] (nb200_forward_warp_conv): conv_term = fp32(shift_size) * conv[b]
    int fill, do_left, do_right, compose;
    float scale_y, scale_x;  // AA resize scales (h-1)/(H-1), (w-1)/(W-1)
    const float4* coltab;    // per output column: {xmin (as int bits), w0, w1, w2} of the AA resize (upsampling only), or null
};

// ATen upsample_bilinear2d_aa (align_corners=True only changes the scale): one output
// sample at (y, X); horizontal pass first, then vertical (separable, fp32).
__device__ float aa_bilinear_sample(const float* __restrict__ src, int h, int w, float scale_y, float scale_x,
                                    int y, int X) {
    const AaTaps ty = aa_taps(scale_y, y, h), tx = aa_taps(scale_x, X, w);
    return aa_sample(ty, tx, aa_weight_sum(ty), aa_weight_sum(tx),
                     [&](int yy, int xx) { return __ldg(src + (size_t)yy * w + xx); });
}

// Horizontal taps of the AA resize depend only on the output column: computed once per call (upsampling: <= 3 taps).
__global__ void depth_coltab_kernel(float4* __restrict__ tab, int W, int w, float scale_x) {
    const int X = blockIdx.x * blockDim.x + threadIdx.x;
    if (X >= W) return;
    const AaTaps tx = aa_taps(scale_x, X, w);
    float wv[3] = {0.f, 0.f, 0.f}, sum = 0.f;
    for (int j = 0; j < tx.size && j < 3; ++j) { wv[j] = aa_weight(tx, j); sum += wv[j]; }
    tab[X] = make_float4(__int_as_float(tx.min), wv[0] / sum, wv[1] / sum, wv[2] / sum);
}

// same arithmetic as aa_bilinear_sample for the upsampling case, with the horizontal taps taken from the table
__device__ __forceinline__ float aa_bilinear_sample_tab(const float* __restrict__ src, int h, int w, float scale_y, int y,
                                                        const float4 ct) {
    const AaTaps ty = aa_taps(scale_y, y, h);
    const int xmin = __float_as_int(ct.x);
    const float sum_y = aa_weight_sum(ty);
    float acc = 0.f;
    for (int i = 0; i < ty.size; ++i) {
        const float* row = src + (size_t)(ty.min + i) * w + xmin;
        float hs = __ldg(row) * ct.y;
        if (xmin + 1 < w) hs += __ldg(row + 1) * ct.z;
        if (xmin + 2 < w) hs += __ldg(row + 2) * ct.w;
        acc += hs * (aa_weight(ty, i) / sum_y);
    }
    return acc;
}

// Full-resolution depth via the AA resize (used when the caller wants the resized
// depth materialised, e.g. tests of the resize alone).
__global__ void depth_resize_aa_kernel(const float* __restrict__ depth, float* __restrict__ out, int B, int H, int W,
                                       int h, int w, float scale_y, float scale_x) {
    int X = blockIdx.x * blockDim.x + threadIdx.x;
    int y = blockIdx.y, b = blockIdx.z;
    if (X >= W) return;
    out[((size_t)b * H + y) * W + X] = aa_bilinear_sample(depth + (size_t)b * h * w, h, w, scale_y, scale_x, y, X);
}

__global__ void __launch_bounds__(FW_THREADS) forward_warp_row_kernel(FwParams p) {
    extern __shared__ __align__(16) unsigned char smem_raw[];
    const int Wp = p.Wp, W = p.W, P = p.P;
    // 7 row arrays of Wp 32-bit cells
    float* DEP = reinterpret_cast<float*>(smem_raw);              // padded depth row (kept for both eyes)
    float* IDF = DEP + Wp;                                        // filled x-index, LOGICAL order
    unsigned* ZF = reinterpret_cast<unsigned*>(IDF + Wp);         // floor z-buffer -> raw x-index -> scratch
    unsigned* ZC = ZF + Wp;                                       // ceil  z-buffer -> r
    int* SF = reinterpret_cast<int*>(ZC + Wp);                    // floor winner   -> g
    int* SC = SF + Wp;                                            // ceil  winner   -> b
    float* SCR = reinterpret_cast<float*>(SC + Wp);               // scratch (windowed min)
    const int y = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const size_t plane = (size_t)p.H * W;
    const float* __restrict__ crow = p.c + ((size_t)b * 3 * p.H + y) * W;
    const bool same = (p.h == p.H) && (p.w == W);
    const float INF = __int_as_float(0x7f800000);

    // ---- step 0: padded depth row (resize :146-148 fused, replicate pad :159-162)
    {
        const float* dsrc = p.depth + (size_t)b * p.h * p.w;
        for (int X = tid; X < W; X += FW_THREADS)
            DEP[X + P] = same ? dsrc[(size_t)y * W + X]
                              : (p.coltab ? aa_bilinear_sample_tab(dsrc, p.h, p.w, p.scale_y, y, __ldg(p.coltab + X))
                                          : aa_bilinear_sample(dsrc, p.h, p.w, p.scale_y, p.scale_x, y, X));
        __syncthreads();
        for (int t = tid; t < P; t += FW_THREADS) {
            DEP[t] = DEP[P];
            DEP[P + W + t] = DEP[P + W - 1];
        }
        __syncthreads();
    }

    // a convergence tensor makes shift_size * convergence an fp32 tensor op (forward_warp.py:167)
    const float conv_term = p.conv ? __fmul_rn(p.shift_size, __ldg(p.conv + b)) : p.conv_term;
    for (int eye = 0; eye < 2; ++eye) {
        if (eye == 0 ? !p.do_left : !p.do_right) continue;
        const float sg = eye == 0 ? 1.f : -1.f;  // left: +index_shift, right: -index_shift (:176-177)

        for (int xp = tid; xp < Wp; xp += FW_THREADS) {
            ZF[xp] = 0u;
            ZC[xp] = 0u;
            SF[xp] = -1;
            SC[xp] = -1;
        }
        __syncthreads();
        // ---- pass 1: z-buffer -- make_bilinear_data :75-85 + ordered_index_copy :88-110
        for (int xp = tid; xp < Wp; xp += FW_THREADS) {
            float d = DEP[xp];
            float is = __fsub_rn(__fmul_rn(d, p.shift_size), conv_term);
            float fi = fminf(fmaxf(__fadd_rn((float)xp, sg * is), 0.f), (float)(Wp - 1));
            int fl = (int)floorf(fi), ce = (int)ceilf(fi);
            unsigned key = order_key(d);
            atomicMax(&ZF[fl], key);
            atomicMax(&ZC[ce], key);
        }
        __syncthreads();
        // ---- pass 2: winners (unique per visible cell, see header)
        for (int xp = tid; xp < Wp; xp += FW_THREADS) {
            float d = DEP[xp];
            float is = __fsub_rn(__fmul_rn(d, p.shift_size), conv_term);
            float fi = fminf(fmaxf(__fadd_rn((float)xp, sg * is), 0.f), (float)(Wp - 1));
            int fl = (int)floorf(fi), ce = (int)ceilf(fi);
            unsigned key = order_key(d);
            if (ZF[fl] == key) SF[fl] = xp;
            if (ZC[ce] == key) SC[ce] = xp;
        }
        __syncthreads();
        // ---- resolve each visible destination (:129-130, unpad :180-183).
        // Results overwrite this thread's own z/s cells (owner-only access => no hazard).
        for (int X = tid; X < W; X += FW_THREADS) {
            const int xd = X + P;
            const int a = SF[xd], cidx = SC[xd];
            float Fw = 0.f, Cw = 0.f, Fv[4] = {-1.f, -1.f, -1.f, -1.f}, Cv[4] = {-1.f, -1.f, -1.f, -1.f};
            if (a >= 0) {
                float d = DEP[a];
                float is = __fsub_rn(__fmul_rn(d, p.shift_size), conv_term);
                float fi = fminf(fmaxf(__fadd_rn((float)a, sg * is), 0.f), (float)(Wp - 1));
                float cw = fminf(fmaxf(__fsub_rn(fi, floorf(fi)), (float)1e-5), (float)(1.0 - 1e-5));
                Fw = __fsub_rn(1.0f, cw);
                int sx = min(max(a - P, 0), W - 1);
                Fv[0] = __ldg(crow + sx);
                Fv[1] = __ldg(crow + plane + sx);
                Fv[2] = __ldg(crow + 2 * plane + sx);
                Fv[3] = (float)a;
            }
            if (cidx >= 0) {
                float d = DEP[cidx];
                float is = __fsub_rn(__fmul_rn(d, p.shift_size), conv_term);
                float fi = fminf(fmaxf(__fadd_rn((float)cidx, sg * is), 0.f), (float)(Wp - 1));
                Cw = fminf(fmaxf(__fsub_rn(fi, floorf(fi)), (float)1e-5), (float)(1.0 - 1e-5));
                int sx = min(max(cidx - P, 0), W - 1);
                Cv[0] = __ldg(crow + sx);
                Cv[1] = __ldg(crow + plane + sx);
                Cv[2] = __ldg(crow + 2 * plane + sx);
                Cv[3] = (float)cidx;
            }
            float o[4];
            const float den = __fadd_rn(Fw, Cw);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                float v = __fdiv_rn(__fadd_rn(__fmul_rn(Fv[k], Fw), __fmul_rn(Cv[k], Cw)), den);
                o[k] = (v != v) ? -1.f : v;  // nan_to_num(out, -1) :130
            }
            reinterpret_cast<float*>(ZC)[xd] = o[0];
            reinterpret_cast<float*>(SF)[xd] = o[1];
            reinterpret_cast<float*>(SC)[xd] = o[2];
            reinterpret_cast<float*>(ZF)[xd] = o[3];
        }
        __syncthreads();
        float* IDX = reinterpret_cast<float*>(ZF) + P;  // raw warped x-index, physical X
        float* CR = reinterpret_cast<float*>(ZC) + P;
        float* CG = reinterpret_cast<float*>(SF) + P;
        float* CB = reinterpret_cast<float*>(SC) + P;

#define PHYS(q) (eye == 0 ? (q) : (W - 1 - (q)))
        // ---- shift_fill on the index image (:187 / shift_fill_pack :33-42)
        for (int q = tid; q < W; q += FW_THREADS) {
            float v = IDX[PHYS(q)];
            if (v < 0.f) {
                float r = (q < FW_MAX_TRIES) ? 0.f : IDX[PHYS(q - FW_MAX_TRIES)];
                for (int t = 1; t <= FW_MAX_TRIES && q - t >= 0; ++t) {
                    float u = IDX[PHYS(q - t)];
                    if (u >= 0.f) { r = u; break; }
                }
                v = r;
            }
            IDF[q] = v;
        }
        __syncthreads();
        // ---- fix_layered_holes (:45-59): mark where a[q] > min(a[q+1..q+100]), a = +-idx.
        // Doubling: m_k[q] = min(a[q..q+2^k-1]); ping-pong SCR (even k) <-> MB (odd k, the dead raw-index row).
        {
            float* MA = SCR;
            float* MB = reinterpret_cast<float*>(ZF);
            for (int q = tid; q < W; q += FW_THREADS) MA[q] = (eye == 0 ? IDF[q] : -IDF[q]);
            __syncthreads();
            for (int lvl = 0; lvl < 6; ++lvl) {
                const int off = 1 << lvl;
                const float* src = (lvl & 1) ? MB : MA;
                float* dst = (lvl & 1) ? MA : MB;
                for (int q = tid; q < W; q += FW_THREADS)
                    dst[q] = fminf(src[q], (q + off < W) ? src[q + off] : INF);
                __syncthreads();
            }
            // after 6 levels the result (window 64) is in MA.  q+1..q+100 = [q+1,q+64] U [q+37,q+100]
            for (int q = tid; q < W; q += FW_THREADS) {
                float a = (eye == 0 ? IDF[q] : -IDF[q]);
                float m1 = (q + 1 < W) ? MA[q + 1] : INF;
                float m2 = (q + 37 < W) ? MA[q + 37] : INF;
                if (a > fminf(m1, m2)) {
                    int X = PHYS(q);
                    CR[X] = -2.f;
                    CG[X] = -2.f;
                    CB[X] = -2.f;
                }
            }
            __syncthreads();
        }
        // ---- masks (gen_mask2 :135-137), fill (:195-197) or clamp (:199-201), store
        float* outp = eye == 0 ? p.left : p.right;
        float* maskp = eye == 0 ? p.left_mask : p.right_mask;
        const int ow = (p.compose == NB200_COMPOSE_SBS) ? 2 * W : W;
        const size_t oplane = (size_t)p.H * ow;
        float* orow = (p.compose == NB200_COMPOSE_SBS ? p.left + (eye == 0 ? 0 : W) : outp) + ((size_t)b * 3 * p.H + y) * ow;
        for (int q = tid; q < W; q += FW_THREADS) {
            const int X = PHYS(q);
            float v[3] = {CR[X], CG[X], CB[X]};
            if (maskp) {
                float m = (v[0] == -1.f ? 1.f : 0.f) + (v[0] == -2.f ? 0.5f : 0.f);
                maskp[((size_t)b * p.H + y) * W + X] = fminf(fmaxf(m, 0.f), 1.f);
            }
            const float* chan[3] = {CR, CG, CB};
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                float val = v[k];
                if (p.fill) {
                    if (val < 0.f) {
                        float r = (q < FW_MAX_TRIES) ? 0.f : chan[k][PHYS(q - FW_MAX_TRIES)];
                        for (int t = 1; t <= FW_MAX_TRIES && q - t >= 0; ++t) {
                            float u = chan[k][PHYS(q - t)];
                            if (u >= 0.f) { r = u; break; }
                        }
                        val = r;
                    }
                    if (p.compose == NB200_COMPOSE_SBS) val = clamp01(val);  // iw3/utils.py:469
                } else {
                    val = clamp01(val);
                }
                orow[k * oplane + X] = val;
            }
        }
        __syncthreads();
#undef PHYS
    }
}

// copy of the source image into an eye (synthetic_view left/right returns src_image, :222-243)
__global__ void copy_eye_kernel(const float* __restrict__ c, float* __restrict__ out, int H, int W, int ow, int xoff,
                                size_t total) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    int x = (int)(i % W);
    size_t r = i / W;  // (b*3 + k)*H + y
    out[r * ow + xoff + x] = c[i];
}

}  // namespace nb200

using namespace nb200;

extern "C" size_t nb200_forward_warp_workspace(int B, int H, int W, int h, int w) {
    (void)B;
    // the depth resize is fused into the row kernel; when it upsamples, the per-column taps live in a small table
    return (h != H || w != W) ? (size_t)W * sizeof(float4) : 0;
}

static int forward_warp(const float* c, const float* depth, int B, int H, int W, int h, int w, double divergence,
                        double convergence, const float* conv, int fill, int synthetic_view, int width_base, int compose,
                        float* left, float* right, float* left_mask, float* right_mask, void* workspace, void* stream) {
    NB_CHECK(c && depth && left, "null pointer");
    NB_CHECK(compose == NB200_COMPOSE_NONE || compose == NB200_COMPOSE_SBS, "compose must be NONE or SBS");
    NB_CHECK(compose == NB200_COMPOSE_SBS || right, "right output required");
    NB_CHECK(synthetic_view >= 0 && synthetic_view <= 2, "synthetic_view must be both/left/right");
    FwParams p;
    p.c = c; p.depth = depth; p.left = left; p.right = right; p.left_mask = left_mask; p.right_mask = right_mask;
    p.B = B; p.H = H; p.W = W; p.h = h; p.w = w;
    double div = divergence;
    if (synthetic_view != NB200_VIEW_BOTH) div *= 2;                 // forward_warp.py:149-150
    const double base = width_base ? (double)W : (double)(H > W ? H : W);  // :153-156
    p.P = (int)(base * div * 0.01 + 2);                              // :158
    p.Wp = W + 2 * p.P;
    const double shift_size = div * 0.01 * base * 0.5;               // :166
    p.shift_size = (float)shift_size;
    p.conv_term = (float)(shift_size * convergence);         // :167
    p.conv = conv;
    p.fill = fill;
    p.do_left = synthetic_view != NB200_VIEW_RIGHT;
    p.do_right = synthetic_view != NB200_VIEW_LEFT;
    p.compose = compose;
    p.scale_y = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f;
    p.scale_x = W > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
    p.coltab = nullptr;
    cudaStream_t st0 = (cudaStream_t)stream;
    if ((h != H || w != W) && workspace && p.scale_x < 1.f && p.scale_y < 1.f) {
        p.coltab = reinterpret_cast<const float4*>(workspace);
        depth_coltab_kernel<<<cdiv(W, 256), 256, 0, st0>>>(reinterpret_cast<float4*>(workspace), W, w, p.scale_x);
        NB_LAUNCHED();
    }
    const size_t smem = (size_t)p.Wp * 7 * sizeof(float);
    NB_CHECK(smem <= 227 * 1024, "row (with divergence padding) does not fit shared memory");
    cudaStream_t st = (cudaStream_t)stream;
    NB_CUDA(cudaFuncSetAttribute(forward_warp_row_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
    {
        ProfScope ps(st, PC_WARP_FW, (double)B * H * W * 4 * 9 + (double)B * h * w * 4);
        forward_warp_row_kernel<<<dim3(H, B), FW_THREADS, smem, st>>>(p);
    }
    NB_LAUNCHED();
    if (synthetic_view != NB200_VIEW_BOTH) {
        // the non-synthesised eye is the source image
        size_t total = (size_t)B * 3 * H * W;
        const bool sbs = compose == NB200_COMPOSE_SBS;
        float* dst = synthetic_view == NB200_VIEW_RIGHT ? left : (sbs ? left : right);
        int ow = sbs ? 2 * W : W, xoff = (sbs && synthetic_view == NB200_VIEW_LEFT) ? W : 0;
        copy_eye_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(c, dst, H, W, ow, xoff, total);
        NB_LAUNCHED();
    }
    return 0;
}

extern "C" int nb200_forward_warp(const float* c, const float* depth, int B, int H, int W, int h, int w,
                                  double divergence, double convergence, int fill, int synthetic_view,
                                  int width_base, int compose, float* left, float* right,
                                  float* left_mask, float* right_mask, void* workspace, void* stream) {
    return forward_warp(c, depth, B, H, W, h, w, divergence, convergence, nullptr, fill, synthetic_view, width_base, compose, left,
                        right, left_mask, right_mask, workspace, stream);
}

extern "C" int nb200_forward_warp_conv(const float* c, const float* depth, int B, int H, int W, int h, int w,
                                       double divergence, const float* convergence, int fill, int synthetic_view,
                                       int width_base, int compose, float* left, float* right,
                                       float* left_mask, float* right_mask, void* workspace, void* stream) {
    NB_CHECK(convergence, "null convergence");
    return forward_warp(c, depth, B, H, W, h, w, divergence, 0.0, convergence, fill, synthetic_view, width_base, compose, left,
                        right, left_mask, right_mask, workspace, stream);
}

extern "C" int nb200_depth_resize_aa(const float* depth, int B, int h, int w, int H, int W, float* out, void* stream) {
    NB_CHECK(depth && out, "null pointer");
    float sy = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f, sx = W > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
    depth_resize_aa_kernel<<<dim3(cdiv(W, 128), H, B), 128, 0, (cudaStream_t)stream>>>(depth, out, B, H, W, h, w, sy, sx);
    NB_LAUNCHED();
    return 0;
}
