// Backward (grid_sample) stereo warp, fused: disparity from low-res depth ->
// 1-D horizontal bilinear gather -> left/right (or SBS / anaglyph) in one pass.
//
// Replaces iw3/backward_warp.py:67-121 (make_grid + F.interpolate(grid) +
// F.grid_sample x2 + clamp) and optionally iw3/utils.py:466-469 (SBS cat) or
// iw3/anaglyph.py:51-92 (dubois).  HBM-bound: algorithmic traffic is
// 3 planes in + 6 planes out (+ the small depth map); the reference moves two
// full-resolution 2-channel grids on top of that.
//
// Design note (DESIGN.md "backward warp"): the reference's y grid coordinate is
// linspace(-1,1) resampled and un-normalised, i.e. the row index up to fp32
// rounding (|dy| < 1e-4 px).  This kernel samples the row exactly, which turns
// the 2-D gather into a 1-D one; the difference is bounded by 1e-4 * |row delta|.
#include "common.cuh"
#include "../../include/nunif_b200.h"

namespace nb200 {

__device__ __forceinline__ float linspace_m1_1(int j, int n, float step) {
    // torch.linspace(-1, 1, n) fp32 (ATen RangeFactories: symmetric evaluation)
    return (j < n / 2) ? (-1.0f + step * (float)j) : (1.0f - step * (float)(n - j - 1));
}

__device__ __forceinline__ float srgb_to_linear(float x) {
    return (x <= 0.04045f) ? x / 12.92f : powf((x + 0.055f) / 1.055f, 2.4f);
}
__device__ __forceinline__ float linear_to_srgb(float x) {
    return (x <= 0.0031308f) ? x * 12.92f : 1.055f * powf(x, 1.0f / 2.4f) - 0.055f;
}

// a*x + b*y with both products and the sum rounded on their own.  Both backward-warp kernels blend through this, so they
// agree bit for bit whichever product the compiler would otherwise fuse into an FMA.
__device__ __forceinline__ float mix2_rn(float a, float x, float b, float y) { return __fadd_rn(__fmul_rn(a, x), __fmul_rn(b, y)); }

// iw3/anaglyph.py:51-92 for one pixel
__device__ __forceinline__ void dubois_px(const float l[3], const float r[3], bool clip_before, float out[3]) {
    const float lm[3][3] = {{0.437f, 0.449f, 0.164f}, {-0.062f, -0.062f, -0.024f}, {-0.048f, -0.050f, -0.017f}};
    const float rm[3][3] = {{-0.011f, -0.032f, -0.007f}, {0.377f, 0.761f, 0.009f}, {-0.026f, -0.093f, 1.234f}};
    float ll[3], rl[3];
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        ll[k] = srgb_to_linear(l[k]);
        rl[k] = srgb_to_linear(r[k]);
    }
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        float a = ll[0] * lm[k][0] + ll[1] * lm[k][1] + ll[2] * lm[k][2];
        float b = rl[0] * rm[k][0] + rl[1] * rm[k][1] + rl[2] * rm[k][2];
        if (clip_before) {
            a = clamp01(a);
            b = clamp01(b);
        }
        out[k] = clamp01(linear_to_srgb(clamp01(a + b)));
    }
}

struct BwParams {
    const float* c;
    const float* depth;
    float* left;
    float* right;
    int B, H, W, h, w;
    float shift;        // divergence * 0.01 (x2 for single-view synthesis)
    float shift_conv;   // shift * convergence
    float delta_scale;  // max(h, w) / w
    float sy, sx;       // (h-1)/(H-1), (w-1)/(W-1)  align_corners scales (fp32, like ATen)
    float step_x;       // 2/(w-1)
    int warp_left, warp_right;
};

// One thread = VEC consecutive output pixels of one row, both eyes, 3 channels.
template <int COMPOSE, int VEC>
__global__ void __launch_bounds__(256) backward_warp_kernel(BwParams p) {
    const int x0 = (blockIdx.x * blockDim.x + threadIdx.x) * VEC;
    const int y = blockIdx.y;
    const int b = blockIdx.z;
    if (x0 >= p.W) return;

    const float* __restrict__ dep = p.depth + (size_t)b * p.h * p.w;
    const float* __restrict__ crow = p.c + ((size_t)b * 3 * p.H + y) * p.W;
    const size_t plane = (size_t)p.H * p.W;

    // vertical source coordinate in the depth map (align_corners=True bilinear)
    const bool same = (p.h == p.H) && (p.w == p.W);
    int i0 = y, i1 = y;
    float ly1 = 0.f;
    if (!same) {
        float srcy = __fmul_rn(p.sy, (float)y);   // rounded like ATen's h1r (no fma into the lambda below)
        i0 = min((int)srcy, p.h - 1);
        i1 = min(i0 + 1, p.h - 1);
        ly1 = srcy - (float)i0;
    }
    const float ly0 = 1.f - ly1;

    float outl[VEC][3], outr[VEC][3];
#pragma unroll
    for (int v = 0; v < VEC; ++v) {
        const int x = x0 + v;
        float gl, gr;  // normalised grid x of left (-delta) and right (+delta)
        if (x < p.W) {
            if (same) {
                float is = __fsub_rn(__fmul_rn(dep[(size_t)y * p.w + x], p.shift), p.shift_conv);
                float lx = linspace_m1_1(x, p.w, p.step_x);
                // each product and sum rounded on its own, as in the row-staged kernel's grid table (no FMA contraction)
                const float d = __fmul_rn(is, p.delta_scale);
                gl = __fsub_rn(lx, d);
                gr = __fadd_rn(lx, d);
            } else {
                float srcx = __fmul_rn(p.sx, (float)x);
                int j0 = min((int)srcx, p.w - 1);
                int j1 = min(j0 + 1, p.w - 1);
                float lx1 = srcx - (float)j0, lx0 = 1.f - lx1;
                float is00 = __fsub_rn(__fmul_rn(__ldg(dep + (size_t)i0 * p.w + j0), p.shift), p.shift_conv);
                float is01 = __fsub_rn(__fmul_rn(__ldg(dep + (size_t)i0 * p.w + j1), p.shift), p.shift_conv);
                float is10 = __fsub_rn(__fmul_rn(__ldg(dep + (size_t)i1 * p.w + j0), p.shift), p.shift_conv);
                float is11 = __fsub_rn(__fmul_rn(__ldg(dep + (size_t)i1 * p.w + j1), p.shift), p.shift_conv);
                float l0 = linspace_m1_1(j0, p.w, p.step_x), l1 = linspace_m1_1(j1, p.w, p.step_x);
                const float ds = p.delta_scale;
                const float d00 = __fmul_rn(is00, ds), d01 = __fmul_rn(is01, ds), d10 = __fmul_rn(is10, ds), d11 = __fmul_rn(is11, ds);
                gl = mix2_rn(ly0, mix2_rn(lx0, __fsub_rn(l0, d00), lx1, __fsub_rn(l1, d01)),
                             ly1, mix2_rn(lx0, __fsub_rn(l0, d10), lx1, __fsub_rn(l1, d11)));
                gr = mix2_rn(ly0, mix2_rn(lx0, __fadd_rn(l0, d00), lx1, __fadd_rn(l1, d01)),
                             ly1, mix2_rn(lx0, __fadd_rn(l0, d10), lx1, __fadd_rn(l1, d11)));
            }
            const float wm1 = (float)(p.W - 1);
#pragma unroll
            for (int eye = 0; eye < 2; ++eye) {
                float (*o)[3] = eye == 0 ? outl : outr;
                const bool do_warp = eye == 0 ? p.warp_left : p.warp_right;
                if (!do_warp) {
#pragma unroll
                    for (int k = 0; k < 3; ++k) o[v][k] = crow[k * plane + x];
                    continue;
                }
                float g = eye == 0 ? gl : gr;
                float ix = ((g + 1.f) * 0.5f) * wm1;       // grid_sampler_unnormalize (align_corners)
                ix = fminf(wm1, fmaxf(ix, 0.f));           // border padding
                float fx = floorf(ix);
                int xa = (int)fx;
                int xb = min(xa + 1, p.W - 1);
                float wb = ix - fx, wa = (fx + 1.f) - ix;
#pragma unroll
                for (int k = 0; k < 3; ++k) {
                    float va = __ldg(crow + k * plane + xa);
                    float vb = __ldg(crow + k * plane + xb);
                    o[v][k] = clamp01(mix2_rn(va, wa, vb, wb));
                }
            }
        }
    }

    // ---- epilogue: write L/R, SBS halves, or the anaglyph mix
    if (COMPOSE == NB200_COMPOSE_ANAGLYPH_DUBOIS) {
        float* orow = p.left + ((size_t)b * 3 * p.H + y) * p.W;
        float res[VEC][3];
#pragma unroll
        for (int v = 0; v < VEC; ++v) dubois_px(outl[v], outr[v], true, res[v]);
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            if (VEC == 4 && x0 + 3 < p.W && (p.W & 3) == 0) {
                *reinterpret_cast<float4*>(orow + k * plane + x0) = make_float4(res[0][k], res[1][k], res[2][k], res[3][k]);
            } else {
                for (int v = 0; v < VEC; ++v)
                    if (x0 + v < p.W) orow[k * plane + x0 + v] = res[v][k];
            }
        }
        return;
    }
    const int ow = (COMPOSE == NB200_COMPOSE_SBS) ? 2 * p.W : p.W;
    const size_t oplane = (size_t)p.H * ow;
    float* lrow = p.left + ((size_t)b * 3 * p.H + y) * ow;
    float* rrow = (COMPOSE == NB200_COMPOSE_SBS) ? lrow + p.W : p.right + ((size_t)b * 3 * p.H + y) * ow;
#pragma unroll
    for (int k = 0; k < 3; ++k) {
        if (VEC == 4 && x0 + 3 < p.W && (p.W & 3) == 0) {
            *reinterpret_cast<float4*>(lrow + k * oplane + x0) = make_float4(outl[0][k], outl[1][k], outl[2][k], outl[3][k]);
            *reinterpret_cast<float4*>(rrow + k * oplane + x0) = make_float4(outr[0][k], outr[1][k], outr[2][k], outr[3][k]);
        } else {
            for (int v = 0; v < VEC; ++v)
                if (x0 + v < p.W) {
                    lrow[k * oplane + x0 + v] = outl[v][k];
                    rrow[k * oplane + x0 + v] = outr[v][k];
                }
        }
    }
}

// Row-staged variant (the production path): one CTA per (row, batch).  The CTA first stages
//   * the three colour rows in shared memory (coalesced 16 B loads, one replicated pad pixel so tap xa+1 needs
//     no clamp), and
//   * a per-depth-column table {gx_left(i0), gx_right(i0), gx_left(i1), gx_right(i1)} = mesh_x -/+ delta*scale
//     of the two depth rows this output row interpolates between (backward_warp.py:68 evaluated once per
//     depth column instead of once per output pixel),
// then every thread produces 4 consecutive pixels of both eyes from shared memory only.  Against the
// gather-from-global kernel above this removes the 64-bit address arithmetic (30% of its issue slots) and the
// per-pixel depth loads; the kernel is then bounded by its HBM stores.
struct __align__(16) GridTab { float l0, r0, l1, r1; };
constexpr int COMPOSE_RIGHT_ONLY = 3;   // internal: only the "+shift" view, written to p.left (nb200_backward_warp_delta)

// F16_PRODUCT: delta * delta_scale is rounded to fp16 (an fp16 delta, nb200_backward_warp_delta_f16; p.delta_scale is then
// fp16-valued as well).
template <int COMPOSE, bool F16_PRODUCT = false>
__global__ void __launch_bounds__(256) backward_warp_row_kernel(BwParams p, int S, int vec_ok) {
    extern __shared__ __align__(16) unsigned char bw_smem[];
    GridTab* gt = reinterpret_cast<GridTab*>(bw_smem);          // [w + 1]
    float* srow = reinterpret_cast<float*>(gt + (p.w + 1));     // [3][S], S >= W + 1, S % 4 == 0
    const int y = blockIdx.x, b = blockIdx.y, tid = threadIdx.x;
    const size_t plane = (size_t)p.H * p.W;
    const float* __restrict__ crow = p.c + ((size_t)b * 3 * p.H + y) * p.W;
    const float* __restrict__ dep = p.depth + (size_t)b * p.h * p.w;

    const bool same = (p.h == p.H) && (p.w == p.W);
    int i0 = y, i1 = y;
    float ly1 = 0.f;
    if (!same) {
        float srcy = __fmul_rn(p.sy, (float)y);   // rounded like ATen's h1r (no fma into the lambda below)
        i0 = min((int)srcy, p.h - 1);
        i1 = min(i0 + 1, p.h - 1);
        ly1 = srcy - (float)i0;
    }
    const float ly0 = 1.f - ly1;

    if (vec_ok) {
        const int w4 = p.W >> 2;
#pragma unroll
        for (int k = 0; k < 3; ++k) {
            const float4* src = reinterpret_cast<const float4*>(crow + k * plane);
            float4* dst = reinterpret_cast<float4*>(srow + k * S);
            for (int i = tid; i < w4; i += 256) dst[i] = __ldg(src + i);
        }
    } else {
        for (int k = 0; k < 3; ++k)
            for (int i = tid; i < p.W; i += 256) srow[k * S + i] = __ldg(crow + k * plane + i);
    }
    for (int j = tid; j <= p.w; j += 256) {
        const int jj = min(j, p.w - 1);
        const float lx = linspace_m1_1(jj, p.w, p.step_x);
        const float is0 = __fsub_rn(__fmul_rn(__ldg(dep + (size_t)i0 * p.w + jj), p.shift), p.shift_conv);
        const float is1 = __fsub_rn(__fmul_rn(__ldg(dep + (size_t)i1 * p.w + jj), p.shift), p.shift_conv);
        float d0 = __fmul_rn(is0, p.delta_scale), d1 = __fmul_rn(is1, p.delta_scale);
        if (F16_PRODUCT) {
            d0 = __half2float(__float2half_rn(d0));
            d1 = __half2float(__float2half_rn(d1));
        }
        GridTab t;
        t.l0 = __fsub_rn(lx, d0); t.r0 = __fadd_rn(lx, d0);
        t.l1 = __fsub_rn(lx, d1); t.r1 = __fadd_rn(lx, d1);
        gt[j] = t;
    }
    __syncthreads();
    if (tid < 3) srow[tid * S + p.W] = srow[tid * S + p.W - 1];
    __syncthreads();

    const float wm1 = (float)(p.W - 1);
    const int ow = (COMPOSE == NB200_COMPOSE_SBS) ? 2 * p.W : p.W;
    const size_t oplane = (size_t)p.H * ow;
    float* lrow = p.left + ((size_t)b * 3 * p.H + y) * ow;
    float* rrow = (COMPOSE == NB200_COMPOSE_SBS) ? lrow + p.W
                  : (COMPOSE == NB200_COMPOSE_NONE ? p.right + ((size_t)b * 3 * p.H + y) * ow : nullptr);

    for (int x0 = tid * 4; x0 < p.W; x0 += 1024) {
        float outl[4][3], outr[4][3];
#pragma unroll
        for (int v = 0; v < 4; ++v) {
            const int x = min(x0 + v, p.W - 1);
            const float srcx = __fmul_rn(p.sx, (float)x);
            const int j0 = min((int)srcx, p.w - 1);
            const float lx1 = srcx - (float)j0, lx0 = 1.f - lx1;
            const float4 t0 = *reinterpret_cast<const float4*>(gt + j0);
            const float4 t1 = *reinterpret_cast<const float4*>(gt + j0 + 1);
            const float gl = mix2_rn(ly0, mix2_rn(lx0, t0.x, lx1, t1.x), ly1, mix2_rn(lx0, t0.z, lx1, t1.z));
            const float gr = mix2_rn(ly0, mix2_rn(lx0, t0.y, lx1, t1.y), ly1, mix2_rn(lx0, t0.w, lx1, t1.w));
#pragma unroll
            for (int eye = 0; eye < 2; ++eye) {
                float* o = eye == 0 ? outl[v] : outr[v];
                const bool do_warp = eye == 0 ? p.warp_left : p.warp_right;
                if (!do_warp) {
#pragma unroll
                    for (int k = 0; k < 3; ++k) o[k] = srow[k * S + x];
                    continue;
                }
                const float g = eye == 0 ? gl : gr;
                float ix = ((g + 1.f) * 0.5f) * wm1;       // grid_sampler_unnormalize (align_corners)
                ix = fminf(wm1, fmaxf(ix, 0.f));           // border padding
                const float fx = floorf(ix);
                const float wb = ix - fx, wa = (fx + 1.f) - ix;
                const float* sp = srow + (int)fx;
#pragma unroll
                for (int k = 0; k < 3; ++k) o[k] = __saturatef(mix2_rn(sp[k * S], wa, sp[k * S + 1], wb));
            }
        }
        if (COMPOSE == NB200_COMPOSE_ANAGLYPH_DUBOIS) {
            float res[4][3];
#pragma unroll
            for (int v = 0; v < 4; ++v) dubois_px(outl[v], outr[v], true, res[v]);
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                if (vec_ok) {
                    *reinterpret_cast<float4*>(lrow + k * oplane + x0) = make_float4(res[0][k], res[1][k], res[2][k], res[3][k]);
                } else {
                    for (int v = 0; v < 4; ++v)
                        if (x0 + v < p.W) lrow[k * oplane + x0 + v] = res[v][k];
                }
            }
        } else {
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                if (COMPOSE == COMPOSE_RIGHT_ONLY) {   // single warped view (learned-delta warp): the "+delta" eye goes to p.left
                    if (vec_ok) {
                        __stcs(reinterpret_cast<float4*>(lrow + k * oplane + x0), make_float4(outr[0][k], outr[1][k], outr[2][k], outr[3][k]));
                    } else {
                        for (int v = 0; v < 4; ++v)
                            if (x0 + v < p.W) lrow[k * oplane + x0 + v] = outr[v][k];
                    }
                } else if (vec_ok) {
                    __stcs(reinterpret_cast<float4*>(lrow + k * oplane + x0), make_float4(outl[0][k], outl[1][k], outl[2][k], outl[3][k]));
                    __stcs(reinterpret_cast<float4*>(rrow + k * oplane + x0), make_float4(outr[0][k], outr[1][k], outr[2][k], outr[3][k]));
                } else {
                    for (int v = 0; v < 4; ++v)
                        if (x0 + v < p.W) {
                            lrow[k * oplane + x0 + v] = outl[v][k];
                            rrow[k * oplane + x0 + v] = outr[v][k];
                        }
                }
            }
        }
    }
}

extern int g_tune[16];  // gemm.cu; [3] != 0 forces the gather-from-global kernel (tests)

template <int COMPOSE, bool F16_PRODUCT = false>
static int launch_bw_row(const BwParams& p, size_t smem, int S, int vec_ok, cudaStream_t st) {
    if (ensure_dyn_smem((const void*)backward_warp_row_kernel<COMPOSE, F16_PRODUCT>, smem)) return 1;
    backward_warp_row_kernel<COMPOSE, F16_PRODUCT><<<dim3(p.H, p.B), 256, smem, st>>>(p, S, vec_ok);
    return 0;
}

__global__ void __launch_bounds__(256) anaglyph_dubois_kernel(const float* __restrict__ l, const float* __restrict__ r,
                                                               float* __restrict__ out, size_t plane, size_t total,
                                                               int clip_before) {
    size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    size_t b = i / plane, px = i % plane;
    const float* lp = l + b * 3 * plane + px;
    const float* rp = r + b * 3 * plane + px;
    float lv[3] = {lp[0], lp[plane], lp[2 * plane]};
    float rv[3] = {rp[0], rp[plane], rp[2 * plane]};
    float o[3];
    dubois_px(lv, rv, clip_before != 0, o);
    float* op = out + b * 3 * plane + px;
    op[0] = o[0];
    op[plane] = o[1];
    op[2 * plane] = o[2];
}

}  // namespace nb200

using namespace nb200;

extern "C" int nb200_backward_warp(const float* c, const float* depth, int B, int H, int W, int h, int w,
                                   double divergence, double convergence, int synthetic_view, int compose,
                                   float* left, float* right, void* stream) {
    NB_CHECK(c && depth && left, "null pointer");
    NB_CHECK(compose != NB200_COMPOSE_NONE || right, "right output required for compose=NONE");
    NB_CHECK(B > 0 && H > 0 && W > 0 && h > 0 && w > 0, "bad shape");
    NB_CHECK(synthetic_view >= 0 && synthetic_view <= 2, "synthetic_view must be both/left/right");
    BwParams p;
    p.c = c; p.depth = depth; p.left = left; p.right = right;
    p.B = B; p.H = H; p.W = W; p.h = h; p.w = w;
    double div = divergence;
    if (synthetic_view != NB200_VIEW_BOTH) div = div * 2;           // backward_warp.py:101-102
    double shift = div * 0.01;                                       // :105
    p.shift = (float)shift;
    p.shift_conv = (float)(shift * convergence);             // :106
    p.delta_scale = (float)((double)(h > w ? h : w) / (double)w);    // :108
    p.sy = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f;
    p.sx = W > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
    p.step_x = w > 1 ? 2.0f / (float)(w - 1) : 0.f;
    p.warp_left = synthetic_view != NB200_VIEW_RIGHT;
    p.warp_right = synthetic_view != NB200_VIEW_LEFT;
    constexpr int VEC = 4;
    dim3 block(256), grid(cdiv(cdiv(W, VEC), 256), H, B);
    cudaStream_t st = (cudaStream_t)stream;
    // algorithmic bytes: 3 planes in + output planes + the depth map (SURVEY.md 8d)
    ProfScope ps(st, PC_WARP_BW, (double)B * H * W * 4 * (3 + (compose == NB200_COMPOSE_ANAGLYPH_DUBOIS ? 3 : 6)) + (double)B * h * w * 4);
    const int S = (W + 1 + 3) & ~3;
    const size_t smem = sizeof(GridTab) * (size_t)(w + 1) + sizeof(float) * 3 * (size_t)S;
    if (smem <= 200 * 1024 && g_tune[3] == 0 && B <= 65535) {
        const bool aligned = (((uintptr_t)c | (uintptr_t)left | (uintptr_t)(right ? right : left)) & 15) == 0;
        const int vec_ok = (W % 4 == 0) && aligned;
        int rc;
        switch (compose) {
            case NB200_COMPOSE_NONE: rc = launch_bw_row<NB200_COMPOSE_NONE>(p, smem, S, vec_ok, st); break;
            case NB200_COMPOSE_SBS: rc = launch_bw_row<NB200_COMPOSE_SBS>(p, smem, S, vec_ok, st); break;
            case NB200_COMPOSE_ANAGLYPH_DUBOIS: rc = launch_bw_row<NB200_COMPOSE_ANAGLYPH_DUBOIS>(p, smem, S, vec_ok, st); break;
            default: return fail("nb200_backward_warp: unknown compose mode");
        }
        if (rc) return rc;
        NB_LAUNCHED();
        return 0;
    }
    switch (compose) {
        case NB200_COMPOSE_NONE: backward_warp_kernel<NB200_COMPOSE_NONE, VEC><<<grid, block, 0, st>>>(p); break;
        case NB200_COMPOSE_SBS: backward_warp_kernel<NB200_COMPOSE_SBS, VEC><<<grid, block, 0, st>>>(p); break;
        case NB200_COMPOSE_ANAGLYPH_DUBOIS:
            backward_warp_kernel<NB200_COMPOSE_ANAGLYPH_DUBOIS, VEC><<<grid, block, 0, st>>>(p); break;
        default: return fail("nb200_backward_warp: unknown compose mode");
    }
    NB_LAUNCHED();
    return 0;
}

extern "C" int nb200_anaglyph_dubois(const float* l, const float* r, int B, int H, int W, int clip_before,
                                     float* out, void* stream) {
    NB_CHECK(l && r && out, "null pointer");
    size_t plane = (size_t)H * W, total = plane * B;
    anaglyph_dubois_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, (cudaStream_t)stream>>>(l, r, out, plane, total, clip_before);
    NB_LAUNCHED();
    return 0;
}

// backward_warp(c, grid, delta, delta_scale) of the learned stereo warps (iw3/backward_warp.py:67-83 as called from
// apply_divergence_nn_delta :213-226): grid x = mesh_x + delta * delta_scale at the delta resolution, bilinearly resized to
// the image (align_corners=True), grid_sample(bilinear, border) and clamp.  Same kernel as the depth-driven warp with
// index_shift := delta (shift = 1, convergence term = 0) and only the "+" view evaluated.
static int backward_warp_delta(const float* c, const float* delta, int B, int H, int W, int h, int w, double delta_scale, bool f16,
                               float* out, cudaStream_t st) {
    NB_CHECK(c && delta && out, "null pointer");
    NB_CHECK(B > 0 && H > 0 && W > 0 && h > 0 && w > 0, "bad shape");
    BwParams p;
    p.c = c; p.depth = delta; p.left = out; p.right = nullptr;
    p.B = B; p.H = H; p.W = W; p.h = h; p.w = w;
    p.shift = 1.0f; p.shift_conv = 0.0f;
    // an fp16 tensor times the 0-dim fp32 CUDA tensor delta_scale: ATen's mul loads both operands as fp16
    // (opmath_symmetric_gpu_kernel_with_scalars -> BinaryFunctor<Half, Half, Half>, ATen/native/cuda/Loops.cuh)
    p.delta_scale = f16 ? __half2float(__float2half_rn((float)delta_scale)) : (float)delta_scale;
    p.sy = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f;
    p.sx = W > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
    p.step_x = w > 1 ? 2.0f / (float)(w - 1) : 0.f;
    p.warp_left = 0; p.warp_right = 1;
    const int S = (W + 1 + 3) & ~3;
    const size_t smem = sizeof(GridTab) * (size_t)(w + 1) + sizeof(float) * 3 * (size_t)S;
    NB_CHECK(smem <= 200 * 1024 && B <= 65535, "image row too wide for the row-staged warp");
    const bool aligned = (((uintptr_t)c | (uintptr_t)out) & 15) == 0;
    ProfScope ps(st, PC_WARP_BW, (double)B * H * W * 4 * 6 + (double)B * h * w * 4);
    const int vec_ok = (W % 4 == 0) && aligned;
    if (f16 ? launch_bw_row<COMPOSE_RIGHT_ONLY, true>(p, smem, S, vec_ok, st) : launch_bw_row<COMPOSE_RIGHT_ONLY>(p, smem, S, vec_ok, st))
        return 1;
    NB_LAUNCHED();
    return 0;
}

extern "C" int nb200_backward_warp_delta(const float* c, const float* delta, int B, int H, int W, int h, int w, double delta_scale,
                                         float* out, void* stream) {
    return backward_warp_delta(c, delta, B, H, W, h, w, delta_scale, false, out, (cudaStream_t)stream);
}

extern "C" int nb200_backward_warp_delta_f16(const float* c, const float* delta, int B, int H, int W, int h, int w, double delta_scale,
                                             float* out, void* stream) {
    return backward_warp_delta(c, delta, B, H, W, h, w, delta_scale, true, out, (cudaStream_t)stream);
}

// apply_divergence_nn_symmetric (iw3/backward_warp.py:344-379): both eyes from one delta.  With index_shift := -delta
// (shift = -1, convergence term 0) the kernel's "-" view is mesh + delta * scale (left) and its "+" view mesh - delta * scale
// (right); negation is exact, so both grids equal the reference's grid + (+-delta) * delta_scale bit for bit.
extern "C" int nb200_backward_warp_delta_sym(const float* c, const float* delta, int B, int H, int W, int h, int w, double delta_scale,
                                             int warp_left, int warp_right, float* left, float* right, void* stream) {
    NB_CHECK(c && delta && left && right, "null pointer");
    NB_CHECK(B > 0 && H > 0 && W > 0 && h > 0 && w > 0, "bad shape");
    BwParams p;
    p.c = c; p.depth = delta; p.left = left; p.right = right;
    p.B = B; p.H = H; p.W = W; p.h = h; p.w = w;
    p.shift = -1.0f; p.shift_conv = 0.0f;
    p.delta_scale = (float)delta_scale;
    p.sy = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f;
    p.sx = W > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
    p.step_x = w > 1 ? 2.0f / (float)(w - 1) : 0.f;
    p.warp_left = warp_left != 0; p.warp_right = warp_right != 0;
    cudaStream_t st = (cudaStream_t)stream;
    const int S = (W + 1 + 3) & ~3;
    const size_t smem = sizeof(GridTab) * (size_t)(w + 1) + sizeof(float) * 3 * (size_t)S;
    NB_CHECK(smem <= 200 * 1024 && B <= 65535, "image row too wide for the row-staged warp");
    const bool aligned = (((uintptr_t)c | (uintptr_t)left | (uintptr_t)right) & 15) == 0;
    ProfScope ps(st, PC_WARP_BW, (double)B * H * W * 4 * 9 + (double)B * h * w * 4);
    if (launch_bw_row<NB200_COMPOSE_NONE>(p, smem, S, (W % 4 == 0) && aligned, st)) return 1;
    NB_LAUNCHED();
    return 0;
}
