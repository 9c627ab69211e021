// iw3 output composition beyond plain SBS (iw3/utils.py:430-487 postprocess_image, SURVEY.md 8a row B14):
//   * the whole red-cyan anaglyph family (iw3/anaglyph.py:4-110): color, gray, half-color, wimmer, wimmer2 (dubois lives
//     in warp_backward.cu),
//   * torchvision TF.resize(..., BICUBIC, antialias=True) on fp32 planes = ATen _upsample_bicubic2d_aa
//     (align_corners=False, A = -0.5): half-SBS / half-TB squeeze and the max-output-size resize; with align_corners=True
//     (F.interpolate) the --max-output-height pre-resize of preprocess_image.
// HBM-bound elementwise / small-stencil kernels.
#include "common.cuh"
#include "../../include/nunif_b200.h"

namespace nb200 {

// torch evaluates `x[0:1] * 0.299 + x[1:2] * 0.587 + x[2:3] * 0.114` as separate fp32 kernels: no FMA contraction here
__device__ __forceinline__ float gray601(float r, float g, float b) {
    return __fadd_rn(__fadd_rn(__fmul_rn(r, 0.299f), __fmul_rn(g, 0.587f)), __fmul_rn(b, 0.114f));
}

__global__ void __launch_bounds__(256) anaglyph_mix_kernel(const float* __restrict__ l, const float* __restrict__ r,
                                                            float* __restrict__ out, size_t plane, size_t total, int type) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const size_t b = i / plane, px = i - b * plane;
    const float* lp = l + b * 3 * plane + px;
    const float* rp = r + b * 3 * plane + px;
    const float lr = lp[0], lg = lp[plane], lb = lp[2 * plane];
    const float rr = rp[0], rg = rp[plane], rb = rp[2 * plane];
    float o0, o1, o2;
    switch (type) {
        case NB200_ANAGLYPH_COLOR: o0 = lr; o1 = rg; o2 = rb; break;                                     // anaglyph.py:9-11 (no clamp)
        case NB200_ANAGLYPH_HALF_COLOR: o0 = clamp01(gray601(lr, lg, lb)); o1 = clamp01(rg); o2 = clamp01(rb); break;   // :14-18
        case NB200_ANAGLYPH_GRAY: {                                                                      // :21-26
            const float ry = gray601(rr, rg, rb);
            o0 = clamp01(gray601(lr, lg, lb)); o1 = clamp01(ry); o2 = clamp01(ry);
            break;
        }
        case NB200_ANAGLYPH_WIMMER:                                                                      // :29-35
            o0 = clamp01(__fadd_rn(__fmul_rn(lg, 0.7f), __fmul_rn(lb, 0.3f))); o1 = clamp01(rg); o2 = clamp01(rb);
            break;
        default: {                                                                                       // wimmer2 :38-48
            const float g_l = __fadd_rn(lg, __fmul_rn(0.45f, fmaxf(__fsub_rn(lr, lg), 0.f)));
            const float b_l = __fadd_rn(lb, __fmul_rn(0.25f, fmaxf(__fsub_rn(lr, lb), 0.f)));
            const float g_r = __fadd_rn(rg, __fmul_rn(0.45f, fmaxf(__fsub_rn(rr, rg), 0.f)));
            const float b_r = __fadd_rn(rb, __fmul_rn(0.25f, fmaxf(__fsub_rn(rr, rb), 0.f)));
            o0 = clamp01(powf(__fadd_rn(__fmul_rn(0.75f, g_l), __fmul_rn(0.25f, b_l)), 1.0f / 1.6f));
            o1 = clamp01(g_r); o2 = clamp01(b_r);
            break;
        }
    }
    float* op = out + b * 3 * plane + px;
    op[0] = o0; op[plane] = o1; op[2 * plane] = o2;
}

struct ResizeParams {
    const float* x;
    float* out;
    int planes, H, W, oh, ow, clamp, align_corners;
    float sy, sx, supy, supx, invy, invx;
};

// Tap window [lo, lo + size) and the filter argument of tap j (aa_arg).  align_corners = 0 keeps the
// fp32-rounded centre (bit-exact to ATen's CPU kernel).  align_corners = 1 follows ATen's CUDA kernel, whose centre
// scale * (i + 0.5) is contracted into each use (one FMA, never rounded on its own): with the inexact scales of
// (in - 1) / (out - 1) a rounded centre moves the 4K -> 1080 output by up to 2e-5.
struct AaSpan { int lo, size; float off; };
__device__ __forceinline__ AaSpan aa_span(int i, float s, float sup, int n, int align_corners) {
    AaSpan a;
    const float t = (float)i + 0.5f;
    if (align_corners) {
        a.lo = max(0, (int)(fmaf(s, t, -sup) + 0.5f));
        a.size = min(n, (int)(fmaf(s, t, sup) + 0.5f)) - a.lo;
        a.off = fmaf(-s, t, (float)a.lo);   // xmin - centre
    } else {
        const float c = __fmul_rn(s, t);
        a.lo = max(0, (int)(c - sup + 0.5f));
        a.size = min(n, (int)(c + sup + 0.5f)) - a.lo;
        a.off = -c;      // arg = (j + lo) - c + 0.5, as before
    }
    return a;
}
__device__ __forceinline__ float aa_arg(const AaSpan& a, int j, float inv, int align_corners) {
    return align_corners ? __fmul_rn(__fadd_rn(__fadd_rn((float)j, a.off), 0.5f), inv) : ((float)(j + a.lo) + a.off + 0.5f) * inv;
}

// one thread per output pixel; horizontal pass inside the vertical loop (ATen order: horizontal first, fp32)
__global__ void __launch_bounds__(128) resize_bicubic_aa_kernel(ResizeParams p) {
    const int ox = blockIdx.x * blockDim.x + threadIdx.x, oy = blockIdx.y, pl = blockIdx.z;
    if (ox >= p.ow) return;
    const AaSpan sy = aa_span(oy, p.sy, p.supy, p.H, p.align_corners), sx = aa_span(ox, p.sx, p.supx, p.W, p.align_corners);
    const int ymin = sy.lo, ysize = sy.size, xmin = sx.lo, xsize = sx.size;
    float wxs = 0.f, wys = 0.f;
    for (int j = 0; j < xsize; ++j) wxs += cubic_aa(aa_arg(sx, j, p.invx, p.align_corners));
    for (int j = 0; j < ysize; ++j) wys += cubic_aa(aa_arg(sy, j, p.invy, p.align_corners));
    const float* src = p.x + (size_t)pl * p.H * p.W;
    float acc = 0.f;
    for (int jy = 0; jy < ysize; ++jy) {
        const float wy = cubic_aa(aa_arg(sy, jy, p.invy, p.align_corners)) / wys;
        const float* row = src + (size_t)(ymin + jy) * p.W + xmin;
        float h = 0.f;
        for (int jx = 0; jx < xsize; ++jx) h += cubic_aa(aa_arg(sx, jx, p.invx, p.align_corners)) / wxs * __ldg(row + jx);
        acc += wy * h;
    }
    p.out[((size_t)pl * p.oh + oy) * p.ow + ox] = p.clamp ? clamp01(acc) : acc;
}


// ---- VR180: iw3/equirectangular.py:7-40.  Zero-pad to (roughly) a square of 1.5 x the longer edge, then
// F.grid_sample(bicubic, zeros, align_corners=True) through the mesh  x' = k tan(az), y' = k tan(el) / cos(az).
// The padded image is never materialised: taps outside the source rectangle contribute 0, exactly like the pad + zeros mode.
__device__ __forceinline__ float linspace_m1_p1(int idx, int steps) {
    // torch.linspace(-1, 1, steps) in fp32: start + step*i on the first half, end - step*(steps-1-i) on the second
    const float step = 2.0f / (float)(steps - 1);
    return idx < steps / 2 ? -1.0f + step * (float)idx : 1.0f - step * (float)(steps - idx - 1);
}
__device__ __forceinline__ void cubic_coeffs(float t, float (&w)[4]) {   // ATen get_cubic_upsample_coefficients, A = -0.75
    const float A = -0.75f;
    auto c1 = [&](float x) { return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; };
    auto c2 = [&](float x) { return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; };
    w[0] = c2(t + 1.f); w[1] = c1(t); w[2] = c1(1.f - t); w[3] = c2(2.f - t);
}
__global__ void __launch_bounds__(256) equirect_kernel(const float* __restrict__ c, int C, int H, int W, int pad_h, int pad_w, int Ho, int Wo,
                                                       float k, float* __restrict__ out) {
    const int j = blockIdx.x * blockDim.x + threadIdx.x, i = blockIdx.y;
    if (j >= Wo) return;
    const float x = linspace_m1_p1(j, Wo), y = linspace_m1_p1(i, Ho);
    const float az = x * 1.5707963267948966f, el = y * 1.5707963267948966f;
    const float gx = k * tanf(az), gy = k * (tanf(el) / cosf(az));
    const float ix = ((gx + 1.f) / 2.f) * (float)(Wo - 1), iy = ((gy + 1.f) / 2.f) * (float)(Ho - 1);   // align_corners=True
    const float fx = floorf(ix), fy = floorf(iy);
    float wx[4], wy[4];
    cubic_coeffs(ix - fx, wx);
    cubic_coeffs(iy - fy, wy);
    // tap coordinates in the SOURCE image; anything outside is the zero pad / zeros padding mode.  Guard the float->int
    // conversion: tan() explodes towards the poles.
    const bool far_away = !(fabsf(fx) < 1e8f && fabsf(fy) < 1e8f);
    const int x0 = far_away ? -1000000 : (int)fx - 1 - pad_w, y0 = far_away ? -1000000 : (int)fy - 1 - pad_h;
    for (int ch = 0; ch < C; ++ch) {
        const float* p = c + (size_t)ch * H * W;
        float acc = 0.f;
#pragma unroll
        for (int a = 0; a < 4; ++a) {
            const int yy = y0 + a;
            float row = 0.f;
#pragma unroll
            for (int b = 0; b < 4; ++b) {
                const int xx = x0 + b;
                const float v = (yy >= 0 && yy < H && xx >= 0 && xx < W) ? __ldg(p + (size_t)yy * W + xx) : 0.f;
                row = row + v * wx[b];
            }
            acc = acc + row * wy[a];
        }
        out[((size_t)ch * Ho + i) * Wo + j] = clamp01(acc);
    }
}

}  // namespace nb200

using namespace nb200;

extern "C" int nb200_anaglyph(const float* l, const float* r, int B, int H, int W, int type, float* out, void* stream) {
    NB_CHECK(l && r && out, "null pointer");
    NB_CHECK(B > 0 && H > 0 && W > 0, "bad shape");
    if (type == NB200_ANAGLYPH_DUBOIS || type == NB200_ANAGLYPH_DUBOIS2)
        return nb200_anaglyph_dubois(l, r, B, H, W, type == NB200_ANAGLYPH_DUBOIS ? 1 : 0, out, stream);
    NB_CHECK(type >= NB200_ANAGLYPH_COLOR && type <= NB200_ANAGLYPH_WIMMER2, "unknown anaglyph type");
    const size_t plane = (size_t)H * W, total = plane * B;
    anaglyph_mix_kernel<<<(unsigned)cdiv64((int64_t)total, 256), 256, 0, (cudaStream_t)stream>>>(l, r, out, plane, total, type);
    NB_LAUNCHED();
    return 0;
}

extern "C" int nb200_resize_bicubic_aa(const float* x, int planes, int H, int W, int oh, int ow, int clamp01_out, float* out,
                                       void* stream) {
    return nb200_resize_bicubic_aa_ac(x, planes, H, W, oh, ow, clamp01_out, 0, out, stream);
}

// ATen upsample_gen2d_aa: align_corners enters through area_pixel_compute_scale only ((in - 1) / (out - 1), 0 for a
// 1-pixel output); the centre stays scale * (i + 0.5) and the support and weights follow from that scale as before.
extern "C" int nb200_resize_bicubic_aa_ac(const float* x, int planes, int H, int W, int oh, int ow, int clamp01_out,
                                          int align_corners, float* out, void* stream) {
    NB_CHECK(x && out, "null pointer");
    NB_CHECK(planes > 0 && planes <= 65535 && H > 0 && W > 0 && oh > 0 && ow > 0, "bad shape");
    ResizeParams p;
    p.x = x; p.out = out; p.planes = planes; p.H = H; p.W = W; p.oh = oh; p.ow = ow; p.clamp = clamp01_out;
    p.align_corners = align_corners ? 1 : 0;
    if (align_corners) {
        p.sy = oh > 1 ? (float)(H - 1) / (float)(oh - 1) : 0.f;
        p.sx = ow > 1 ? (float)(W - 1) / (float)(ow - 1) : 0.f;
    } else {
        p.sy = (float)H / (float)oh; p.sx = (float)W / (float)ow;
    }
    p.supy = p.sy >= 1.f ? 2.f * p.sy : 2.f; p.supx = p.sx >= 1.f ? 2.f * p.sx : 2.f;
    p.invy = p.sy >= 1.f ? 1.f / p.sy : 1.f; p.invx = p.sx >= 1.f ? 1.f / p.sx : 1.f;
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope ps(st, PC_OTHER, (double)planes * ((double)H * W + (double)oh * ow) * 4);
    resize_bicubic_aa_kernel<<<dim3(cdiv(ow, 128), oh, planes), 128, 0, st>>>(p);
    NB_LAUNCHED();
    return 0;
}

// iw3/equirectangular.py:7-40 (VR180 output): c [C][H][W] -> out [C][H + 2*pad_h][W + 2*pad_w] (nb200_equirectangular_size)
extern "C" int nb200_equirectangular_size(int H, int W, int* out_h, int* out_w) {
    NB_CHECK(out_h && out_w && H > 0 && W > 0, "bad arguments");
    const int max_edge = H > W ? H : W, output_size = max_edge + max_edge / 2;
    *out_h = H + 2 * ((output_size - H) / 2);
    *out_w = W + 2 * ((output_size - W) / 2);
    return 0;
}
extern "C" int nb200_equirectangular(const float* c, int C, int H, int W, float* out, void* stream) {
    NB_CHECK(c && out, "null pointer");
    NB_CHECK(C > 0 && H > 0 && W > 0, "bad shape");
    const int max_edge = H > W ? H : W, output_size = max_edge + max_edge / 2;
    const int pad_h = (output_size - H) / 2, pad_w = (output_size - W) / 2;
    const int Ho = H + 2 * pad_h, Wo = W + 2 * pad_w;
    NB_CHECK(Ho > 1 && Wo > 1, "image too small");
    const float k = (float)((double)max_edge / (double)output_size);
    equirect_kernel<<<dim3(cdiv(Wo, 256), Ho), 256, 0, (cudaStream_t)stream>>>(c, C, H, W, pad_h, pad_w, Ho, Wo, k, out);
    NB_LAUNCHED();
    return 0;
}
