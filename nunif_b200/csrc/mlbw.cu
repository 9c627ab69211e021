// Kernels of `sbs.mlbw` (iw3/models/mlbw.py:36-127), the multi-layer learned stereo warp (methods mlbw_l2 / mlbw_l4 [s]): its input
// and output stages.  Like row_flow_v3 the network works on a (1, 8) pixel-unshuffled token grid, through window-attention
// blocks (window_mha.cu and the wgmma GEMM); it predicts L horizontal flow layers and L blending weights per pixel.
#include "mlbw_kernels.h"

namespace nb200 {

namespace {

__global__ void __launch_bounds__(256) mlbw_prep_kernel(const float* __restrict__ x, __half* __restrict__ out, int B, int H, int W, int ph1,
                                                         int pw1, int Hp, int Wt, int C1, const float* __restrict__ w_in,
                                                         const float* __restrict__ b_in) {
    extern __shared__ float sw[];            // [C1][3][9] + [C1]
    if (threadIdx.x == 0) NB_PDL_TRIGGER();
    for (int i = threadIdx.x; i < C1 * 27; i += blockDim.x) sw[i] = w_in[i];
    for (int i = threadIdx.x; i < C1; i += blockDim.x) sw[C1 * 27 + i] = b_in[i];
    __syncthreads();
    const long long total = (long long)B * Hp * Wt * C1;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int c = (int)(i % C1);
    long long t = i / C1;
    const int xt = (int)(t % Wt);
    t /= Wt;
    const int y = (int)(t % Hp), b = (int)(t / Hp);
    const int sy = min(max(y - ph1, 0), H - 1);                       // replication_pad2d (pw1, pw2, ph1, ph2)
    float acc[8];
#pragma unroll
    for (int s = 0; s < 8; ++s) acc[s] = sw[C1 * 27 + c];
#pragma unroll
    for (int ci = 0; ci < 3; ++ci) {
        const float* row = x + (((size_t)b * 3 + ci) * H + sy) * W;
        float v[16];
#pragma unroll
        for (int k = 0; k < 16; ++k) v[k] = __ldg(row + min(max(xt * 8 + k - 4 - pw1, 0), W - 1));    // both pads are replications: one clamp
#pragma unroll
        for (int tap = 0; tap < 9; ++tap) {
            const float wv = sw[(c * 3 + ci) * 9 + tap];
#pragma unroll
            for (int s = 0; s < 8; ++s) acc[s] = fmaf(wv, v[s + tap], acc[s]);
        }
    }
    __align__(16) __half2 o[4];
#pragma unroll
    for (int s = 0; s < 4; ++s) {
        const float a0 = acc[2 * s] > 0.f ? acc[2 * s] : 0.2f * acc[2 * s], a1 = acc[2 * s + 1] > 0.f ? acc[2 * s + 1] : 0.2f * acc[2 * s + 1];
        o[s] = __floats2half2_rn(a0, a1);
    }
    *reinterpret_cast<uint4*>(out + (((size_t)b * Hp + y) * Wt + xt) * (8 * C1) + c * 8) = *reinterpret_cast<const uint4*>(o);
}

// HOLE: the hole_mask head (mask_mlbw_l2, mlbw.py:70-74,104-107): output channel 2L is the hole logit, written to `hole`
template <int L, bool HOLE>
__global__ void __launch_bounds__(256) mlbw_out_kernel(const __half* __restrict__ t, const __half* __restrict__ t0, int B, int H, int W, int ph1,
                                                        int pw1, int Hp, int Wt, int C1, const float* __restrict__ w_out,
                                                        const float* __restrict__ b_out, float* __restrict__ delta, float* __restrict__ lw,
                                                        float* __restrict__ hole) {
    constexpr int NO = 2 * L + (HOLE ? 1 : 0);
    extern __shared__ float sw[];            // [NO][C1][9] + [NO]
    for (int i = threadIdx.x; i < NO * C1 * 9 + NO; i += blockDim.x) sw[i] = i < NO * C1 * 9 ? w_out[i] : b_out[i - NO * C1 * 9];
    __syncthreads();
    const long long total = (long long)B * H * W;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int X = (int)(i % W), Y = (int)((i / W) % H), b = (int)(i / ((long long)W * H));
    const int py = Y + ph1, px = X + pw1, Wp = Wt * 8;               // F.pad with negative padding = crop
    float acc[NO];
#pragma unroll
    for (int o = 0; o < NO; ++o) acc[o] = sw[NO * C1 * 9 + o];
    const size_t rowtok = ((size_t)b * Hp + py) * Wt;
#pragma unroll 1
    for (int tap = 0; tap < 9; ++tap) {
        const int qx = min(max(px + tap - 4, 0), Wp - 1);              // ReplicationPad2d (4, 4, 0, 0)
        const size_t base = (rowtok + (qx >> 3)) * (size_t)(8 * C1) + (qx & 7);
        for (int c = 0; c < C1; ++c) {
            // pixel_shuffle (1, 8): S[c][y][x] = token(y, x / 8)[c * 8 + x % 8]; x + x1 is rounded to fp16 like the reference's tensor
            const float v = __half2float(__float2half_rn(__half2float(t[base + c * 8]) + __half2float(t0[base + c * 8])));
#pragma unroll
            for (int o = 0; o < NO; ++o) acc[o] = fmaf(sw[(o * C1 + c) * 9 + tap], v, acc[o]);
        }
    }
    if (HOLE) hole[(size_t)b * H * W + (size_t)Y * W + X] = __half2float(__float2half_rn(acc[2 * L]));   // .float() of the fp16 logit
    float lg[L], mx = -1e30f;
#pragma unroll
    for (int l = 0; l < L; ++l) {
        delta[((size_t)b * L + l) * H * W + (size_t)Y * W + X] = __half2float(__float2half_rn(acc[l]));   // conv output is fp16 under autocast
        lg[l] = __half2float(__float2half_rn(acc[L + l]));
        mx = fmaxf(mx, lg[l]);
    }
    float sum = 0.f;
#pragma unroll
    for (int l = 0; l < L; ++l) { lg[l] = __expf(lg[l] - mx); sum += lg[l]; }
    const float inv = 1.f / sum;
#pragma unroll
    for (int l = 0; l < L; ++l) lw[((size_t)b * L + l) * H * W + (size_t)Y * W + X] = lg[l] * inv;
}

// postprocess_hole_mask's closing, resize and threshold (iw3/backward_warp.py:382-388), one output pixel per thread.  The bilinear
// resize reads the closed logits at source rows y0, y0 + 1 and columns x0, x0 + 1; closing = a 3x3 max (dilation) then a 3x3 min
// (erosion), both with -inf padding, so those four values need the 6x6 logits around them.  Outside the image a logit is -inf
// (never wins the max) and a dilated value is +inf (never wins the min): exactly max_pool2d's padding, so the closed logits are
// bit-exact.  The resize follows ATen's align_corners=True bilinear (upsample_bilinear2d): scale = (in - 1) / (out - 1) in fp32,
// src = scale * dst, i0 = min(floor(src), in - 1), i1 = i0 + (i0 < in - 1), l1 = clamp(src - i0, 0, 1), l0 = 1 - l1; an axis of
// equal size copies (l0 = 1, l1 = 0).  The products that feed the floor and the threshold are rounded explicitly (no FMA
// contraction).  mirror: the coordinates are evaluated in the flipped frame, where forward_left evaluates them; scale * x is not
// flip-symmetric in floating point.
__global__ void __launch_bounds__(256) hole_mask_kernel(const float* __restrict__ logits, int B, int h, int w, int H, int W, float sy,
                                                         float sx, float threshold, int mirror, float* __restrict__ out) {
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= (long long)B * H * W) return;
    const int X = (int)(i % W), Y = (int)((i / W) % H), b = (int)(i / ((long long)W * H));
    const float* l = logits + (size_t)b * h * w;
    int y0 = Y, y1 = Y, x0, x1;
    float ly0 = 1.f, ly1 = 0.f, lx0 = 1.f, lx1 = 0.f;
    if (h != H) {
        const float src = __fmul_rn(sy, (float)Y);
        y0 = min((int)floorf(src), h - 1);
        y1 = y0 + (y0 < h - 1 ? 1 : 0);
        ly1 = fminf(fmaxf(__fsub_rn(src, (float)y0), 0.f), 1.f);
        ly0 = __fsub_rn(1.f, ly1);
    }
    const int xf = mirror ? W - 1 - X : X;                          // column in the frame the reference resizes
    if (w != W) {
        const float src = __fmul_rn(sx, (float)xf);
        x0 = min((int)floorf(src), w - 1);
        x1 = x0 + (x0 < w - 1 ? 1 : 0);
        lx1 = fminf(fmaxf(__fsub_rn(src, (float)x0), 0.f), 1.f);
        lx0 = __fsub_rn(1.f, lx1);
    } else {
        x0 = x1 = xf;
    }
    if (mirror) { x0 = w - 1 - x0; x1 = w - 1 - x1; }                // back to image columns (closing is flip-symmetric)
    // 6x6 logits at rows ya - 2 .. ya + 3, columns xa - 2 .. xa + 3, where (ya, xa) is the top-left of the 2x2 source block
    const int ya = min(y0, y1), xa = min(x0, x1);
    float v[6][6];
#pragma unroll
    for (int r = 0; r < 6; ++r) {
        const int yy = ya - 2 + r;
#pragma unroll
        for (int c = 0; c < 6; ++c) {
            const int xx = xa - 2 + c;
            v[r][c] = (yy >= 0 && yy < h && xx >= 0 && xx < w) ? __ldg(l + (size_t)yy * w + xx) : -INFINITY;
        }
    }
    float d[4][4];                                                  // dilation at rows ya - 1 .. ya + 2, columns xa - 1 .. xa + 2
#pragma unroll
    for (int r = 0; r < 4; ++r)
#pragma unroll
        for (int c = 0; c < 4; ++c) {
            float m = -INFINITY;
#pragma unroll
            for (int dy = 0; dy < 3; ++dy)
#pragma unroll
                for (int dx = 0; dx < 3; ++dx) m = fmaxf(m, v[r + dy][c + dx]);
            const int yy = ya - 1 + r, xx = xa - 1 + c;
            d[r][c] = (yy >= 0 && yy < h && xx >= 0 && xx < w) ? m : INFINITY;
        }
    float cl[2][2];                                                 // closing at rows ya, ya + 1, columns xa, xa + 1
#pragma unroll
    for (int r = 0; r < 2; ++r)
#pragma unroll
        for (int c = 0; c < 2; ++c) {
            float m = INFINITY;
#pragma unroll
            for (int dy = 0; dy < 3; ++dy)
#pragma unroll
                for (int dx = 0; dx < 3; ++dx) m = fminf(m, d[r + dy][c + dx]);
            cl[r][c] = m;
        }
    // select, not index, so that cl stays in registers (each offset is 0 or 1)
    const bool r0 = y0 != ya, r1 = y1 != ya, c0 = x0 != xa, c1 = x1 != xa;
    const float a00 = r0 ? (c0 ? cl[1][1] : cl[1][0]) : (c0 ? cl[0][1] : cl[0][0]);
    const float a01 = r0 ? (c1 ? cl[1][1] : cl[1][0]) : (c1 ? cl[0][1] : cl[0][0]);
    const float a10 = r1 ? (c0 ? cl[1][1] : cl[1][0]) : (c0 ? cl[0][1] : cl[0][0]);
    const float a11 = r1 ? (c1 ? cl[1][1] : cl[1][0]) : (c1 ? cl[0][1] : cl[0][0]);
    // ATen's nested order: rows outer, columns inner, each as w0 * v0 + w1 * v1
    const float t0 = __fadd_rn(__fmul_rn(a00, lx0), __fmul_rn(a01, lx1));
    const float t1 = __fadd_rn(__fmul_rn(a10, lx0), __fmul_rn(a11, lx1));
    const float z = __fadd_rn(__fmul_rn(t0, ly0), __fmul_rn(t1, ly1));
    const float sig = 1.f / (1.f + expf(-z));                       // torch.sigmoid in fp32, then the compare
    out[i] = threshold != threshold ? z : (sig > threshold ? 1.f : 0.f);   // NaN threshold: the resized closed logits (tests)
}

}  // namespace

int hole_mask(cudaStream_t st, const float* logits, int B, int h, int w, int H, int W, float threshold, int mirror, float* out) {
    const long long n = (long long)B * H * W;
    // ATen area_pixel_compute_scale with align_corners: (float)(in - 1) / (out - 1), 0 for a one-pixel output
    const float sy = H > 1 ? (float)(h - 1) / (float)(H - 1) : 0.f, sx = W > 1 ? (float)(w - 1) / (float)(W - 1) : 0.f;
    ProfScope ps(st, PC_HOLE_MASK, 4.0 * ((double)B * h * w + (double)n), 4.0 * B * h * w, 4.0 * n);
    hole_mask_kernel<<<(unsigned)cdiv64(n, 256), 256, 0, st>>>(logits, B, h, w, H, W, sy, sx, threshold, mirror, out);
    NB_LAUNCHED();
    return 0;
}

int mlbw_prep(cudaStream_t st, const float* x, int B, int H, int W, int ph1, int pw1, int Hp, int Wt, int C1, const float* w_in,
              const float* b_in, __half* out) {
    const long long total = (long long)B * Hp * Wt * C1;
    mlbw_prep_kernel<<<(unsigned)cdiv64(total, 256), 256, (size_t)(C1 * 28) * 4, st>>>(x, out, B, H, W, ph1, pw1, Hp, Wt, C1, w_in, b_in);
    NB_LAUNCHED();
    return 0;
}

int mlbw_out(cudaStream_t st, const __half* t, const __half* t0, int B, int H, int W, int ph1, int pw1, int Hp, int Wt, int C1, int L,
             const float* w_out, const float* b_out, float* delta, float* lw, float* hole) {
    const long long total = (long long)B * H * W;
    const int NO = 2 * L + (hole ? 1 : 0);
    const size_t smem = (size_t)(NO * C1 * 9 + NO) * 4;
    const unsigned grid = (unsigned)cdiv64(total, 256);
    if (L == 2 && hole) mlbw_out_kernel<2, true><<<grid, 256, smem, st>>>(t, t0, B, H, W, ph1, pw1, Hp, Wt, C1, w_out, b_out, delta, lw, hole);
    else if (L == 2) mlbw_out_kernel<2, false><<<grid, 256, smem, st>>>(t, t0, B, H, W, ph1, pw1, Hp, Wt, C1, w_out, b_out, delta, lw, nullptr);
    else if (L == 4 && !hole) mlbw_out_kernel<4, false><<<grid, 256, smem, st>>>(t, t0, B, H, W, ph1, pw1, Hp, Wt, C1, w_out, b_out, delta, lw, nullptr);
    else return fail("mlbw_out: num_layers must be 2 or 4 (the hole head exists for 2 only)");
    NB_LAUNCHED();
    return 0;
}

}  // namespace nb200
