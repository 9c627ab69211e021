// The small kernels of TransNetV2 (nunif/utils/transnetv2.py); the convolutions and fc1 run on the wgmma GEMM
// (transnet_model.cu).  Every kernel works on one frame or one (frame, branch) pair per CTA with a fixed reduction order, so
// a window's result does not depend on the other windows of the batch.
//
//   * tn_prep_kernel: [n][3][27][48] fp32 -> NHWC fp16 with the channels padded to 32.
//   * tn_tail_kernel: the end of a StackedDDCNNV2 (:122-140): relu(block2) + block1, AvgPool3d(1,2,2) and the spatial mean
//     that FrameSimilarity (:241) takes of the stack output.
//   * tn_hist_kernel: ColorHistograms.compute_color_histograms (:274-296), exact integer counts.
//   * tn_project_kernel: FrameSimilarity.projection + F.normalize (:244-245).
//   * tn_band_kernel: the T x T similarities, the zero-padded 101-wide band and fc + ReLU of both similarity branches.
//   * tn_heads_kernel: cls_layer1 / cls_layer2.
#include "transnet_kernels.h"
#include <cmath>

namespace nb200 {

__global__ void __launch_bounds__(256) tn_prep_kernel(const float* __restrict__ x, int total, __half* __restrict__ x16) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;   // pixel of [n][27][48]
    if (i >= total) return;
    const int P = TN_H * TN_W, f = i / P, p = i % P;
    const float* src = x + (size_t)f * 3 * P + p;
    __align__(16) __half v[8];
    v[0] = __float2half_rn(__ldg(src));
    v[1] = __float2half_rn(__ldg(src + P));
    v[2] = __float2half_rn(__ldg(src + 2 * P));
    for (int c = 3; c < 8; ++c) v[c] = __float2half_rn(0.f);
    uint4* o = reinterpret_cast<uint4*>(x16 + (size_t)i * TN_CIN);
    o[0] = *reinterpret_cast<const uint4*>(v);
    o[1] = o[2] = o[3] = make_uint4(0, 0, 0, 0);
}

// one CTA per frame; thread = (pixel group, channel pair)
__global__ void __launch_bounds__(256) tn_tail_kernel(const __half* __restrict__ y1, const __half* __restrict__ y2, int H, int W, int C,
                                                      __half* __restrict__ out, long long out_stride, float* __restrict__ mean,
                                                      int mean_off) {
    __shared__ float2 part[256];
    const int f = blockIdx.x, P = C / 2, G = 256 / P;
    const int pair = threadIdx.x % P, grp = threadIdx.x / P;
    const int Ho = H / 2, Wo = W / 2;
    const size_t img = (size_t)f * H * W * C;
    float2 acc = make_float2(0.f, 0.f);
    if (grp < G) {
        for (int p = grp; p < Ho * Wo; p += G) {
            const int y = p / Wo, x = p % Wo;
            float sx = 0.f, sy = 0.f;
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const size_t o = img + ((size_t)(2 * y + (q >> 1)) * W + 2 * x + (q & 1)) * C + 2 * pair;
                const float2 a = __half22float2(*reinterpret_cast<const __half2*>(y1 + o));
                const float2 b = __half22float2(*reinterpret_cast<const __half2*>(y2 + o));
                sx += fmaxf(b.x, 0.f) + a.x;
                sy += fmaxf(b.y, 0.f) + a.y;
            }
            sx *= 0.25f;
            sy *= 0.25f;
            *reinterpret_cast<__half2*>(out + f * out_stride + (size_t)p * C + 2 * pair) = __floats2half2_rn(sx, sy);
            acc.x += sx;
            acc.y += sy;
        }
    }
    part[threadIdx.x] = acc;
    __syncthreads();
    if (threadIdx.x < P) {
        float2 s = make_float2(0.f, 0.f);
        for (int g = 0; g < G; ++g) {
            s.x += part[g * P + threadIdx.x].x;
            s.y += part[g * P + threadIdx.x].y;
        }
        const float inv = 1.f / (float)(Ho * Wo);
        mean[(size_t)f * TN_FEAT + mean_off + 2 * threadIdx.x] = s.x * inv;
        mean[(size_t)f * TN_FEAT + mean_off + 2 * threadIdx.x + 1] = s.y * inv;
    }
}

// frames.int() truncates toward zero; bin = (R >> 5) << 6 | (G >> 5) << 3 | (B >> 5).  A pixel whose bin falls outside
// [0, 512) (channel values outside (-1, 256)) is not counted: the reference would add it to a neighbouring frame's histogram.
__global__ void __launch_bounds__(256) tn_hist_kernel(const float* __restrict__ x, int* __restrict__ counts) {
    __shared__ int h[512];
    const int f = blockIdx.x, P = TN_H * TN_W;
    for (int i = threadIdx.x; i < 512; i += 256) h[i] = 0;
    __syncthreads();
    const float* src = x + (size_t)f * 3 * P;
    for (int p = threadIdx.x; p < P; p += 256) {
        const int r = (int)__ldg(src + p), g = (int)__ldg(src + P + p), b = (int)__ldg(src + 2 * P + p);
        const int bin = ((r >> 5) << 6) + ((g >> 5) << 3) + (b >> 5);
        if (bin >= 0 && bin < 512) atomicAdd(&h[bin], 1);
    }
    __syncthreads();
    for (int i = threadIdx.x; i < 512; i += 256) counts[(size_t)f * 512 + i] = h[i];
}

// one CTA of 128 threads per frame: projection (448 -> 128, bias) and F.normalize(p=2, eps=1e-12)
__global__ void __launch_bounds__(TN_SIM) tn_project_kernel(const float* __restrict__ feat, const float* __restrict__ w,
                                                            const float* __restrict__ b, float* __restrict__ emb) {
    __shared__ float xs[TN_FEAT];
    __shared__ float red[TN_SIM / 32];
    const int f = blockIdx.x, j = threadIdx.x;
    for (int k = j; k < TN_FEAT; k += TN_SIM) xs[k] = feat[(size_t)f * TN_FEAT + k];
    __syncthreads();
    float acc = __ldg(b + j);
    const float* wr = w + (size_t)j * TN_FEAT;
    for (int k = 0; k < TN_FEAT; ++k) acc = fmaf(__ldg(wr + k), xs[k], acc);
    float ss = acc * acc;
    ss = warp_sum(ss);
    if ((j & 31) == 0) red[j >> 5] = ss;
    __syncthreads();
    const float norm = sqrtf(red[0] + red[1] + red[2] + red[3]);
    emb[(size_t)f * TN_SIM + j] = acc / fmaxf(norm, 1e-12f);
}

// grid (n, 2): y = 0 the colour-histogram branch, y = 1 the frame-similarity branch.  Frame f = (window, t); the band entry
// j compares t with t + j - 50 of the same window, zero outside [0, T) (the F.pad of the reference).
__global__ void __launch_bounds__(128) tn_band_kernel(const int* __restrict__ counts, const float* __restrict__ emb, int T,
                                                      const float* __restrict__ hist_w, const float* __restrict__ hist_b,
                                                      const float* __restrict__ sim_w, const float* __restrict__ sim_b,
                                                      float* __restrict__ bands, __half* __restrict__ row) {
    __shared__ float band[TN_BAND];
    const int f = blockIdx.x, br = blockIdx.y, n = gridDim.x;
    const int t = f % T, w0 = f - t;
    for (int j = threadIdx.x; j < TN_BAND; j += blockDim.x) {
        const int t2 = t + j - (TN_BAND - 1) / 2;
        float v = 0.f;
        if (t2 >= 0 && t2 < T) {
            if (br == 0) {
                // cosine similarity of two count vectors from exact integer sums (each <= 1296^2), rounded once
                const int* a = counts + (size_t)f * 512;
                const int* c = counts + (size_t)(w0 + t2) * 512;
                long long dot = 0, sa = 0, sc = 0;
                for (int k = 0; k < 512; ++k) {
                    const long long x = __ldg(a + k), y = __ldg(c + k);
                    dot += x * y;
                    sa += x * x;
                    sc += y * y;
                }
                v = (sa > 0 && sc > 0) ? (float)((double)dot / sqrt((double)sa * (double)sc)) : 0.f;
            } else {
                const float* a = emb + (size_t)f * TN_SIM;
                const float* c = emb + (size_t)(w0 + t2) * TN_SIM;
                float acc = 0.f;
                for (int k = 0; k < TN_SIM; ++k) acc = fmaf(__ldg(a + k), __ldg(c + k), acc);
                v = acc;
            }
        }
        band[j] = v;
        bands[((size_t)br * n + f) * TN_BAND + j] = v;
    }
    __syncthreads();
    const float* w = br == 0 ? hist_w : sim_w;
    const float* b = br == 0 ? hist_b : sim_b;
    for (int o = threadIdx.x; o < TN_SIM; o += blockDim.x) {
        float acc = __ldg(b + o);
        const float* wr = w + (size_t)o * TN_BAND;
        for (int j = 0; j < TN_BAND; ++j) acc = fmaf(__ldg(wr + j), band[j], acc);
        row[(size_t)f * TN_ROW + br * TN_SIM + o] = __float2half_rn(fmaxf(acc, 0.f));
    }
}

// one warp per frame
__global__ void __launch_bounds__(256) tn_heads_kernel(const __half* __restrict__ hidden, int n, const float* __restrict__ cls,
                                                       float* __restrict__ one_hot, float* __restrict__ many_hot) {
    const int f = blockIdx.x * 8 + (threadIdx.x >> 5), lane = threadIdx.x & 31;
    if (f >= n) return;
    const __half* h = hidden + (size_t)f * TN_HIDDEN;
    float a = 0.f, m = 0.f;
    for (int k = lane * 2; k < TN_HIDDEN; k += 64) {
        const float2 v = __half22float2(*reinterpret_cast<const __half2*>(h + k));
        a = fmaf(v.x, __ldg(cls + k), fmaf(v.y, __ldg(cls + k + 1), a));
        m = fmaf(v.x, __ldg(cls + TN_HIDDEN + k), fmaf(v.y, __ldg(cls + TN_HIDDEN + k + 1), m));
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) {
        a += __shfl_xor_sync(0xffffffffu, a, o);
        m += __shfl_xor_sync(0xffffffffu, m, o);
    }
    if (lane == 0) {
        one_hot[f] = a + cls[2 * TN_HIDDEN];
        many_hot[f] = m + cls[2 * TN_HIDDEN + 1];
    }
}

int tn_prep(cudaStream_t st, const float* x, int n, __half* x16) {
    const int total = n * TN_H * TN_W;
    ProfScope ps(st, PC_OTHER, 0.0, (double)total * 12.0, (double)total * TN_CIN * 2.0);
    tn_prep_kernel<<<cdiv(total, 256), 256, 0, st>>>(x, total, x16);
    NB_LAUNCHED();
    return 0;
}

int tn_stack_tail(cudaStream_t st, const __half* y1, const __half* y2, int n, int H, int W, int C, __half* out, long long out_stride,
                  float* mean, int mean_off) {
    NB_CHECK(C % 2 == 0 && C / 2 <= 256 && 256 % (C / 2) == 0, "stack tail: unsupported channel count");
    ProfScope ps(st, PC_OTHER, 0.0, (double)n * H * W * C * 4.0, (double)n * (H / 2) * (W / 2) * C * 2.0);
    tn_tail_kernel<<<n, 256, 0, st>>>(y1, y2, H, W, C, out, out_stride, mean, mean_off);
    NB_LAUNCHED();
    return 0;
}

int tn_hist(cudaStream_t st, const float* x, int n, int* counts) {
    ProfScope ps(st, PC_OTHER, 0.0, (double)n * 3 * TN_H * TN_W * 4.0, (double)n * 512 * 4.0);
    tn_hist_kernel<<<n, 256, 0, st>>>(x, counts);
    NB_LAUNCHED();
    return 0;
}

int tn_project(cudaStream_t st, const float* feat, int n, const float* w, const float* b, float* emb) {
    ProfScope ps(st, PC_OTHER, 2.0 * n * TN_SIM * TN_FEAT);
    tn_project_kernel<<<n, TN_SIM, 0, st>>>(feat, w, b, emb);
    NB_LAUNCHED();
    return 0;
}

int tn_bands(cudaStream_t st, const int* counts, const float* emb, int B, int T, const float* hist_w, const float* hist_b,
             const float* sim_w, const float* sim_b, float* bands, __half* row) {
    const int n = B * T;
    ProfScope ps(st, PC_OTHER, 2.0 * n * TN_BAND * (512.0 * 3 + TN_SIM + 2 * TN_SIM));
    tn_band_kernel<<<dim3(n, 2), 128, 0, st>>>(counts, emb, T, hist_w, hist_b, sim_w, sim_b, bands, row);
    NB_LAUNCHED();
    return 0;
}

int tn_heads(cudaStream_t st, const __half* hidden, int n, const float* cls, float* one_hot, float* many_hot) {
    ProfScope ps(st, PC_OTHER, 4.0 * n * TN_HIDDEN);
    tn_heads_kernel<<<cdiv(n, 8), 256, 0, st>>>(hidden, n, cls, one_hot, many_hot);
    NB_LAUNCHED();
    return 0;
}

}  // namespace nb200
