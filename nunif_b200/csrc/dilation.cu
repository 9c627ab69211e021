// iw3 depth post-processing: dilate_edge, per-frame min/max normalise + mapper.
//
// Replaces iw3/dilation.py:101-142 (~20 ATen launches + 4 global reductions per
// iteration) with 3 launches per iteration:
//   K1  range3x3 = max3x3 - min3x3, per-block partial {sum, sum^2 (double), min, max}
//   K2  finalise per-image stats.  The reference's normalised weight
//         w = (clamp((r-mean)/(rms+1e-6), +-3) - w_min) / (w_max - w_min + 1e-6)
//       is monotone in r, so w_min/w_max follow from r_min/r_max: one reduction pass
//       instead of three.
//   K3  x' = x*(1-w) + maxpool_k(gauss3x3_replicate(x))*w  (5x5 footprint, fused)
// and iw3/depth_scaler.py:4-17 + iw3/mapper.py (any mapper, csrc/mapper.cuh) with 2 launches.
// These maps are ~1 MB per frame: latency-bound, reported in microseconds.
#include "common.cuh"
#include "mapper.cuh"
#include "../../include/nunif_b200.h"

namespace nb200 {

constexpr int DL_THREADS = 256;
constexpr int DL_MAX_BLOCKS = 256;  // partials per image

struct DlPartial {
    double sum, sumsq;
    float mn, mx;
};

// K1: grid (nblk, B).  Each block strides over the image.
__global__ void __launch_bounds__(DL_THREADS) range_stats_kernel(const float* __restrict__ x, float* __restrict__ range,
                                                                 DlPartial* __restrict__ partials, int h, int w) {
    const int b = blockIdx.y;
    const float* xb = x + (size_t)b * h * w;
    float* rb = range + (size_t)b * h * w;
    const int n = h * w;
    double s = 0.0, ss = 0.0;
    float mn = __int_as_float(0x7f800000), mx = -mn;
    for (int i = blockIdx.x * DL_THREADS + threadIdx.x; i < n; i += gridDim.x * DL_THREADS) {
        int yy = i / w, xx = i - yy * w;
        float vmax = -__int_as_float(0x7f800000), vmin = __int_as_float(0x7f800000);
#pragma unroll
        for (int dy = -1; dy <= 1; ++dy) {
            int y2 = yy + dy;
            if (y2 < 0 || y2 >= h) continue;  // max_pool2d pads with -inf => ignore
#pragma unroll
            for (int dx = -1; dx <= 1; ++dx) {
                int x2 = xx + dx;
                if (x2 < 0 || x2 >= w) continue;
                float v = __ldg(xb + (size_t)y2 * w + x2);
                vmax = fmaxf(vmax, v);
                vmin = fminf(vmin, v);
            }
        }
        float r = vmax - vmin;
        rb[i] = r;
        s += (double)r;
        ss += (double)r * (double)r;
        mn = fminf(mn, r);
        mx = fmaxf(mx, r);
    }
    __shared__ double sh_s[DL_THREADS / 32], sh_ss[DL_THREADS / 32];
    __shared__ float sh_mn[DL_THREADS / 32], sh_mx[DL_THREADS / 32];
    s = warp_sum(s); ss = warp_sum(ss); mn = warp_min(mn); mx = warp_max(mx);
    const int wid = threadIdx.x >> 5, lane = threadIdx.x & 31;
    if (lane == 0) { sh_s[wid] = s; sh_ss[wid] = ss; sh_mn[wid] = mn; sh_mx[wid] = mx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int k = 1; k < DL_THREADS / 32; ++k) {
            s += sh_s[k]; ss += sh_ss[k]; mn = fminf(mn, sh_mn[k]); mx = fmaxf(mx, sh_mx[k]);
        }
        DlPartial p; p.sum = s; p.sumsq = ss; p.mn = mn; p.mx = mx;
        partials[(size_t)b * gridDim.x + blockIdx.x] = p;
    }
}

// K2: one block per image. stats[b] = {mean, 1/(rms+1e-6), w_min, 1/(w_max-w_min+1e-6)}
__global__ void range_finalize_kernel(const DlPartial* __restrict__ partials, int nblk, int n, float4* __restrict__ stats) {
    const int b = blockIdx.x;
    if (threadIdx.x != 0) return;
    double s = 0.0, ss = 0.0;
    float mn = __int_as_float(0x7f800000), mx = -mn;
    for (int k = 0; k < nblk; ++k) {
        DlPartial p = partials[(size_t)b * nblk + k];
        s += p.sum; ss += p.sumsq; mn = fminf(mn, p.mn); mx = fmaxf(mx, p.mx);
    }
    double mean = s / n;
    double var = ss / n - mean * mean;  // E[(r-mean)^2]
    if (var < 0) var = 0;
    float meanf = (float)mean;
    float rms = (float)sqrt(var);
    float denom = rms + 1e-6f;
    float wmin = fminf(fmaxf((mn - meanf) / denom, -3.f), 3.f);
    float wmax = fminf(fmaxf((mx - meanf) / denom, -3.f), 3.f);
    stats[b] = make_float4(meanf, denom, wmin, (wmax - wmin) + 1e-6f);
}

// K3: kh x kw max-pool (stride 1, -inf pad) of the 3x3 gaussian (replicate pad), lerp by w.
__global__ void __launch_bounds__(DL_THREADS) dilate_apply_kernel(const float* __restrict__ x, const float* __restrict__ range,
                                                                  const float4* __restrict__ stats, float* __restrict__ out,
                                                                  int h, int w, int kh, int kw) {
    const int b = blockIdx.y;
    const int i = blockIdx.x * DL_THREADS + threadIdx.x;
    if (i >= h * w) return;
    const float* xb = x + (size_t)b * h * w;
    const int yy = i / w, xx = i - yy * w;
    const float4 st = stats[b];
    float wgt = fminf(fmaxf((range[(size_t)b * h * w + i] - st.x) / st.y, -3.f), 3.f);
    wgt = (wgt - st.z) / st.w;
    const int ph = kh / 2, pw = kw / 2;
    float best = -__int_as_float(0x7f800000);
    for (int dy = -ph; dy <= ph; ++dy) {
        int yc = yy + dy;
        if (yc < 0 || yc >= h) continue;
        for (int dx = -pw; dx <= pw; ++dx) {
            int xc = xx + dx;
            if (xc < 0 || xc >= w) continue;
            // gaussian_blur dilation.py:30-38: [[21,31,21],[31,48,31],[21,31,21]]/256, replicate pad
            float g = 0.f;
#pragma unroll
            for (int ky = -1; ky <= 1; ++ky) {
                int y2 = min(max(yc + ky, 0), h - 1);
#pragma unroll
                for (int kx = -1; kx <= 1; ++kx) {
                    int x2 = min(max(xc + kx, 0), w - 1);
                    float kv = (ky == 0 ? (kx == 0 ? 48.f : 31.f) : (kx == 0 ? 31.f : 21.f)) / 256.f;
                    g += __ldg(xb + (size_t)y2 * w + x2) * kv;
                }
            }
            best = fmaxf(best, g);
        }
    }
    float xv = xb[i];
    out[(size_t)b * h * w + i] = (xv * (1.f - wgt)) + (best * wgt);
}

// ---- min/max normalise + mapper -------------------------------------------
__global__ void __launch_bounds__(DL_THREADS) minmax_partial_kernel(const float* __restrict__ x, float2* __restrict__ partials, int n) {
    const int b = blockIdx.y;
    const float* xb = x + (size_t)b * n;
    float mn = __int_as_float(0x7f800000), mx = -mn;
    for (int i = blockIdx.x * DL_THREADS + threadIdx.x; i < n; i += gridDim.x * DL_THREADS) {
        float v = __ldg(xb + i);
        mn = fminf(mn, v);
        mx = fmaxf(mx, v);
    }
    __shared__ float sh_mn[DL_THREADS / 32], sh_mx[DL_THREADS / 32];
    mn = warp_min(mn); mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) { sh_mn[threadIdx.x >> 5] = mn; sh_mx[threadIdx.x >> 5] = mx; }
    __syncthreads();
    if (threadIdx.x == 0) {
        for (int k = 1; k < DL_THREADS / 32; ++k) { mn = fminf(mn, sh_mn[k]); mx = fmaxf(mx, sh_mx[k]); }
        partials[(size_t)b * gridDim.x + blockIdx.x] = make_float2(mn, mx);
    }
}

__global__ void __launch_bounds__(DL_THREADS) minmax_apply_kernel(const float* __restrict__ x, const float2* __restrict__ partials,
                                                                  int nblk, int n, const nb200_mapper mapper, float* __restrict__ out,
                                                                  float* __restrict__ minmax_out) {
    const int b = blockIdx.y;
    __shared__ float s_mn, s_mx;
    if (threadIdx.x == 0) {
        float mn = __int_as_float(0x7f800000), mx = -mn;
        for (int k = 0; k < nblk; ++k) {
            float2 p = partials[(size_t)b * nblk + k];
            mn = fminf(mn, p.x);
            mx = fmaxf(mx, p.y);
        }
        s_mn = mn; s_mx = mx;
        if (minmax_out && blockIdx.x == 0) { minmax_out[2 * b] = mn; minmax_out[2 * b + 1] = mx; }
    }
    __syncthreads();
    const float mn = s_mn, scale = s_mx - s_mn;
    for (int i = blockIdx.x * DL_THREADS + threadIdx.x; i < n; i += gridDim.x * DL_THREADS) {
        float v = x[(size_t)b * n + i];
        if (scale > 0.f) v = (v - mn) / scale;  // depth_scaler.py:9-12
        v = clamp01(v);
        out[(size_t)b * n + i] = mapper_eval(mapper, v);
    }
}

}  // namespace nb200

using namespace nb200;

static int dl_blocks(int n) { int nb = cdiv(n, DL_THREADS * 4); return nb < 1 ? 1 : (nb > DL_MAX_BLOCKS ? DL_MAX_BLOCKS : nb); }

extern "C" size_t nb200_dilate_edge_workspace(int B, int h, int w) {
    size_t n = (size_t)B * h * w * sizeof(float);
    // ping buffer + range + partials + stats
    return 2 * n + (size_t)B * DL_MAX_BLOCKS * sizeof(DlPartial) + (size_t)B * sizeof(float4) + 256;
}

extern "C" int nb200_dilate_edge(const float* x, int B, int h, int w, int x_iter, int y_iter, float* out,
                                 void* workspace, void* stream) {
    NB_CHECK(x && out, "null pointer");
    NB_CHECK(x_iter >= 0 && y_iter >= 0, "iteration counts must be >= 0");
    cudaStream_t st = (cudaStream_t)stream;
    const size_t n = (size_t)B * h * w;
    const int xy = x_iter < y_iter ? x_iter : y_iter;              // dilation.py:117-120
    const int total = xy + (y_iter - xy) + (x_iter - xy);
    if (total == 0) {
        if (out != x) NB_CUDA(cudaMemcpyAsync(out, x, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
        return 0;
    }
    NB_CHECK(workspace, "workspace required");
    char* ws = (char*)workspace;
    float* ping = (float*)ws; ws += n * sizeof(float);
    float* range = (float*)ws; ws += n * sizeof(float);
    DlPartial* partials = (DlPartial*)(((uintptr_t)ws + 15) & ~(uintptr_t)15); ws = (char*)(partials + (size_t)B * DL_MAX_BLOCKS);
    float4* stats = (float4*)(((uintptr_t)ws + 15) & ~(uintptr_t)15);
    const int nblk = dl_blocks(h * w);
    const float* src = x;
    for (int it = 0; it < total; ++it) {
        int kh, kw;
        if (it < xy) { kh = 3; kw = 3; }                            // :126-130
        else if (it < xy + (y_iter - xy)) { kh = 3; kw = 1; }       // :132-136
        else { kh = 1; kw = 3; }                                    // :138-142
        // choose destinations so the last iteration lands in `out` and never aliases src
        float* dst = ((total - 1 - it) % 2 == 0) ? out : ping;
        if (dst == src) dst = (dst == out) ? ping : out;
        ProfScope ps(st, PC_DILATE, (double)n * 4 * 2);
        range_stats_kernel<<<dim3(nblk, B), DL_THREADS, 0, st>>>(src, range, partials, h, w);
        NB_LAUNCHED();
        range_finalize_kernel<<<B, 32, 0, st>>>(partials, nblk, h * w, stats);
        NB_LAUNCHED();
        dilate_apply_kernel<<<dim3(cdiv(h * w, DL_THREADS), B), DL_THREADS, 0, st>>>(src, range, stats, dst, h, w, kh, kw);
        NB_LAUNCHED();
        src = dst;
    }
    if (src != out) NB_CUDA(cudaMemcpyAsync(out, src, n * sizeof(float), cudaMemcpyDeviceToDevice, st));
    return 0;
}

static int minmax_map(const float* depth, int B, int n_per_frame, const nb200_mapper& mapper, float* out,
                      float* minmax_out, void* stream) {
    NB_CHECK(depth && out, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    const int nblk = dl_blocks(n_per_frame);
    float2* partials = nullptr;
    NB_CUDA(cudaMallocAsync((void**)&partials, (size_t)B * nblk * sizeof(float2), st));
    ProfScope ps(st, PC_MINMAX, (double)B * n_per_frame * 4 * 3);
    minmax_partial_kernel<<<dim3(nblk, B), DL_THREADS, 0, st>>>(depth, partials, n_per_frame);
    NB_LAUNCHED();
    minmax_apply_kernel<<<dim3(nblk, B), DL_THREADS, 0, st>>>(depth, partials, nblk, n_per_frame, mapper, out, minmax_out);
    NB_LAUNCHED();
    NB_CUDA(cudaFreeAsync(partials, st));
    return 0;
}

extern "C" int nb200_minmax_map(const float* depth, int B, int n_per_frame, float mapper_c, float* out,
                                float* minmax_out, void* stream) {
    return minmax_map(depth, B, n_per_frame, mapper_from_c(mapper_c), out, minmax_out, stream);
}

extern "C" int nb200_minmax_mapper(const float* depth, int B, int n_per_frame, const nb200_mapper* mapper_host, float* out,
                                   float* minmax_out, void* stream) {
    NB_CHECK(mapper_host, "null mapper");
    NB_CHECK(!*mapper_invalid(*mapper_host), mapper_invalid(*mapper_host));
    return minmax_map(depth, B, n_per_frame, *mapper_host, out, minmax_out, stream);
}
