// The autocrop detector (nunif/utils/autocrop.py:6-207): per-row (detect_tb) and per-column (detect_lr) bar masks of an fp32
// RGB frame, the device-resident bar counts of AutoCropDetector.update, and the first / last non-bar index of get_crop.
//   Y = r*0.299 + g*0.587 + b*0.114, each op rounded like ATen's elementwise kernels (no FMA contraction);
//   black modes: Y clamped to [16/255, 235/255]; bar = mean <= 32/255 && max|Y - mean| < 16/255.  fl(Y - mean) is monotonic
//     in Y, so the max deviation is max(|fl(ymax - mean)|, |fl(ymin - mean)|): sum, min and max per line are enough.  The
//     mean is sum * fl(1/n) like ATen's CUDA MeanOps; only the summation order differs from torch.
//   flat modes: bar = fl(count(|fl(Y - median)| < 16/255) * fl(1/n)) > 0.99 with the exact lower median (element (n-1)/2
//     of the sorted line, torch.median), found by a 4 x 8-bit radix select on the float bits in shared memory.
// One warp per line.  Rows are read straight from the planes; columns are staged 8 at a time (one 32-byte sector per row) in
// shared memory so that their reads stay coalesced.  Rows and columns each read the frame once; black mode is HBM-bound,
// the flat-mode select is bound by shared memory.
#include "common.cuh"
#include "../../include/nunif_b200.h"

namespace nb200 {

constexpr int AC_ROW_WARPS = 4;   // rows per block (flat mode stages 4 rows: 60 KB at W = 3840)
constexpr int AC_COLS = 8;        // columns per block: one 32-byte sector of each row
constexpr int AC_SMEM_MAX = 200 * 1024;

struct AutocropParams {
    const float* x;
    int B, H, W, black;
    float lo, hi;                        // TV-range clamp
    float factor_row, factor_col;        // ATen's MeanOps factor: fl(out / numel) = fl(1 / n)
    unsigned char* mask_tb;              // [B][H] or NULL
    unsigned char* mask_lr;              // [B][W] or NULL
    int* count_tb;                       // [H] or NULL, += mask over the B frames
    int* count_lr;                       // [W] or NULL
    float* stat_tb;                      // [B][H] or NULL: black: the mean, flat: the lower median
    float* stat_lr;                      // [B][W] or NULL
};

__device__ __forceinline__ float luma(const float* p, size_t plane, const AutocropParams& a) {
    // torch: r * 0.299 + g * 0.587 + b * 0.114 as three multiplies and two adds, then clamp(min, max)
    const float y = __fadd_rn(__fadd_rn(__fmul_rn(__ldg(p), 0.299f), __fmul_rn(__ldg(p + plane), 0.587f)),
                              __fmul_rn(__ldg(p + 2 * plane), 0.114f));
    return a.black ? fminf(fmaxf(y, a.lo), a.hi) : y;
}

// element k of the sorted v[0..n) (one warp; hist: 256 words of this warp's shared memory)
__device__ float warp_select(const float* v, int n, unsigned k, unsigned* hist) {
    const int lane = threadIdx.x & 31;
    unsigned prefix = 0u, mask = 0u;
    for (int shift = 24; shift >= 0; shift -= 8) {
        for (int i = lane; i < 256; i += 32) hist[i] = 0u;
        __syncwarp();
        for (int base = 0; base < n; base += 32) {
            const int i = base + lane;
            unsigned digit = 256u;                       // no bin
            if (i < n) {
                const unsigned key = order_key(v[i]);
                if ((key & mask) == prefix) digit = (key >> shift) & 255u;
            }
            // equal digits are frequent (a bar is one value): one shared atomic per distinct digit
            const unsigned peers = __match_any_sync(0xffffffffu, digit);
            if (digit < 256u && lane == __ffs(peers) - 1) atomicAdd(&hist[digit], (unsigned)__popc(peers));
        }
        __syncwarp();
        unsigned c[8], s = 0u;
#pragma unroll
        for (int j = 0; j < 8; ++j) { c[j] = hist[lane * 8 + j]; s += c[j]; }
        unsigned incl = s;
#pragma unroll
        for (int o = 1; o < 32; o <<= 1) {
            const unsigned t = __shfl_up_sync(0xffffffffu, incl, o);
            if (lane >= o) incl += t;
        }
        const unsigned excl = incl - s;
        const int src = __ffs(__ballot_sync(0xffffffffu, excl <= k && k < incl)) - 1;
        unsigned bin = 0u, below = excl;
        if (lane == src) {
#pragma unroll
            for (int j = 0; j < 8; ++j) {
                if (k < below + c[j]) { bin = lane * 8 + j; break; }
                below += c[j];
            }
        }
        bin = __shfl_sync(0xffffffffu, bin, src);
        below = __shfl_sync(0xffffffffu, below, src);
        k -= below;
        prefix |= bin << shift;
        mask |= 255u << shift;
        __syncwarp();
    }
    return order_key_inv(prefix);
}

// black-mode decision from the line's sum, min and max
__device__ __forceinline__ bool black_bar(float sum, float mn, float mx, float factor, float* mean_out) {
    const float mean = __fmul_rn(sum, factor);
    *mean_out = mean;
    const float dev = fmaxf(fabsf(__fsub_rn(mx, mean)), fabsf(__fsub_rn(mn, mean)));
    return mean <= (float)(32.0 / 255.0) && dev < (float)(16.0 / 255.0);
}

// flat-mode decision for the staged line v[0..n): the lower median and the share of values within 16/255 of it
__device__ __forceinline__ bool flat_bar(const float* v, int n, float factor, unsigned* hist, float* median_out) {
    const int lane = threadIdx.x & 31;
    const float med = warp_select(v, n, (unsigned)(n - 1) / 2u, hist);
    *median_out = med;
    int cnt = 0;
    for (int i = lane; i < n; i += 32) cnt += fabsf(__fsub_rn(v[i], med)) < (float)(16.0 / 255.0) ? 1 : 0;
    cnt = warp_sum(cnt);
    // (diff < t).float().mean(): an exact count times fl(1/n) (ATen's CUDA mean), compared with fl(0.99)
    return __fmul_rn((float)cnt, factor) > 0.99f;
}

__device__ __forceinline__ void emit(bool bar, float stat, int b, int i, int n, unsigned char* mask, int* count, float* st) {
    if (mask) mask[(size_t)b * n + i] = bar ? 1 : 0;
    if (st) st[(size_t)b * n + i] = stat;
    if (count && bar) atomicAdd(count + i, 1);
}

// grid (ceil(H / AC_ROW_WARPS), B); one warp per row
__global__ void __launch_bounds__(AC_ROW_WARPS * 32) autocrop_rows_kernel(AutocropParams a) {
    extern __shared__ float smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int y = blockIdx.x * AC_ROW_WARPS + warp, b = blockIdx.y;
    if (y >= a.H) return;
    const size_t plane = (size_t)a.H * a.W;
    const float* row = a.x + (size_t)b * 3 * plane + (size_t)y * a.W;
    float stat;
    bool bar;
    if (a.black) {
        float s = 0.f, mn = INFINITY, mx = -INFINITY;
        for (int i = lane; i < a.W; i += 32) {
            const float v = luma(row + i, plane, a);
            s += v; mn = fminf(mn, v); mx = fmaxf(mx, v);
        }
        bar = black_bar(warp_sum(s), warp_min(mn), warp_max(mx), a.factor_row, &stat);
    } else {
        unsigned* hist = reinterpret_cast<unsigned*>(smem) + warp * 256;
        float* v = smem + AC_ROW_WARPS * 256 + (size_t)warp * a.W;
        for (int i = lane; i < a.W; i += 32) v[i] = luma(row + i, plane, a);
        __syncwarp();
        bar = flat_bar(v, a.W, a.factor_row, hist, &stat);
    }
    if (lane == 0) emit(bar, stat, b, y, a.H, a.mask_tb, a.count_tb, a.stat_tb);
}

// grid (ceil(W / AC_COLS), B); the block stages columns [x0, x0 + 8) of every row, then one warp per column
__global__ void __launch_bounds__(AC_COLS * 32) autocrop_cols_kernel(AutocropParams a) {
    extern __shared__ float smem[];
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    const int x0 = blockIdx.x * AC_COLS, b = blockIdx.y;
    const int ncol = min(AC_COLS, a.W - x0);
    const size_t plane = (size_t)a.H * a.W;
    const float* img = a.x + (size_t)b * 3 * plane + x0;
    unsigned* hist = reinterpret_cast<unsigned*>(smem) + warp * 256;
    float* tile = smem + AC_COLS * 256;                  // [8][H]: column-major so each warp's line is contiguous
    for (int t = threadIdx.x; t < a.H * AC_COLS; t += blockDim.x) {
        const int c = t % AC_COLS, yy = t / AC_COLS;
        if (c < ncol) tile[(size_t)c * a.H + yy] = luma(img + (size_t)yy * a.W + c, plane, a);
    }
    __syncthreads();
    if (warp >= ncol) return;
    const float* v = tile + (size_t)warp * a.H;
    float stat;
    bool bar;
    if (a.black) {
        float s = 0.f, mn = INFINITY, mx = -INFINITY;
        for (int i = lane; i < a.H; i += 32) { const float t = v[i]; s += t; mn = fminf(mn, t); mx = fmaxf(mx, t); }
        bar = black_bar(warp_sum(s), warp_min(mn), warp_max(mx), a.factor_col, &stat);
    } else {
        bar = flat_bar(v, a.H, a.factor_col, hist, &stat);
    }
    if (lane == 0) emit(bar, stat, b, x0 + warp, a.W, a.mask_lr, a.count_lr, a.stat_lr);
}

// blockIdx.x = 0: rows, 1: columns.  bar_i = fl(count_i * fl(1 / frame_count)) >= threshold (ATen's CUDA true division by a
// host scalar multiplies by its reciprocal); out[2 axis], out[2 axis + 1] = first / last non-bar index, -1 if none.
__global__ void __launch_bounds__(256) autocrop_bounds_kernel(const int* __restrict__ count_tb, int H, const int* __restrict__ count_lr,
                                                              int W, float inv_frames, float threshold, int* __restrict__ out) {
    __shared__ int first, last;
    const int* c = blockIdx.x ? count_lr : count_tb;
    const int n = blockIdx.x ? W : H;
    if (threadIdx.x == 0) { first = INT_MAX; last = -1; }
    __syncthreads();
    if (c) {
        int f = INT_MAX, l = -1;
        for (int i = threadIdx.x; i < n; i += blockDim.x) {
            if (!(__fmul_rn((float)c[i], inv_frames) >= threshold)) { f = min(f, i); l = max(l, i); }
        }
        if (l >= 0) { atomicMin(&first, f); atomicMax(&last, l); }
    }
    __syncthreads();
    if (threadIdx.x == 0) {
        out[2 * blockIdx.x] = last >= 0 ? first : -1;
        out[2 * blockIdx.x + 1] = last;
    }
}

}  // namespace nb200

using namespace nb200;

static size_t row_smem(int W) { return (size_t)AC_ROW_WARPS * (256 + (size_t)W) * 4; }
static size_t col_smem(int H) { return (size_t)AC_COLS * (256 + (size_t)H) * 4; }

extern "C" int nb200_autocrop_detect(const float* x, int B, int H, int W, int black, int axes, unsigned char* mask_tb,
                                     unsigned char* mask_lr, int* count_tb, int* count_lr, float* stat_tb, float* stat_lr,
                                     void* stream) {
    NB_CHECK(x, "null pointer");
    NB_CHECK(B > 0 && B <= 65535 && H > 0 && W > 0, "bad shape");
    NB_CHECK(axes >= 1 && axes <= 3, "axes must be 1 (rows), 2 (columns) or 3 (both)");
    NB_CHECK(black || (row_smem(W) <= AC_SMEM_MAX && col_smem(H) <= AC_SMEM_MAX), "frame too large for the flat-mode median");
    NB_CHECK(col_smem(H) <= AC_SMEM_MAX, "frame too tall for the column pass");
    AutocropParams a;
    a.x = x; a.B = B; a.H = H; a.W = W; a.black = black ? 1 : 0;
    a.lo = (float)(16.0 / 255.0); a.hi = (float)(235.0 / 255.0);
    const float numel = (float)((long long)H * W);       // ATen: static_cast<float>(num_output_elements) / numel
    a.factor_row = (float)H / numel;
    a.factor_col = (float)W / numel;
    a.mask_tb = mask_tb; a.mask_lr = mask_lr; a.count_tb = count_tb; a.count_lr = count_lr; a.stat_tb = stat_tb; a.stat_lr = stat_lr;
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope ps(st, PC_OTHER, (double)B * H * W * 12 * ((axes & 1) + ((axes >> 1) & 1)));
    if (axes & 1) {
        const size_t sm = a.black ? 0 : row_smem(W);
        if (sm > 48 * 1024) NB_CUDA(cudaFuncSetAttribute(autocrop_rows_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
        autocrop_rows_kernel<<<dim3(cdiv(H, AC_ROW_WARPS), B), AC_ROW_WARPS * 32, sm, st>>>(a);
        NB_LAUNCHED();
    }
    if (axes & 2) {
        const size_t sm = col_smem(H);
        if (sm > 48 * 1024) NB_CUDA(cudaFuncSetAttribute(autocrop_cols_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)sm));
        autocrop_cols_kernel<<<dim3(cdiv(W, AC_COLS), B), AC_COLS * 32, sm, st>>>(a);
        NB_LAUNCHED();
    }
    return 0;
}

extern "C" int nb200_autocrop_bounds(const int* count_tb, int H, const int* count_lr, int W, int frame_count, float threshold,
                                     int* out, void* stream) {
    NB_CHECK(out && (count_tb || count_lr), "null pointer");
    NB_CHECK(H > 0 && W > 0 && frame_count > 0, "bad shape");
    const float inv_frames = 1.0f / (float)frame_count;
    autocrop_bounds_kernel<<<2, 256, 0, (cudaStream_t)stream>>>(count_tb, H, count_lr, W, inv_frames, threshold, out);
    NB_LAUNCHED();
    return 0;
}
