// Stateful depth normaliser of iw3: MinMaxBuffer + EMAMinMaxScaler (iw3/depth_scaler.py:33-142) with the whole state on
// the device.  The reference keeps min/max as 0-dim tensors but branches on them on the host (`if scale > 0`, .to(device)):
// one sync per frame.  Here a frame costs three small launches and no sync:
//   ema_reduce_kernel     per-block (min, max) of the new frame
//   ema_step_kernel       MinMaxBuffer.add (:46-58: the first add fills every slot, later adds are ring writes), ring
//                         amin/amax (:63-64), EMA update min = decay*min + (1-decay)*new (:108-113, fp32 like torch)
//   ema_normalize_kernel  (x - min) / (max - min) clamp[0,1] (:4-17) or x / max (:20-31) with the DEVICE-resident values,
//                         optionally followed by the disparity mapper (iw3/mapper.py, csrc/mapper.cuh)
// Whether the look-ahead buffer is filled (and so whether a frame comes out) depends only on call counts: the host
// mirror (nunif_b200/iw3/depth_scaler.py) tracks that without reading the device.
#include "common.cuh"
#include "mapper.cuh"
#include "../../include/nunif_b200.h"

namespace nb200 {
namespace {

constexpr int ER_THREADS = 256, ER_MAX_BLOCKS = 256;

__device__ __forceinline__ void block_minmax(float& mn, float& mx) {
    __shared__ float s_mn[ER_THREADS / 32], s_mx[ER_THREADS / 32];
    mn = warp_min(mn); mx = warp_max(mx);
    if ((threadIdx.x & 31) == 0) { s_mn[threadIdx.x >> 5] = mn; s_mx[threadIdx.x >> 5] = mx; }
    __syncthreads();
    if (threadIdx.x < 32) {
        mn = threadIdx.x < ER_THREADS / 32 ? s_mn[threadIdx.x] : __int_as_float(0x7f800000);
        mx = threadIdx.x < ER_THREADS / 32 ? s_mx[threadIdx.x] : __int_as_float(0xff800000);
        mn = warp_min(mn); mx = warp_max(mx);
    }
    __syncthreads();
}

__global__ void __launch_bounds__(ER_THREADS) ema_reduce_kernel(const float* __restrict__ x, int n, float2* __restrict__ partials) {
    float mn = __int_as_float(0x7f800000), mx = __int_as_float(0xff800000);
    for (int i = blockIdx.x * ER_THREADS + threadIdx.x; i < n; i += gridDim.x * ER_THREADS) {
        const float v = __ldg(x + i);
        mn = fminf(mn, v); mx = fmaxf(mx, v);
    }
    block_minmax(mn, mx);
    if (threadIdx.x == 0) partials[blockIdx.x] = make_float2(mn, mx);
}

// state: [0] min_value [1] max_value [2] ring amin [3] ring amax | ring at [4 .. 4 + size)
__global__ void __launch_bounds__(ER_THREADS) ema_step_kernel(float* __restrict__ state, const float2* __restrict__ partials, int nblk,
                                                              int count_before, int size, float decay, float one_minus_decay,
                                                              int filled, int first) {
    float mn = __int_as_float(0x7f800000), mx = __int_as_float(0xff800000);
    for (int i = threadIdx.x; i < nblk; i += ER_THREADS) { const float2 p = partials[i]; mn = fminf(mn, p.x); mx = fmaxf(mx, p.y); }
    block_minmax(mn, mx);
    __shared__ float s_new[2];
    if (threadIdx.x == 0) { s_new[0] = mn; s_new[1] = mx; }
    __syncthreads();
    mn = s_new[0]; mx = s_new[1];
    float* ring = state + 4;
    if (count_before == 0) {                       // MinMaxBuffer._fill (:51-53)
        for (int i = threadIdx.x; i < size; i += ER_THREADS) ring[i] = (i & 1) ? mx : mn;
    } else if (threadIdx.x == 0) {                 // two ring writes (:46-49)
        ring[count_before % size] = mn;
        ring[(count_before + 1) % size] = mx;
    }
    __syncthreads();
    float rmn = __int_as_float(0x7f800000), rmx = __int_as_float(0xff800000);
    for (int i = threadIdx.x; i < size; i += ER_THREADS) { const float v = ring[i]; rmn = fminf(rmn, v); rmx = fmaxf(rmx, v); }
    block_minmax(rmn, rmx);
    if (threadIdx.x == 0) {
        state[2] = rmn; state[3] = rmx;
        if (filled) {
            if (first) { state[0] = rmn; state[1] = rmx; }
            else {   // torch: python-float * fp32 0-dim tensor -> fp32 multiply, then an fp32 add (no FMA contraction)
                state[0] = __fadd_rn(__fmul_rn(decay, state[0]), __fmul_rn(one_minus_decay, rmn));
                state[1] = __fadd_rn(__fmul_rn(decay, state[1]), __fmul_rn(one_minus_decay, rmx));
            }
        }
    }
}

// mode 0: minmax_normalize, 1: max_normalize; mm == nullptr: no normalisation (mapper only)
__global__ void __launch_bounds__(ER_THREADS) ema_normalize_kernel(const float* __restrict__ x, int n, const float* __restrict__ mm, int mode,
                                                                   const nb200_mapper mapper, float* __restrict__ out,
                                                                   float* __restrict__ mm_out) {
    float mn = 0.f, mx = 0.f;
    if (mm) { mn = mm[0]; mx = mm[1]; }
    if (mm_out && blockIdx.x == 0 && threadIdx.x == 0) { mm_out[0] = mn; mm_out[1] = mx; }
    const float scale = mode == 0 ? mx - mn : mx;
    for (int i = blockIdx.x * ER_THREADS + threadIdx.x; i < n; i += gridDim.x * ER_THREADS) {
        float v = x[i];
        if (mm) {
            if (scale > 0.f) v = mode == 0 ? (v - mn) / scale : v / scale;
            v = clamp01(v);
        }
        out[i] = mapper_eval(mapper, v);
    }
}

int er_blocks(int n) { int nb = cdiv(n, ER_THREADS * 4); return nb < 1 ? 1 : (nb > ER_MAX_BLOCKS ? ER_MAX_BLOCKS : nb); }

}  // namespace
}  // namespace nb200

using namespace nb200;

struct nb200_ema_scaler {
    int buffer_size = 1, mode = 0, count = 0, has_value = 0;
    double decay = 0.0;
    float* state = nullptr;      // 4 + 2*buffer_size floats
    float2* partials = nullptr;  // ER_MAX_BLOCKS
    int cap = 0;
};

static int ema_alloc(nb200_ema_scaler* s) {
    const int need = 4 + 2 * s->buffer_size;
    if (need > s->cap) {
        if (s->state) cudaFree(s->state);
        s->state = nullptr; s->cap = 0;
        NB_CUDA(cudaMalloc((void**)&s->state, (size_t)need * sizeof(float)));
        s->cap = need;
    }
    if (!s->partials) NB_CUDA(cudaMalloc((void**)&s->partials, ER_MAX_BLOCKS * sizeof(float2)));
    return 0;
}

extern "C" int nb200_ema_scaler_create(int buffer_size, double decay, int mode, nb200_ema_scaler** out) {
    NB_CHECK(out, "null pointer");
    NB_CHECK(buffer_size > 0, "buffer_size must be positive");              // depth_scaler.py:73
    NB_CHECK(mode == 0 || mode == 1, "mode: 0 = minmax, 1 = max");
    auto* s = new nb200_ema_scaler();
    s->buffer_size = buffer_size; s->decay = decay; s->mode = mode;
    if (ema_alloc(s)) { delete s; return 1; }
    *out = s;
    return 0;
}

extern "C" void nb200_ema_scaler_destroy(nb200_ema_scaler* s) {
    if (!s) return;
    if (s->state) cudaFree(s->state);
    if (s->partials) cudaFree(s->partials);
    delete s;
}

// EMAMinMaxScaler.reset (:76-86): decay < 0 / buffer_size <= 0 keep the current setting
extern "C" int nb200_ema_scaler_reset(nb200_ema_scaler* s, double decay, int buffer_size) {
    NB_CHECK(s, "null scaler");
    if (decay >= 0.0) s->decay = decay;
    if (buffer_size > 0) s->buffer_size = buffer_size;
    s->count = 0; s->has_value = 0;
    return ema_alloc(s);
}

// EMAMinMaxScaler.update up to the `is_filled` test (:94-113): *filled = a frame can be normalised now
extern "C" int nb200_ema_scaler_update(nb200_ema_scaler* s, const float* frame, int n, int* filled, void* stream) {
    NB_CHECK(s && frame && filled, "null pointer");
    NB_CHECK(n > 0, "empty frame");
    cudaStream_t st = (cudaStream_t)stream;
    const int size = 2 * s->buffer_size, nblk = er_blocks(n);
    const int count_after = s->count == 0 ? 2 : s->count + 2;
    const int fl = count_after >= size ? 1 : 0;                             // MinMaxBuffer.is_filled (:60-61)
    const int first = fl && !s->has_value;
    ProfScope ps(st, PC_MINMAX, (double)n * 4);
    ema_reduce_kernel<<<nblk, ER_THREADS, 0, st>>>(frame, n, s->partials);
    NB_LAUNCHED();
    ema_step_kernel<<<1, ER_THREADS, 0, st>>>(s->state, s->partials, nblk, s->count, size, (float)s->decay, (float)(1.0 - s->decay), fl, first);
    NB_LAUNCHED();
    s->count = count_after;
    if (fl) s->has_value = 1;
    *filled = fl;
    return 0;
}

// normalise a frame with the scaler's values: from_ring = 0 -> the EMA min/max (:115-116), 1 -> the ring's amin/amax
// (flush before any EMA value exists, :127-128).  mapper_c < 0: no mapper.  minmax_out: optional 2 floats (device).
extern "C" int nb200_ema_scaler_normalize(nb200_ema_scaler* s, const float* frame, int n, int from_ring, float mapper_c, float* out,
                                          float* minmax_out, void* stream) {
    NB_CHECK(s && frame && out, "null pointer");
    NB_CHECK(n > 0, "empty frame");
    NB_CHECK(s->count > 0, "normalize before any update");
    NB_CHECK(from_ring || s->has_value, "the look-ahead buffer is not filled yet");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope ps(st, PC_MINMAX, (double)n * 8);
    ema_normalize_kernel<<<er_blocks(n), ER_THREADS, 0, st>>>(frame, n, s->state + (from_ring ? 2 : 0), s->mode, mapper_from_c(mapper_c),
                                                              out, minmax_out);
    NB_LAUNCHED();
    return 0;
}

static int mapper_apply(const float* depth, long long n, const nb200_mapper& mapper, float* out, void* stream) {
    NB_CHECK(depth && out, "null pointer");
    NB_CHECK(n > 0 && n < (1ll << 31), "bad size");
    cudaStream_t st = (cudaStream_t)stream;
    ema_normalize_kernel<<<er_blocks((int)n), ER_THREADS, 0, st>>>(depth, (int)n, nullptr, 0, mapper, out, nullptr);
    NB_LAUNCHED();
    return 0;
}

// disparity mapper alone (iw3/mapper.py:29-32 div_*: distance_to_disparity(x, c)); in place allowed
extern "C" int nb200_depth_mapper(const float* depth, long long n, float mapper_c, float* out, void* stream) {
    NB_CHECK(mapper_c >= 0.f, "mapper constant must be >= 0");
    return mapper_apply(depth, n, mapper_from_c(mapper_c), out, stream);
}

// any mapper alone (iw3/mapper.py:129-151 get_mapper(name)(x)); in place allowed
extern "C" int nb200_mapper_apply(const float* depth, long long n, const nb200_mapper* mapper_host, float* out, void* stream) {
    NB_CHECK(mapper_host, "null mapper");
    NB_CHECK(!*mapper_invalid(*mapper_host), mapper_invalid(*mapper_host));
    return mapper_apply(depth, n, *mapper_host, out, stream);
}
