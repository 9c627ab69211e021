// Shared helpers for the nunif_b200 CUDA sources (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <atomic>
#include <initializer_list>
#include <type_traits>

struct nb200_tile_config;  // include/nunif_b200.h

namespace nb200 {

extern thread_local std::string g_last_error;
extern std::atomic<uint64_t> g_launches;

inline int fail(const std::string& msg) {
    g_last_error = msg;
    return 1;
}

#define NB_CHECK(cond, msg)                                                     \
    do {                                                                        \
        if (!(cond)) return ::nb200::fail(std::string(__func__) + ": " + (msg)); \
    } while (0)

#define NB_CUDA(expr)                                                                      \
    do {                                                                                   \
        cudaError_t _e = (expr);                                                           \
        if (_e != cudaSuccess)                                                             \
            return ::nb200::fail(std::string(__func__) + ": " #expr " -> " + cudaGetErrorString(_e)); \
    } while (0)

// call after every kernel launch: counts it and surfaces launch-config errors
#define NB_LAUNCHED()                                                                      \
    do {                                                                                   \
        ::nb200::g_launches.fetch_add(1, std::memory_order_relaxed);                       \
        cudaError_t _e = cudaGetLastError();                                               \
        if (_e != cudaSuccess)                                                             \
            return ::nb200::fail(std::string(__func__) + ": launch -> " + cudaGetErrorString(_e)); \
    } while (0)

// ---- optional in-library kernel timing (bench.py roofline): CUDA events around each launch
enum ProfCat : int { PC_GEMM = 0, PC_ATTN, PC_STEM, PC_TOIMG, PC_UNFOLD, PC_BLEND, PC_SE, PC_TAIL, PC_WARP_FW, PC_WARP_BW,
                     PC_DILATE, PC_MINMAX, PC_OTHER, PC_FUSED_MLP, PC_FUSED_ATTN, PC_HOLE_MASK, PC_COUNT };
extern std::atomic<int> g_prof_enabled;
void prof_begin(cudaStream_t st, int cat, double work, double rbytes, double wbytes);
void prof_end(cudaStream_t st);
struct ProfScope {
    cudaStream_t st;
    bool on;
    // work = FLOPs (tensor-bound classes) or algorithmic bytes; rbytes/wbytes = algorithmic HBM reads/writes (0 = unknown)
    ProfScope(cudaStream_t s, int cat, double work, double rbytes = 0, double wbytes = 0)
        : st(s), on(g_prof_enabled.load(std::memory_order_relaxed) != 0) {
        if (on) prof_begin(st, cat, work, rbytes, wbytes);
    }
    ~ProfScope() {
        if (on) prof_end(st);
    }
};

// ---- optional launch recorder (nb200_record_launches): the host code of the recorded kernels appends one line per launch
// describing it without its pointers, so tests can replay every configuration a network uses.  The recorder's mask selects
// the kinds: REC_GEMMS the GEMM, ViT attention and fused Swin block; REC_AUX the WABlock core, add + LayerNorm, DPT upsample
// and ZoeDepth bins head; REC_CONV the waifu2x stem / tail / head convolutions, the SE block, to_image and the SOD REBNCONV;
// REC_STEREO the input / output stages of row_flow_v3, mlbw and depth_aa, the fused row_flow_v2 kernel and the hole mask;
// REC_WARP the backward and forward stereo warps and the antialiased depth resize; REC_DEPTH the depth networks' patch
// embedding, token assembly, hook cast and readout concat, and the DPT reassemble, fusion and output kernels.
enum { REC_GEMMS = 1, REC_AUX = 2, REC_CONV = 4, REC_STEREO = 8, REC_WARP = 16, REC_DEPTH = 32 };
extern std::atomic<int> g_rec_enabled;
inline bool rec_on(int kinds = REC_GEMMS) { return (g_rec_enabled.load(std::memory_order_relaxed) & kinds) != 0; }
// one field of a recorded line: integers and flags print as integers, floating-point values with 9 significant digits
struct RecField {
    const char* name;
    std::string value;
    template <typename T, typename std::enable_if<std::is_integral<T>::value, int>::type = 0>
    RecField(const char* n, T v) : name(n), value(std::to_string(v)) {}
    RecField(const char* n, double v);
};
// appends the line `kind,name=value,...`; the call sites are the record format's only definition
void rec_launch(const char* kind, std::initializer_list<RecField> fields);

// debug taps (nb200_debug_tap, model.cu) that a kernel writes itself: *buf = the armed buffer when tap `id` is armed, else
// null; an armed buffer smaller than `bytes` is refused
int debug_tap_target(int id, size_t bytes, void** buf);

// seam_blend.cu: rows [y0, y1) of the blended output (used by the band-pipelined host render in model.cu)
int tile_gather_blend_rows(const void* z_all, int z_f32, int C, const ::nb200_tile_config* cfg, int scale, int offset, int tile_size,
                           int blend_size, float* out, int y0, int y1, void* stream);

// Programmatic dependent launch (sm_90+): a kernel that executes this lets a PDL-attributed successor (the
// GEMM, gemm.cu launch_t) be scheduled as soon as every CTA of this grid has issued it or exited; the successor blocks in
// griddepcontrol.wait until this grid has completed and flushed.  A no-op for ordinary successors.
#define NB_PDL_TRIGGER() asm volatile("griddepcontrol.launch_dependents;" ::: "memory")

// cudaFuncAttributeMaxDynamicSharedMemorySize is a PER-DEVICE attribute: cache the configured size per (device, function)
// (api.cu).  Thread-safe; a second device in the same process gets its own opt-in.  carveout > 0 also sets the function's
// preferred shared-memory carveout (percent, also per device), again whenever it changes.  The carveout form is hidden so
// that the library's dynamic symbol table does not depend on it.
int ensure_dyn_smem(const void* func, size_t bytes);
__attribute__((visibility("hidden"))) int ensure_dyn_smem(const void* func, size_t bytes, int carveout);
// multiprocessor count of the CURRENT device (cached per device)
int device_sm_count();

inline int cdiv(int a, int b) { return (a + b - 1) / b; }
inline int64_t cdiv64(int64_t a, int64_t b) { return (a + b - 1) / b; }

__device__ __forceinline__ float clamp01(float v) { return fminf(fmaxf(v, 0.f), 1.f); }

// full-warp xor butterflies: every lane gets the reduction over all 32 lanes
template <typename T>
__device__ __forceinline__ T warp_sum(T v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
    return v;
}
__device__ __forceinline__ float warp_min(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fminf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}
__device__ __forceinline__ float warp_max(float v) {
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) v = fmaxf(v, __shfl_xor_sync(0xffffffffu, v, o));
    return v;
}

// v rounded to fp16 and back: where the reference stores an fp16 tensor
__host__ __device__ __forceinline__ float round_f16(float v) { return __half2float(__float2half_rn(v)); }

// order-preserving float -> uint key (unsigned order = float order for non-NaN values, -0 below +0; every such key > 0)
// and its inverse
__device__ __forceinline__ uint32_t order_key(float f) {
    const uint32_t u = __float_as_uint(f);
    return (u & 0x80000000u) ? ~u : (u | 0x80000000u);
}
__device__ __forceinline__ float order_key_inv(uint32_t k) { return __uint_as_float((k & 0x80000000u) ? (k & 0x7fffffffu) : ~k); }

// Philox4x32-10 (Salmon et al., "Parallel random numbers: as easy as 1, 2, 3", SC'11): four 32-bit words that are a pure
// function of a 128-bit counter and a 64-bit key, so any element of a random field can be recomputed by any thread
__host__ __device__ __forceinline__ uint4 philox4x32_10(uint4 c, uint2 k) {
#pragma unroll
    for (int i = 0; i < 10; ++i) {
        const uint64_t p0 = (uint64_t)0xD2511F53u * c.x, p1 = (uint64_t)0xCD9E8D57u * c.z;
        c = make_uint4((uint32_t)(p1 >> 32) ^ c.y ^ k.x, (uint32_t)p1, (uint32_t)(p0 >> 32) ^ c.w ^ k.y, (uint32_t)p0);
        k.x += 0x9E3779B9u;
        k.y += 0xBB67AE85u;
    }
    return c;
}

// ATen's CUDA bilinear resize (align_corners=False, no antialias, output size given), UpSampleBilinear2d.cu: the scale is
// (float)in / out, the source index scale * (dst + 0.5) - 0.5 is one FMA there, clamped at 0, and so is the first product
// of each lerp pair.  Used by the sod_v1 resizes (sod.cu) and the NULL depth model (null_depth.cu).
struct BilTap {
    int i0, i1;
    float l0, l1;
};

__device__ __forceinline__ BilTap bil_tap(float scale, int dst, int in_size) {
    float r = fmaf(scale, (float)dst + 0.5f, -0.5f);
    r = r < 0.f ? 0.f : r;
    BilTap t;
    t.i0 = (int)r;
    t.i1 = t.i0 + ((t.i0 < in_size - 1) ? 1 : 0);
    t.l1 = r - (float)t.i0;
    t.l0 = 1.f - t.l1;
    return t;
}

__device__ __forceinline__ float bil_mix(const BilTap& ty, const BilTap& tx, float v00, float v01, float v10, float v11) {
    return fmaf(ty.l0, fmaf(tx.l0, v00, tx.l1 * v01), ty.l1 * fmaf(tx.l0, v10, tx.l1 * v11));
}

// bicubic weight with A = -0.5 (ATen's antialiased bicubic filter)
__device__ __forceinline__ float cubic_aa(float x) {
    const float a = -0.5f;
    x = fabsf(x);
    if (x < 1.f) return ((a + 2.f) * x - (a + 3.f)) * x * x + 1.f;
    if (x < 2.f) return (((x - 5.f) * x + 8.f) * x - 4.f) * a;
    return 0.f;
}

}  // namespace nb200
