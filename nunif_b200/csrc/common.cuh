// Shared helpers for the nunif_b200 CUDA sources (sm_90a only).
#pragma once
#include <cuda_runtime.h>
#include <cuda_fp16.h>
#include <stdint.h>
#include <stdio.h>
#include <string>
#include <atomic>

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

// seam_blend.cu: rows [y0, y1) of the blended output (used by the band-pipelined host render in model.cu)
int tile_gather_blend_rows(const void* z_all, int z_f32, int C, const ::nb200_tile_config* cfg, int scale, int offset, int tile_size,
                           int blend_size, float* out, int y0, int y1, void* stream);

// Programmatic dependent launch (sm_90+): a kernel that executes this lets a PDL-attributed successor (the
// GEMM, gemm.cu launch_t) be scheduled as soon as every CTA of this grid has issued it or exited; the successor blocks in
// griddepcontrol.wait until this grid has completed and flushed.  A no-op for ordinary successors.
#define NB_PDL_TRIGGER() asm volatile("griddepcontrol.launch_dependents;" ::: "memory")

// cudaFuncAttributeMaxDynamicSharedMemorySize is a PER-DEVICE attribute: cache the configured size per (device, function)
// (api.cu).  Thread-safe; a second device in the same process gets its own opt-in.
int ensure_dyn_smem(const void* func, size_t bytes);
// multiprocessor count of the CURRENT device (cached per device)
int device_sm_count();

inline int cdiv(int a, int b) { return (a + b - 1) / b; }
inline int64_t cdiv64(int64_t a, int64_t b) { return (a + b - 1) / b; }

__device__ __forceinline__ float clamp01(float v) { return fminf(fmaxf(v, 0.f), 1.f); }

}  // namespace nb200
