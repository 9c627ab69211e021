// wgmma implicit-GEMM for NHWC fp16 activations (sm_90a).
//
//   D[m, n] = act( sum_taps sum_c A[pixel(m) + tap, c] * Wt[n, tap, c] + bias[n] ) (+ residual)
//
// One kernel covers every dense contraction on path A:
//   * Linear layers of the Swin blocks (1 tap, "pixel" = token)            swin_transformer.py:177,228,444
//   * 3x3 valid convolutions of CUNet / the Swin patch stem (9 taps)       cunet.py:14-17,38,41 ; swin_unet.py:133-136
//   * 2x2 stride-2 convolutions (2 taps over a (2C, W/2, 2, H/2, B) view)  cunet.py:36,78,80 ; swin_unet.py:49
//   * ConvTranspose 2x2 s2 / Linear+pixel_shuffle(2) (N = 4*Cout, scatter) cunet.py:38,82,84 ; swin_unet.py:69-82
//
// Structure (Hopper):
//   warp 8     : TMA producer - one 5-D box load per (tap, channel chunk) for A, one 2-D box for B,
//                128B/64B hardware swizzle, mbarrier complete_tx
//   warps 0-7  : two consumer warpgroups; warpgroup g owns accumulator rows [64g, 64g+64) of the 128 x BLOCK_N tile and
//                issues wgmma.mma_async (M=64, N=BLOCK_N, K=16) straight from the swizzled stages, fp32 in registers.
//                Epilogue: bias + activation (+ residual tile fetched by TMA), fp16 results staged in swizzled shared
//                memory and written with TMA tensor stores (cp.async.bulk.tensor ... bulk_group), so every global access
//                of the kernel is a full-line bulk copy
// Non-persistent, one 128 x BLOCK_N output tile per CTA; shared memory and registers are sized so that two CTAs are
// co-resident per SM, which overlaps one tile's epilogue with the next tile's loads.
#pragma once
#include "common.cuh"
#include "gemm.h"
#include "ptx.cuh"
#include <cuda.h>

namespace nb200 {

struct GemmParams {
    // output tiling: the M dimension is (b, y, x) over Ho x Wo pixels, tiled TH x TW (TH*TW == 128)
    int B, Ho, Wo, TH, TW, tiles_x, tiles_y;
    int N;               // output channels (GEMM N)
    int taps, cpt;       // taps and BK-chunks per tap (K = taps*cpt*BK)
    int8_t tap_dx[16], tap_dy[16], tap_dyi[16];
    int n_tiles;
    // epilogue (output / residual tensors are described by the tensor maps in GemmMaps)
    const float* bias;   // [N] or null
    int act;
    int out_mode, cout;  // OUT_PIXSHUF2: N = 4*cout ordered (dy,dx,co); maps o[g]/r[g] are the stride-2 views
                         // OUT_SPLIT: N = nsplit*cout, block g goes to its own dense [M][cout] plane (maps o[g])
    int has_res, res_cy, res_cx;
    int res_before_act;  // 0: out = act(acc+bias) + res ; 1: out = act(acc+bias+res)
    int k2;              // OUT_PIXSHUF2 with a second A operand (maps.a2): its BK-chunks, after the taps*cpt of A
};

// All tensor maps of one launch (a single __grid_constant__ parameter).
struct GemmMaps {
    CUtensorMap a, b;
    CUtensorMap o[4];    // output: NHWC view (c, x, y, b); pixel-shuffle mode: one stride-2 view per (dy,dx)
    union {
        CUtensorMap r[4];    // residual, same tiling as the output
        CUtensorMap a2;      // or the second A operand (the two exclude each other): full-resolution pixels of a pixel-shuffle
                             // output as (c, dx, x, dy, b*Ho + y), stride-2 in x and y
    };
};

// ---------------------------------------------------------------------------------------------
// mbarrier and TMA wrappers (smem_u32 and the other generic PTX wrappers: ptx.cuh)
// ---------------------------------------------------------------------------------------------
__device__ __forceinline__ void mbar_init(uint64_t* bar, uint32_t count) {
    asm volatile("mbarrier.init.shared::cta.b64 [%0], %1;" ::"r"(smem_u32(bar)), "r"(count));
}
__device__ __forceinline__ void mbar_expect_tx(uint64_t* bar, uint32_t bytes) {
    asm volatile("mbarrier.arrive.expect_tx.shared::cta.b64 _, [%0], %1;" ::"r"(smem_u32(bar)), "r"(bytes) : "memory");
}
__device__ __forceinline__ void mbar_arrive(uint64_t* bar) {
    asm volatile("mbarrier.arrive.shared::cta.b64 _, [%0];" ::"r"(smem_u32(bar)) : "memory");
}
__device__ __forceinline__ void mbar_wait(uint64_t* bar, uint32_t parity) {
    const uint32_t addr = smem_u32(bar);
    uint32_t done = 0;
    // try_wait WITH a suspend-time hint: the thread sleeps in hardware until the phase completes (or 20 us pass) instead of
    // re-issuing the instruction, so waiting warps do not take issue slots from the working ones.  Bounded: a protocol bug
    // traps instead of hanging the GPU.  The trap is inline and there is no diagnostic printf: a function call inside a wgmma
    // pipeline (between a wgmma and the wait_group that retires it) makes ptxas serialise every wgmma of the kernel (C7510).
#pragma unroll 1
    for (uint32_t it = 0; it < (1u << 18) && !done; ++it)     // (unroll 1: otherwise the loop is unrolled at every call site)
        asm volatile(
            "{\n\t.reg .pred p;\n\t"
            "mbarrier.try_wait.parity.shared::cta.b64 p, [%1], %2, %3;\n\t"
            "selp.u32 %0, 1, 0, p;\n\t}"
            : "=r"(done) : "r"(addr), "r"(parity), "r"(20000u) : "memory");
    if (!done) __trap();
}
__device__ __forceinline__ void fence_barrier_init() {
    asm volatile("fence.mbarrier_init.release.cluster;" ::: "memory");
    asm volatile("fence.proxy.async.shared::cta;" ::: "memory");
}
__device__ __forceinline__ void tma_load_5d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, int c2, int c3, int c4) {
    asm volatile(
        "cp.async.bulk.tensor.5d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6, %7}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3), "r"(c4) : "memory");
}
__device__ __forceinline__ void tma_load_2d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1) {
    asm volatile(
        "cp.async.bulk.tensor.2d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_load_4d(const CUtensorMap* map, uint64_t* bar, void* dst, int c0, int c1, int c2, int c3) {
    asm volatile(
        "cp.async.bulk.tensor.4d.shared::cluster.global.tile.mbarrier::complete_tx::bytes [%0], [%1, {%3, %4, %5, %6}], [%2];"
        ::"r"(smem_u32(dst)), "l"(map), "r"(smem_u32(bar)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_store_4d(const CUtensorMap* map, const void* src, int c0, int c1, int c2, int c3) {
    asm volatile("cp.async.bulk.tensor.4d.global.shared::cta.tile.bulk_group [%0, {%2, %3, %4, %5}], [%1];"
                 ::"l"(map), "r"(smem_u32(src)), "r"(c0), "r"(c1), "r"(c2), "r"(c3) : "memory");
}
__device__ __forceinline__ void tma_store_2d(const CUtensorMap* map, const void* src, int c0, int c1) {
    asm volatile("cp.async.bulk.tensor.2d.global.shared::cta.tile.bulk_group [%0, {%2, %3}], [%1];"
                 ::"l"(map), "r"(smem_u32(src)), "r"(c0), "r"(c1) : "memory");
}
__device__ __forceinline__ void tma_store_commit() { asm volatile("cp.async.bulk.commit_group;" ::: "memory"); }
__device__ __forceinline__ void tma_store_wait_read() { asm volatile("cp.async.bulk.wait_group.read 0;" ::: "memory"); }
__device__ __forceinline__ void fence_async_smem() { asm volatile("fence.proxy.async.shared::cta;" ::: "memory"); }
// named barrier of the 256 consumer threads (the producer warp does not take part)
__device__ __forceinline__ void consumer_bar_sync() { asm volatile("bar.sync 1, 256;" ::: "memory"); }
__device__ __forceinline__ void tma_prefetch_desc(const CUtensorMap* map) {
    asm volatile("prefetch.tensormap [%0];" ::"l"(map) : "memory");
}
__device__ __forceinline__ bool elect_one() {
    uint32_t pred;
    asm volatile(
        "{\n\t.reg .pred p;\n\t"
        "elect.sync _|p, 0xffffffff;\n\t"
        "selp.u32 %0, 1, 0, p;\n\t}"
        : "=r"(pred));
    return pred != 0;
}
__device__ __forceinline__ void wgmma_fence() { asm volatile("wgmma.fence.sync.aligned;" ::: "memory"); }
__device__ __forceinline__ void wgmma_commit() { asm volatile("wgmma.commit_group.sync.aligned;" ::: "memory"); }
template <int N>
__device__ __forceinline__ void wgmma_wait() { asm volatile("wgmma.wait_group.sync.aligned %0;" ::"n"(N) : "memory"); }
// pins register accumulators behind the preceding wgmma_wait: the compiler may not move their reads above it
template <int K>
__device__ __forceinline__ void wgmma_fence_operands(float (&d)[K]) {
#pragma unroll
    for (int j = 0; j < K; ++j) asm volatile("" : "+f"(d[j])::"memory");
}

// K-major shared-memory matrix descriptor of wgmma (PTX ISA "Matrix Descriptor Format", sm_90):
// start>>4 [0,14) | LBO>>4 [16,30) (unused for swizzled K-major) | SBO>>4 [32,46) | base offset [49,52) = 0 | layout [62,64)
// The stage bases are 1024-byte aligned, so the base offset is 0; a K step of 16 halves advances the start by 32 bytes inside
// the swizzle atom, as the hardware applies the XOR pattern to the final address.
template <int SWIZZLE_BYTES>
__device__ __forceinline__ uint64_t make_kmajor_desc(uint32_t saddr) {
    constexpr uint64_t layout = SWIZZLE_BYTES == 128 ? 1 : (SWIZZLE_BYTES == 64 ? 2 : 3);
    constexpr uint64_t sbo = (8 * SWIZZLE_BYTES) >> 4;  // 8 rows of one swizzle span
    return (uint64_t)((saddr & 0x3FFFF) >> 4) | (1ull << 16) | (sbo << 32) | (layout << 62);
}

// D(64 x N, fp32 registers) (+)= A(64 x 16, smem) * B(N x 16, smem)^T; acc == 0 overwrites D.  Fragment of thread t of the
// warpgroup: d[4j + 2i + c] = D[16 (t/32) + (t%32)/4 + 8i][8j + 2 (t%4) + c].
template <int N>
__device__ void wgmma_f16(float (&d)[N / 2], uint64_t a, uint64_t b, uint32_t acc);
template <> __device__ __forceinline__ void wgmma_f16<16>(float (&d)[8], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %10, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n16k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7}, %8, %9, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7])
                 : "l"(a), "l"(b), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma_f16<32>(float (&d)[16], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %18, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n32k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15}, %16, %17, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15])
                 : "l"(a), "l"(b), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma_f16<48>(float (&d)[24], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %26, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n48k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23}, %24, %25, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23])
                 : "l"(a), "l"(b), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma_f16<64>(float (&d)[32], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %34, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n64k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31}, %32, %33, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31])
                 : "l"(a), "l"(b), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma_f16<96>(float (&d)[48], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %50, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, %48, %49, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
                 : "l"(a), "l"(b), "r"(acc));
}
template <> __device__ __forceinline__ void wgmma_f16<128>(float (&d)[64], uint64_t a, uint64_t b, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %66, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n128k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47, %48, %49, %50, %51, %52, %53, %54, %55, %56, %57, %58, %59, %60, %61, %62, %63}, %64, %65, p, 1, 1, 0, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47]), "+f"(d[48]), "+f"(d[49]), "+f"(d[50]), "+f"(d[51]), "+f"(d[52]), "+f"(d[53]), "+f"(d[54]), "+f"(d[55]), "+f"(d[56]), "+f"(d[57]), "+f"(d[58]), "+f"(d[59]), "+f"(d[60]), "+f"(d[61]), "+f"(d[62]), "+f"(d[63])
                 : "l"(a), "l"(b), "r"(acc));
}

// the same with A (64 x 16 fp16) from registers: a[0..3] = the m16k16 fragment of warp w of the warpgroup (rows 16w..16w+15),
// laid out like an accumulator pair of n8 blocks (the FlashAttention-3 register reuse of a GEMM result as the next A operand)
__device__ __forceinline__ void wgmma_f16_rs96(float (&d)[48], const uint32_t (&a)[4], uint64_t b, uint32_t acc) {
    asm volatile("{\n\t.reg .pred p;\n\tsetp.ne.b32 p, %53, 0;\n\t"
                 "wgmma.mma_async.sync.aligned.m64n96k16.f32.f16.f16 {%0, %1, %2, %3, %4, %5, %6, %7, %8, %9, %10, %11, %12, %13, %14, %15, %16, %17, %18, %19, %20, %21, %22, %23, %24, %25, %26, %27, %28, %29, %30, %31, %32, %33, %34, %35, %36, %37, %38, %39, %40, %41, %42, %43, %44, %45, %46, %47}, {%48, %49, %50, %51}, %52, p, 1, 1, 0;\n\t}"
                 : "+f"(d[0]), "+f"(d[1]), "+f"(d[2]), "+f"(d[3]), "+f"(d[4]), "+f"(d[5]), "+f"(d[6]), "+f"(d[7]), "+f"(d[8]), "+f"(d[9]), "+f"(d[10]), "+f"(d[11]), "+f"(d[12]), "+f"(d[13]), "+f"(d[14]), "+f"(d[15]), "+f"(d[16]), "+f"(d[17]), "+f"(d[18]), "+f"(d[19]), "+f"(d[20]), "+f"(d[21]), "+f"(d[22]), "+f"(d[23]), "+f"(d[24]), "+f"(d[25]), "+f"(d[26]), "+f"(d[27]), "+f"(d[28]), "+f"(d[29]), "+f"(d[30]), "+f"(d[31]), "+f"(d[32]), "+f"(d[33]), "+f"(d[34]), "+f"(d[35]), "+f"(d[36]), "+f"(d[37]), "+f"(d[38]), "+f"(d[39]), "+f"(d[40]), "+f"(d[41]), "+f"(d[42]), "+f"(d[43]), "+f"(d[44]), "+f"(d[45]), "+f"(d[46]), "+f"(d[47])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "l"(b), "r"(acc));
}

// Exact-erf GELU with ONE special-function op.  erfc(|x|/sqrt2) = 2^-q(|x|) with q a degree-5 polynomial
// (least-squares/minimax fit on [0, 6], max |gelu error| 5.3e-7 - below fp32 rounding of the surrounding math,
// and far below the fp16 rounding of the stored result).  gelu(x) = x * Phi(x), Phi = 1 - E/2 (x>0) or E/2 (x<0).
// nn.GELU (erf form) in torchvision's MLP, swin_transformer.py:444.  erff() costs ~40 instructions and two MUFU ops,
// which made the fc1 epilogue ALU/MUFU-bound; this is ~12 instructions and one MUFU.EX2.
__device__ __forceinline__ float gelu_erf(float x) {
    const float a = fabsf(x);
    float q = fmaf(a, 4.88118734e-04f, -7.19881030e-03f);
    q = fmaf(q, a, 5.21468017e-02f);
    q = fmaf(q, a, 4.59595724e-01f);
    q = fmaf(q, a, 1.15100057e+00f);
    const float e = ex2(fmaf(-q, a, -1.0f));   // Phi(-|x|) = erfc(|x|/sqrt2)/2: one MUFU.EX2
    // x*Phi(x) = max(x, 0) - |x|*Phi(-|x|) on both sides of zero: no select, 9 instructions per value
    return fmaxf(x, 0.f) - a * e;
}

// activation over a few values; `act` is warp-uniform, so the switch is hoisted out of the element loop
template <int K>
__device__ __forceinline__ void apply_act(float (&v)[K], int act) {
    switch (act) {
        case ACT_LRELU01:
#pragma unroll
            for (int j = 0; j < K; ++j) v[j] = v[j] > 0.f ? v[j] : 0.1f * v[j];
            break;
        case ACT_GELU:
#pragma unroll
            for (int j = 0; j < K; ++j) v[j] = gelu_erf(v[j]);
            break;
        case ACT_RELU:
#pragma unroll
            for (int j = 0; j < K; ++j) v[j] = fmaxf(v[j], 0.f);
            break;
        default: break;
    }
}

constexpr int GEMM_CONSUMER_THREADS = 256;                   // two warpgroups, 64 accumulator rows each
constexpr int GEMM_THREADS = GEMM_CONSUMER_THREADS + 32;     // + the TMA producer warp

template <int BLOCK_N, int BK>
struct GemmCfg {
    static_assert(BLOCK_N % 16 == 0 && BLOCK_N <= 128, "BLOCK_N: 16..128 (the fp32 accumulators live in registers)");
    static constexpr int SWIZZLE = BK * 2;  // bytes per K-row of a stage: 128 (BK=64) or 64 (BK=32)
    static constexpr int A_BYTES = 128 * BK * 2;
    static constexpr int B_BYTES = BLOCK_N * BK * 2;
    static constexpr int STAGE_BYTES = A_BYTES + ((B_BYTES + 1023) / 1024) * 1024;
    // ~96 KB of stages: two CTAs per SM (227 KB of shared memory each)
    static constexpr int STAGES = (98304 / STAGE_BYTES) < 2 ? 2 : ((98304 / STAGE_BYTES) > 6 ? 6 : (98304 / STAGE_BYTES));
    // epilogue staging: BLOCK_N/CW chunks of [128 rows][CW cols] fp16, swizzle span = CW*2 bytes
    static constexpr int CW = (BLOCK_N % 64 == 0) ? 64 : ((BLOCK_N % 32 == 0) ? 32 : 16);
    static constexpr int NCH = BLOCK_N / CW;
    static constexpr int CH_BYTES = 128 * CW * 2;
    static_assert(NCH * CH_BYTES <= STAGES * STAGE_BYTES, "epilogue staging must fit in the (drained) pipeline stages");
    static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + 1024 /*align slack*/ + 256 /*barriers*/;
};

// byte offset of 16-byte chunk j of row r inside a [128][CW] staging tile with the TMA swizzle of span CW*2
template <int CW>
__device__ __forceinline__ uint32_t stage_off(int r, int j) {
    if (CW == 64) return (uint32_t)(r * 128 + ((j ^ (r & 7)) << 4));
    if (CW == 32) return (uint32_t)(r * 64 + ((j ^ ((r >> 1) & 3)) << 4));
    return (uint32_t)(r * 32 + ((j ^ ((r >> 2) & 1)) << 4));
}

// byte offset of element (r, col) of a [ROWS][K] fp16 operand stored as K/32 TMA boxes of [ROWS][32] with the 64B swizzle
template <int ROWS>
__device__ __forceinline__ uint32_t sw64_off(int r, int col) {
    return (uint32_t)((col >> 5) * (ROWS * 64)) + stage_off<32>(r, (col & 31) >> 3) + (uint32_t)((col & 7) * 2);
}

// A2: OUT_PIXSHUF2 with a second A operand.  Its K-chunks follow those of A, and each output pixel (2y+dy, 2x+dx) reads the
// second operand at that same position; (dy, dx) is fixed by the CTA's N-block, so BLOCK_N must divide cout.
template <int BLOCK_N, int BK, bool A2 = false>
__global__ void __launch_bounds__(GEMM_THREADS, 2) gemm_conv_kernel(const __grid_constant__ GemmMaps maps,
                                                                    const __grid_constant__ GemmParams p) {
    using Cfg = GemmCfg<BLOCK_N, BK>;
    constexpr int STAGES = Cfg::STAGES;
    constexpr int CW = Cfg::CW;
    extern __shared__ uint8_t smem_dyn[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + STAGES * Cfg::STAGE_BYTES);
    uint64_t* empty_bar = full_bar + STAGES;
    uint64_t* res_bar = empty_bar + STAGES;

    const int warp = threadIdx.x >> 5;
    // n tile is the fast grid index so CTAs sharing an A tile run together (A re-reads hit L2)
    const int n_tile = blockIdx.x % p.n_tiles;
    const int tile = blockIdx.x / p.n_tiles;
    const int tx_i = tile % p.tiles_x;
    const int ty_i = (tile / p.tiles_x) % p.tiles_y;
    const int b = tile / (p.tiles_x * p.tiles_y);
    const int x0 = tx_i * p.TW, y0 = ty_i * p.TH;
    const int n0 = n_tile * BLOCK_N;
    const int k_iters = p.taps * p.cpt + (A2 ? p.k2 : 0);

    if (threadIdx.x == GEMM_CONSUMER_THREADS) {
        tma_prefetch_desc(&maps.a);
        tma_prefetch_desc(&maps.b);
        tma_prefetch_desc(&maps.o[0]);
        for (int s = 0; s < STAGES; ++s) {
            mbar_init(&full_bar[s], 1);
            mbar_init(&empty_bar[s], 2);   // one arrival per consumer warpgroup
        }
        mbar_init(res_bar, 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == GEMM_CONSUMER_THREADS / 32) {
        // ===================== TMA producer =====================
        if (elect_one()) {
            // programmatic dependent launch: everything above overlapped the previous kernel of the stream; its outputs
            // (this GEMM's activations and residual) are complete and visible once this returns
            asm volatile("griddepcontrol.wait;" ::: "memory");
            for (int it = 0; it < k_iters; ++it) {
                const int s = it % STAGES;
                const uint32_t ph = (it / STAGES) & 1;
                mbar_wait(&empty_bar[s], ph ^ 1);
                const int tap = it / p.cpt, ch = it - tap * p.cpt;
                uint8_t* sa = smem + s * Cfg::STAGE_BYTES;
                uint8_t* sb = sa + Cfg::A_BYTES;
                mbar_expect_tx(&full_bar[s], Cfg::A_BYTES + Cfg::B_BYTES);
                if (A2 && tap >= p.taps) {
                    // rows y >= Ho of a bottom edge tile read the next image; the output store clips them
                    const int q = n0 / p.cout;
                    tma_load_5d(&maps.a2, &full_bar[s], sa, (it - p.taps * p.cpt) * BK, q & 1, x0, q >> 1, b * p.Ho + y0);
                } else {
                    tma_load_5d(&maps.a, &full_bar[s], sa, ch * BK, x0 + p.tap_dx[tap], p.tap_dyi[tap], y0 + p.tap_dy[tap], b);
                }
                tma_load_2d(&maps.b, &full_bar[s], sb, it * BK, n0);
            }
        }
        return;
    }

    // ===================== consumers (warps 0..7) =====================
    const int wg = threadIdx.x >> 7;        // accumulator rows [64 wg, 64 wg + 64)
    const int t = threadIdx.x & 127;
    float acc[BLOCK_N / 2];
#pragma unroll
    for (int j = 0; j < BLOCK_N / 2; ++j) acc[j] = 0.f;
    for (int it = 0; it < k_iters; ++it) {
        const int s = it % STAGES;
        mbar_wait(&full_bar[s], (it / STAGES) & 1);
        const uint32_t sa = smem_u32(smem + s * Cfg::STAGE_BYTES) + wg * 64 * Cfg::SWIZZLE;
        const uint32_t sb = smem_u32(smem + s * Cfg::STAGE_BYTES) + Cfg::A_BYTES;
        wgmma_fence();
#pragma unroll
        for (int k = 0; k < BK / 16; ++k)
            wgmma_f16<BLOCK_N>(acc, make_kmajor_desc<Cfg::SWIZZLE>(sa + k * 32), make_kmajor_desc<Cfg::SWIZZLE>(sb + k * 32), 1u);
        wgmma_commit();
        // keep one group in flight: the stage read by the previous group is released once that group retired
        wgmma_wait<1>();
        if (it > 0 && t == 0) mbar_arrive(&empty_bar[(it - 1) % STAGES]);
    }
    wgmma_wait<0>();
    wgmma_fence_operands(acc);
    if (threadIdx.x == 0) NB_PDL_TRIGGER();   // the next GEMM of the stream may start its prologue while this grid drains
    // both warpgroups have retired all their MMAs => every pipeline stage is drained and reusable as epilogue staging
    consumer_bar_sync();
    uint8_t* stg = smem;
    const bool leader = threadIdx.x == 0;
    if (p.has_res) {
        if (leader) {
            mbar_expect_tx(res_bar, Cfg::NCH * Cfg::CH_BYTES);
#pragma unroll 1
            for (int c = 0; c < Cfg::NCH; ++c) {
                const int n = n0 + c * CW;
                const int g = p.out_mode != OUT_NHWC ? n / p.cout : 0;
                const int co = p.out_mode != OUT_NHWC ? n - g * p.cout : n;
                tma_load_4d(&maps.r[g], res_bar, stg + c * Cfg::CH_BYTES, co, x0 + p.res_cx, y0 + p.res_cy, b);
            }
        }
        mbar_wait(res_bar, 0);
    }
    const int act = p.act;
    const bool has_res = p.has_res != 0, res_first = p.res_before_act != 0;
    const int row0 = wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2);   // accumulator row == pixel within the tile == staging row
    const int cq = 2 * (t & 3);
#pragma unroll
    for (int j = 0; j < BLOCK_N / 8; ++j) {
        const int col = 8 * j + cq;
        const int c = (8 * j) / CW;
        float2 bq = make_float2(0.f, 0.f);
        if (p.bias) bq = __ldg(reinterpret_cast<const float2*>(p.bias + n0 + col));
        float v[4] = {acc[4 * j] + bq.x, acc[4 * j + 1] + bq.y, acc[4 * j + 2] + bq.x, acc[4 * j + 3] + bq.y};
        __half2* s0 = reinterpret_cast<__half2*>(stg + c * Cfg::CH_BYTES + stage_off<CW>(row0, (8 * j % CW) / 8) + 2 * cq);
        __half2* s1 = reinterpret_cast<__half2*>(stg + c * Cfg::CH_BYTES + stage_off<CW>(row0 + 8, (8 * j % CW) / 8) + 2 * cq);
        if (has_res) {
            const float2 r0 = __half22float2(*s0), r1 = __half22float2(*s1);
            const float rv[4] = {r0.x, r0.y, r1.x, r1.y};
            if (res_first) {
#pragma unroll
                for (int q = 0; q < 4; ++q) v[q] += rv[q];
                apply_act(v, act);
            } else {
                apply_act(v, act);
#pragma unroll
                for (int q = 0; q < 4; ++q) v[q] += rv[q];
            }
        } else {
            apply_act(v, act);
        }
        *s0 = __floats2half2_rn(v[0], v[1]);
        *s1 = __floats2half2_rn(v[2], v[3]);
    }
    fence_async_smem();  // generic-proxy smem writes -> visible to the TMA (async proxy)
    consumer_bar_sync();
    if (leader) {
#pragma unroll 1
        for (int c = 0; c < Cfg::NCH; ++c) {
            const int n = n0 + c * CW;
            const int g = p.out_mode != OUT_NHWC ? n / p.cout : 0;
            const int co = p.out_mode != OUT_NHWC ? n - g * p.cout : n;
            // out-of-range rows/cols of edge tiles are clipped by TMA
            tma_store_4d(&maps.o[g], stg + c * Cfg::CH_BYTES, co, x0, y0, b);
        }
        tma_store_commit();
        tma_store_wait_read();  // smem must stay valid until the bulk stores have read it
    }
}

}  // namespace nb200
