// Fused tail of one SwinTransformerBlock (torchvision swin_transformer.py:228 proj, :453-455; MLP = Linear-GELU-Linear,
// ratio 2, Identity norms: waifu2x/models/swin_unet.py:16-17,31):
//   x1 = x + att . Wp^T + bp   (att == nullptr: x1 = x);   x <- x1 + gelu(x1 . W1^T + b1) . W2^T + b2
// x1 and the 2C hidden tensor never reach HBM.  One CTA = 128 tokens = two wgmma warpgroups of 64 rows.
//   warp 8    : TMA: the x (and att) tile once, then the weight blocks [rows][32] (64B swizzle) through a ring, in the
//               order the consumers use them: Wp (C/32 blocks), then per 64-wide hidden chunk W1 (C/32) and W2 (2)
//   warps 0-7 : proj into registers, x1 written in place over the x tile (A operand of fc1, residual of fc2); per hidden
//               chunk fc1 into registers, bias + GELU, packed to fp16 A fragments in registers and fed straight to the fc2
//               wgmma (A from registers), whose C-wide accumulator lives in registers for the whole tile; the output is
//               written in place over the x tile and stored with TMA.
// The two entry points of include/nunif_b200.h that expose the fused block kernels (head: swin_attention_mma.cu).
#include "gemm_wgmma.cuh"
#include "swin_kernels.h"
#include "tmap.h"

namespace nb200 {

constexpr int FM_ROWS = 128, FM_STAGES = 6, FM_THREADS = GEMM_CONSUMER_THREADS + 32;

template <int C>
struct FmCfg {
    static constexpr int TILE = FM_ROWS * C * 2;   // one [128][C] activation tile (C/32 boxes of [128][32])
    static constexpr int SLOT = C * 64;            // largest weight block: [C rows][32]
    static constexpr int SMEM = 2 * TILE + FM_STAGES * SLOT + (2 * FM_STAGES + 1) * 8 + 1024;
};

struct FmMaps {
    CUtensorMap x, att, wp, w1, w2;
};

template <int K>
__device__ __forceinline__ float (&half96(float (&acc)[K], int h))[48] { return *reinterpret_cast<float(*)[48]>(&acc[48 * h]); }

template <int C>
__global__ void __launch_bounds__(FM_THREADS, 1) swin_mlp_fused_kernel(const __grid_constant__ FmMaps maps, const float* __restrict__ bp,
                                                                       const float* __restrict__ b1, const float* __restrict__ b2,
                                                                       int has_proj) {
    using Cfg = FmCfg<C>;
    constexpr int KB = C / 32, NH = 2 * C / 64, NHALF = C / 96;
    extern __shared__ uint8_t smem_dyn[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    uint8_t* sx = smem;
    uint8_t* satt = smem + Cfg::TILE;
    uint8_t* ring = smem + 2 * Cfg::TILE;
    uint64_t* full = reinterpret_cast<uint64_t*>(ring + FM_STAGES * Cfg::SLOT);
    uint64_t* empty = full + FM_STAGES;
    uint64_t* xbar = empty + FM_STAGES;
    const int tid = threadIdx.x, warp = tid >> 5;
    const int row_base = blockIdx.x * FM_ROWS;
    if (tid == GEMM_CONSUMER_THREADS) {
        tma_prefetch_desc(&maps.x);
        tma_prefetch_desc(&maps.w1);
        tma_prefetch_desc(&maps.w2);
        for (int s = 0; s < FM_STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 2);   // one arrival per consumer warpgroup
        }
        mbar_init(xbar, 1);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp == GEMM_CONSUMER_THREADS / 32) {
        // ===================== TMA producer =====================
        if (elect_one()) {
            mbar_expect_tx(xbar, (has_proj ? 2 : 1) * Cfg::TILE);
            for (int kb = 0; kb < KB; ++kb) {
                tma_load_2d(&maps.x, xbar, sx + kb * (FM_ROWS * 64), kb * 32, row_base);
                if (has_proj) tma_load_2d(&maps.att, xbar, satt + kb * (FM_ROWS * 64), kb * 32, row_base);
            }
            int it = 0;
            auto push = [&](const CUtensorMap* m, int k, int n, int rows) {
                const int s = it % FM_STAGES;
                mbar_wait(&empty[s], ((it / FM_STAGES) & 1) ^ 1);
                mbar_expect_tx(&full[s], rows * 64);
                tma_load_2d(m, &full[s], ring + s * Cfg::SLOT, k, n);
                ++it;
            };
            if (has_proj)
                for (int kb = 0; kb < KB; ++kb) push(&maps.wp, kb * 32, 0, C);
            for (int hc = 0; hc < NH; ++hc) {
                for (int kb = 0; kb < KB; ++kb) push(&maps.w1, kb * 32, hc * 64, 64);
                for (int kb = 0; kb < 2; ++kb) push(&maps.w2, hc * 64 + kb * 32, 0, C);
            }
        }
        return;
    }

    // ===================== consumers (warps 0..7) =====================
    const int wg = tid >> 7, t = tid & 127;
    const int row0 = wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2);   // accumulator rows row0 and row0 + 8
    const int cq = 2 * (t & 3);
    const uint32_t x_base = smem_u32(sx) + wg * 64 * 64, att_base = smem_u32(satt) + wg * 64 * 64;
    int it = 0;
    auto take = [&]() -> uint32_t {
        const int s = it % FM_STAGES;
        mbar_wait(&full[s], (it / FM_STAGES) & 1);
        return smem_u32(ring + s * Cfg::SLOT);
    };
    auto release = [&]() {
        if (t == 0) mbar_arrive(&empty[it % FM_STAGES]);
        ++it;
    };
    mbar_wait(xbar, 0);

    if (has_proj) {
        // x1 = x + att Wp^T + bp  (x :453)
        float acc[C / 2];
#pragma unroll
        for (int j = 0; j < C / 2; ++j) acc[j] = 0.f;
#pragma unroll 1
        for (int kb = 0; kb < KB; ++kb) {
            const uint32_t bb = take(), a = att_base + kb * (FM_ROWS * 64);
            wgmma_fence();
#pragma unroll
            for (int s = 0; s < 2; ++s)
#pragma unroll
                for (int h = 0; h < NHALF; ++h)
                    wgmma_f16<96>(half96(acc, h), make_kmajor_desc<64>(a + 32 * s), make_kmajor_desc<64>(bb + h * 96 * 64 + 32 * s), 1u);
            wgmma_commit();
            wgmma_wait<0>();
            release();
        }
        wgmma_fence_operands(acc);
#pragma unroll
        for (int j = 0; j < C / 8; ++j) {
            const int col = 8 * j + cq;
            const float2 bq = __ldg(reinterpret_cast<const float2*>(bp + col));
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                __half2* p = reinterpret_cast<__half2*>(sx + sw64_off<FM_ROWS>(row0 + 8 * i, col));
                const float2 xv = __half22float2(*p);
                *p = __floats2half2_rn(xv.x + (acc[4 * j + 2 * i] + bq.x), xv.y + (acc[4 * j + 2 * i + 1] + bq.y));
            }
        }
        fence_async_smem();   // x1 (generic-proxy writes) -> A operand of this warpgroup's fc1 wgmma
        asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
    }

    float oacc[C / 2];
#pragma unroll
    for (int j = 0; j < C / 2; ++j) oacc[j] = 0.f;
#pragma unroll 1
    for (int hc = 0; hc < NH; ++hc) {
        // hidden chunk: gelu(x1 W1[64 hc : 64 hc + 64]^T + b1) (:444), rounded to fp16 as the reference stores it
        float hacc[32];
#pragma unroll
        for (int j = 0; j < 32; ++j) hacc[j] = 0.f;
#pragma unroll 1
        for (int kb = 0; kb < KB; ++kb) {
            const uint32_t bb = take(), a = x_base + kb * (FM_ROWS * 64);
            wgmma_fence();
            wgmma_f16<64>(hacc, make_kmajor_desc<64>(a), make_kmajor_desc<64>(bb), 1u);
            wgmma_f16<64>(hacc, make_kmajor_desc<64>(a + 32), make_kmajor_desc<64>(bb + 32), 1u);
            wgmma_commit();
            wgmma_wait<0>();
            release();
        }
        wgmma_fence_operands(hacc);
        uint32_t af[4][4];   // k16 block kk of the chunk: {row g | g+8} x {cols 2t, 2t+8} as in the m16n8k16 A fragment
#pragma unroll
        for (int kk = 0; kk < 4; ++kk)
#pragma unroll
            for (int q = 0; q < 4; ++q) {
                const int j = 2 * kk + (q >> 1), i = q & 1;
                const float2 bq = __ldg(reinterpret_cast<const float2*>(b1 + 64 * hc + 8 * j + cq));
                const __half2 h = __floats2half2_rn(gelu_erf(hacc[4 * j + 2 * i] + bq.x), gelu_erf(hacc[4 * j + 2 * i + 1] + bq.y));
                af[kk][q] = *reinterpret_cast<const uint32_t*>(&h);
            }
        // out += hidden_chunk W2[:, 64 hc : 64 hc + 64]^T
#pragma unroll 1
        for (int kb = 0; kb < 2; ++kb) {
            const uint32_t bb = take();
            wgmma_fence();
#pragma unroll
            for (int s = 0; s < 2; ++s)
#pragma unroll
                for (int h = 0; h < NHALF; ++h)
                    wgmma_f16_rs96(half96(oacc, h), af[2 * kb + s], make_kmajor_desc<64>(bb + h * 96 * 64 + 32 * s), 1u);
            wgmma_commit();
            wgmma_wait<0>();
            release();
        }
    }
    wgmma_fence_operands(oacc);
    // x <- x1 + mlp(x1) (:454), in place over the x1 tile, then one TMA store per 32-column box
#pragma unroll
    for (int j = 0; j < C / 8; ++j) {
        const int col = 8 * j + cq;
        const float2 bq = __ldg(reinterpret_cast<const float2*>(b2 + col));
#pragma unroll
        for (int i = 0; i < 2; ++i) {
            __half2* p = reinterpret_cast<__half2*>(sx + sw64_off<FM_ROWS>(row0 + 8 * i, col));
            const float2 xv = __half22float2(*p);
            *p = __floats2half2_rn(xv.x + (oacc[4 * j + 2 * i] + bq.x), xv.y + (oacc[4 * j + 2 * i + 1] + bq.y));
        }
    }
    fence_async_smem();
    consumer_bar_sync();
    if (tid == 0) {
        for (int kb = 0; kb < KB; ++kb) tma_store_2d(&maps.x, sx + kb * (FM_ROWS * 64), kb * 32, row_base);   // rows >= T are clipped
        tma_store_commit();
        tma_store_wait_read();
    }
}

static int map2d(CUtensorMap* m, const void* base, int cols, long long rows, int box_rows) {
    const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
    const cuuint32_t box[2] = {32, (cuuint32_t)box_rows};
    return encode(m, base, 2, dims, strides, box, 64);
}

int swin_mlp_fused(cudaStream_t st, __half* x, const __half* att, long long T, int C, const __half* wp, const float* bp,
                   const __half* w1, const float* b1, const __half* w2, const float* b2) {
    NB_CHECK(x && w1 && b1 && w2 && b2 && (!att || (wp && bp)), "null pointer");
    NB_CHECK(C == 96 || C == 192, "C must be 96 or 192");
    NB_CHECK(T > 0 && T < (1LL << 31), "token count out of range");
    FmMaps maps;
    memset(&maps, 0, sizeof(maps));
    if (map2d(&maps.x, x, C, T, FM_ROWS)) return 1;
    if (att && (map2d(&maps.att, att, C, T, FM_ROWS) || map2d(&maps.wp, wp, C, C, C))) return 1;
    if (map2d(&maps.w1, w1, C, 2 * C, 64) || map2d(&maps.w2, w2, 2 * C, C, C)) return 1;
    const double Td = (double)T;
    ProfScope ps(st, PC_FUSED_MLP, Td * C * C * 2 * ((att ? 1 : 0) + 4), Td * C * 2 * (att ? 2 : 1), Td * C * 2);
    const unsigned grid = (unsigned)((T + FM_ROWS - 1) / FM_ROWS);
    if (C == 96) {
        if (ensure_dyn_smem((const void*)swin_mlp_fused_kernel<96>, FmCfg<96>::SMEM)) return 1;
        swin_mlp_fused_kernel<96><<<grid, FM_THREADS, FmCfg<96>::SMEM, st>>>(maps, bp, b1, b2, att ? 1 : 0);
    } else {
        if (ensure_dyn_smem((const void*)swin_mlp_fused_kernel<192>, FmCfg<192>::SMEM)) return 1;
        swin_mlp_fused_kernel<192><<<grid, FM_THREADS, FmCfg<192>::SMEM, st>>>(maps, bp, b1, b2, att ? 1 : 0);
    }
    NB_LAUNCHED();
    return 0;
}

}  // namespace nb200

using namespace nb200;

extern "C" int nb200_swin_mlp_fused_f16(void* x, const void* att, long long T, int C, const void* wp, const float* bp,
                                        const void* w1, const float* b1, const void* w2, const float* b2, void* stream) {
    return swin_mlp_fused((cudaStream_t)stream, (__half*)x, (const __half*)att, T, C, (const __half*)wp, bp, (const __half*)w1, b1,
                          (const __half*)w2, b2);
}

extern "C" int nb200_swin_attn_fused_f16(const void* x, const void* wqkv, const float* bqkv, const float* bias_table, void* att,
                                         int B, int H, int W, int C, int shift, void* stream) {
    NB_CHECK(bias_table, "null pointer");
    cudaStream_t st = (cudaStream_t)stream;
    float* frag = nullptr;   // relative-position bias in the attention core's fragment order (the model packs it at load)
    NB_CUDA(cudaMallocAsync((void**)&frag, BIAS_FRAG_FLOATS * sizeof(float), st));
    int rc = build_bias_frag(st, bias_table, frag);
    if (!rc) rc = swin_attn_fused(st, (const __half*)x, (const __half*)wqkv, bqkv, frag, (__half*)att, B, H, W, C, shift);
    cudaFreeAsync(frag, st);
    return rc;
}
