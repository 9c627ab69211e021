// Fused tail of one SwinTransformerBlock (torchvision swin_transformer.py:228 proj, :453-455; MLP = Linear-GELU-Linear,
// ratio 2, Identity norms: waifu2x/models/swin_unet.py:16-17,31):
//   x1 = x + att . Wp^T + bp   (att == nullptr: x1 = x);   x <- x1 + gelu(x1 . W1^T + b1) . W2^T + b2
// x1 and the 2C hidden tensor never reach HBM.  A tile is 128 tokens = two wgmma warpgroups of 64 rows.  The grid is
// persistent: min(tiles, SMs) CTAs, CTA i takes tiles i, i + grid, ... (j below counts a CTA's own tiles).  Roles:
//   warp 8    : TMA: the weights through a ring of [128 C]-byte stages, in the order the consumers use them: Wp two K-blocks
//               per stage ([C][64]), then per 64-wide hidden chunk h one stage of W1 rows ([64][C]) and one of W2 columns
//               ([C][64]), with W1(h + 1) ahead of W2(h).  Every tile takes the same sequence; the ring runs straight on
//               from one tile to the next.  The weights do not depend on the previous kernel, so this warp never waits
//               for it.
//   warp 9    : TMA: the activations.  After griddepcontrol.wait it loads att (one barrier per 32-column K-block) and x
//               of the CTA's tiles ahead of the consumers, and issues each tile's output store once the consumers have
//               written it.  No thread waits on both the ring and an activation buffer.
//   warps 0-7 : proj into registers as the att K-blocks land, x1 written over the att tile (A operand of fc1, residual of
//               fc2); per hidden chunk fc1 into registers, bias + GELU, packed to fp16 A fragments in registers and fed
//               straight to the fc2 wgmma (A from registers), whose C-wide accumulator lives in registers for the whole tile;
//               the output is written in place over the x1 tile.
// Activation buffers: NBUF tiles of [C/32][128][32] (64B swizzle).  Tile j's att and x1 live in buffer j % NBUF, its x in
// buffer (j + PROJ) % NBUF.  With PROJ the x tile is dead once both warpgroups have finished the proj epilogue, and att of
// tile j + 1 loads into it while tile j runs fc1/fc2; x of tile j + NBUF - 1 (PROJ) or j + NBUF loads into x1(j)'s buffer
// once its store has read it.  NBUF = 2 at C = 192 (the shared memory of the non-persistent tail), 3 at C = 96, where x
// then arrives a whole tile ahead.
// With CS > 0 (the last block of the network) the output tile is not stored: it is the A operand of one more wgmma,
// y = x . Wy^T + by (to_image's Linear, [T][CS]), whose weights come through the ring as one more stage after the last W2
// stage; y is staged in the x1 buffer and stored instead.  This block's x is dead afterwards, so it never reaches HBM.
// Each ring stage is one wgmma commit group and is released when that group has retired, so the tensor pipe is never drained
// inside a GEMM.  fc1 of chunk h + 1 goes into a second hidden accumulator before the GELU of chunk h, so that it runs with
// tensor work in flight.  That takes ~210 registers per consumer thread (fc2's accumulator alone is C/2): with 288 threads
// three warps share an SM sub-partition's 64 KB register file, which caps a thread at 168, so the producers are a whole
// warpgroup (warps 8-11, two of them working) that gives its registers to the consumers with setmaxnreg.
//
// Barriers (j: the CTA's tile counter; q: its weight-stage counter; a wait for use u of a barrier waits for parity u mod 2):
//   barrier       count            arrives                                                     waits
//   full[s]       1 + tx bytes     warp 8 expect_tx, TMA completes                              consumers, stage q
//   empty[s]      2                thread 0 of each warpgroup once the stage's group retired    warp 8, before stage q + 5
//   abar[b][kb]   1 + tx bytes     warp 9 expect_tx, TMA completes (att K-block kb of tile j)   consumers, tile j (b = j mod NBUF)
//   xbar[b]       1 + tx bytes     warp 9 expect_tx, TMA completes (x of tile j)                consumers, tile j (b = j mod NBUF)
//   xfree         2                thread 0 of each warpgroup after its proj epilogue            warp 9, before att of tile j + 1
//   outw[b]       2                thread 0 of each warpgroup after its output (or y) epilogue  warp 9, before the store of tile j
// Every waiter waits on every phase of its barriers, in order, so a parity wait is exact when the arrivals cannot run a
// phase ahead of it:
//   * abar[b] is armed for tile j + NBUF after warp 9's wait on xfree(j + NBUF - 1), which the consumers pass only after
//     their wait on abar[b] for tile j; xbar[b] for tile j + NBUF after outw of tile j + NBUF - 1 (PROJ) or j, likewise.
//   * xfree of tile j + 1 needs att of tile j + 1, which warp 9 loads after its wait on xfree(j).
//   * outw[b] of tile j + NBUF needs att (PROJ) or x of tile j + NBUF, which warp 9 loads after its wait on outw[b](j).
//   * A warpgroup takes stage q only after the other has released stage q - 5, and a tile has more than 5 stages, so one
//     warpgroup cannot arrive twice on a count-2 barrier before the other has arrived once.
// No wait closes a cycle: warp 9's waits need only loads it issued before them, and warp 8 waits only on the consumers' use
// of the ring.
#include "gemm_wgmma.cuh"
#include "swin_kernels.h"
#include "tmap.h"
#include <algorithm>

namespace nb200 {

extern int g_tune[16];  // gemm.cu (nb200_tune_set)

constexpr int FM_ROWS = 128, FM_STAGES = 5, FM_THREADS = GEMM_CONSUMER_THREADS + 128;
constexpr int FM_PRODUCER_REGS = 40, FM_CONSUMER_REGS = 232;   // 2 x 232 + 40 per sub-partition: 504 x 32 <= 16384

template <int C>
struct FmCfg {
    static constexpr int KB = C / 32;
    static constexpr int NBUF = C == 96 ? 3 : 2;     // activation tiles
    static constexpr int TILE = FM_ROWS * C * 2;   // one [128][C] activation tile (C/32 boxes of [128][32])
    static constexpr int STAGE = 128 * C;          // [64][C] of W1, [C][64] of W2 or of Wp
    static constexpr int SMEM = NBUF * TILE + FM_STAGES * STAGE + (2 * FM_STAGES + NBUF * (KB + 2) + 1) * 8 + 1024;
    static_assert(SMEM <= 232448, "shared memory per CTA exceeds the opt-in limit");
};

struct FmMaps {
    CUtensorMap x, att, wp, w1, w2, y, wy;
};

template <int K>
__device__ __forceinline__ float (&half96(float (&acc)[K], int h))[48] { return *reinterpret_cast<float(*)[48]>(&acc[48 * h]); }

// wgmma.wait_group 0 or 1, with a count that is a constant after unrolling
__device__ __forceinline__ void wgmma_wait_n(int n) {
    if (n == 0) wgmma_wait<0>();
    else wgmma_wait<1>();
}

// PROJ (att != nullptr) and CS (the width of y, 0: store x) are template parameters: wgmmas under a run-time branch make
// ptxas serialise all of them.
template <int C, bool PROJ, int CS>
__global__ void __launch_bounds__(FM_THREADS, 1) swin_mlp_fused_kernel(const __grid_constant__ FmMaps maps, const float* __restrict__ bp,
                                                                     const float* __restrict__ b1, const float* __restrict__ b2,
                                                                     const float* __restrict__ by, int ntiles) {
    using Cfg = FmCfg<C>;
    static_assert(CS % 16 == 0 && 2 * C * CS <= Cfg::STAGE && CS * 256 <= Cfg::TILE, "Wy must fit a ring stage, y a tile");
    constexpr int KB = Cfg::KB, NP = (KB + 1) / 2, NH = 2 * C / 64, NHALF = C / 96, NBUF = Cfg::NBUF;
    constexpr int SPT = (PROJ ? NP : 0) + 2 * NH + (CS ? 1 : 0);   // ring stages per tile
    static_assert(SPT > FM_STAGES, "the barrier protocol needs more stages per tile than the ring holds");
    constexpr int XAHEAD = PROJ ? NBUF - 1 : NBUF;   // x tiles in flight ahead of the consumers
    extern __shared__ uint8_t smem_dyn[];
    // aligned by an offset from smem_dyn, not by integer arithmetic on its address: the compiler then knows every pointer
    // below is a shared-memory one and keeps 32-bit addresses (LDS/STS) instead of 64-bit generic ones
    uint8_t* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
    uint8_t* ring = smem + NBUF * Cfg::TILE;
    uint64_t* full = reinterpret_cast<uint64_t*>(ring + FM_STAGES * Cfg::STAGE);
    uint64_t* empty = full + FM_STAGES;
    uint64_t* abar = empty + FM_STAGES;   // [NBUF][KB]: att K-block kb
    uint64_t* xbar = abar + NBUF * KB;    // [NBUF]
    uint64_t* outw = xbar + NBUF;         // [NBUF]
    uint64_t* xfree = outw + NBUF;
    auto buf = [&](int b) { return smem + b * Cfg::TILE; };
    const int tid = threadIdx.x, warp = tid >> 5;
    const int nt = (ntiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;   // this CTA's tiles
    if (tid == GEMM_CONSUMER_THREADS) {
        tma_prefetch_desc(&maps.x);
        tma_prefetch_desc(&maps.w1);
        tma_prefetch_desc(&maps.w2);
        if (CS) {
            tma_prefetch_desc(&maps.wy);
            tma_prefetch_desc(&maps.y);
        }
        if (PROJ) {
            tma_prefetch_desc(&maps.att);
            tma_prefetch_desc(&maps.wp);
        }
        for (int s = 0; s < FM_STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 2);   // one arrival per consumer warpgroup
        }
        for (int b = 0; b < NBUF; ++b) {
            for (int kb = 0; kb < KB; ++kb) mbar_init(&abar[b * KB + kb], 1);
            mbar_init(&xbar[b], 1);
            mbar_init(&outw[b], 2);
        }
        mbar_init(xfree, 2);
        fence_barrier_init();
    }
    __syncthreads();

    if (warp >= GEMM_CONSUMER_THREADS / 32) {
        asm volatile("setmaxnreg.dec.sync.aligned.u32 %0;" ::"n"(FM_PRODUCER_REGS));
        if (warp == GEMM_CONSUMER_THREADS / 32 && elect_one()) {
            // ===================== weight producer =====================
            int it = 0;
            // one ring stage: nbox boxes of `rows` x 32 columns, box b at column k0 + 32 b, row n0
            auto push = [&](const CUtensorMap* m, int k0, int n0, int rows, int nbox) {
                const int s = it % FM_STAGES;
                mbar_wait(&empty[s], ((it / FM_STAGES) & 1) ^ 1);
                mbar_expect_tx(&full[s], nbox * rows * 64);
                for (int b = 0; b < nbox; ++b) tma_load_2d(m, &full[s], ring + s * Cfg::STAGE + b * rows * 64, k0 + 32 * b, n0);
                ++it;
            };
            for (int j = 0; j < nt; ++j) {
                if (PROJ)
                    for (int p = 0; p < NP; ++p) push(&maps.wp, 64 * p, 0, C, min(2, KB - 2 * p));
                push(&maps.w1, 0, 0, 64, KB);
                for (int hc = 0; hc < NH; ++hc) {
                    if (hc + 1 < NH) push(&maps.w1, 0, (hc + 1) * 64, 64, KB);
                    push(&maps.w2, hc * 64, 0, C, 2);
                }
                if (CS) push(&maps.wy, 0, 0, CS, KB);
            }
        } else if (warp == GEMM_CONSUMER_THREADS / 32 + 1 && elect_one()) {
            // ===================== activation loads and output stores =====================
            auto row = [&](int j) { return ((int)blockIdx.x + j * (int)gridDim.x) * FM_ROWS; };
            auto load_att = [&](int j) {
                const int b = j % NBUF;
                for (int kb = 0; kb < KB; ++kb) {
                    mbar_expect_tx(&abar[b * KB + kb], FM_ROWS * 64);
                    tma_load_2d(&maps.att, &abar[b * KB + kb], buf(b) + kb * (FM_ROWS * 64), kb * 32, row(j));
                }
            };
            auto load_x = [&](int j) {
                uint8_t* dst = buf((j + PROJ) % NBUF);
                mbar_expect_tx(&xbar[j % NBUF], Cfg::TILE);
                for (int kb = 0; kb < KB; ++kb) tma_load_2d(&maps.x, &xbar[j % NBUF], dst + kb * (FM_ROWS * 64), kb * 32, row(j));
            };
            // programmatic dependent launch: everything before this overlapped the previous kernel of the stream (the head,
            // which writes att); once it returns, that kernel's outputs are complete and visible
            asm volatile("griddepcontrol.wait;" ::: "memory");
            if (PROJ) load_att(0);
            for (int j = 0; j < XAHEAD && j < nt; ++j) load_x(j);
            for (int j = 0; j < nt; ++j) {
                if (PROJ) {
                    mbar_wait(xfree, j & 1);   // x of tile j is dead: its buffer takes att of tile j + 1
                    if (j + 1 < nt) load_att(j + 1);
                }
                const int b = j % NBUF;
                mbar_wait(&outw[b], (j / NBUF) & 1);
                if constexpr (CS > 0)
                    for (int c = 0; c < CS / 16; ++c) tma_store_2d(&maps.y, buf(b) + c * (FM_ROWS * 32), 16 * c, row(j));
                else
                    for (int kb = 0; kb < KB; ++kb) tma_store_2d(&maps.x, buf(b) + kb * (FM_ROWS * 64), kb * 32, row(j));   // rows >= T are clipped
                tma_store_commit();
                tma_store_wait_read();   // the buffer stays valid until the store has read it
                if (j + XAHEAD < nt) load_x(j + XAHEAD);
            }
        }
        return;
    }

    // ===================== consumers (warps 0..7) =====================
    asm volatile("setmaxnreg.inc.sync.aligned.u32 %0;" ::"n"(FM_CONSUMER_REGS));
    const int wg = tid >> 7, t = tid & 127;
    const int row0 = wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2);   // accumulator rows row0 and row0 + 8
    const int cq = 2 * (t & 3);
    // the ring position is the only loop-carried register: the tile counter and the loop bound are recomputed from it,
    // blockIdx, gridDim and ntiles (at C = 192 without PROJ one more live register spills at the GELU)
#pragma unroll 1
    for (int it0 = 0; (int)blockIdx.x + it0 / SPT * (int)gridDim.x < ntiles; it0 += SPT) {
        const int j = it0 / SPT;
        int it = it0;   // ring stages taken
        const int b = j % NBUF;
        const uint32_t par = (j / NBUF) & 1;
        uint8_t* sx1 = buf(b);                       // att, then x1, then the output (and y)
        const uint8_t* sxin = buf((j + PROJ) % NBUF);   // x
        const uint32_t x1_base = smem_u32(sx1) + wg * 64 * 64;
        // every stage taken is one commit group; the `pending` groups before stage `it` are not released yet.  pending is a
        // constant at every point of the unrolled tile body, so the release loops unroll and no branch sits between the
        // wgmmas.
        int pending = 0;
        auto take = [&]() -> uint32_t {
            const int s = it % FM_STAGES;
            mbar_wait(&full[s], (it / FM_STAGES) & 1);
            return smem_u32(ring + s * Cfg::STAGE);
        };
        auto commit = [&]() {
            wgmma_commit();
            ++it;
            ++pending;
        };
        // wait until at most n groups are in flight and release the stages of the retired ones
        auto retire = [&](int n) {
            wgmma_wait_n(n);
#pragma unroll
            for (int k = 0; k < FM_STAGES; ++k)
                if (k < pending - n && t == 0) mbar_arrive(&empty[(it - pending + k) % FM_STAGES]);
            pending = min(pending, n);
        };

        if (PROJ) {
            // x1 = x + att Wp^T + bp  (x :453)
            float acc[C / 2];
#pragma unroll
            for (int i = 0; i < C / 2; ++i) acc[i] = 0.f;
            wgmma_fence_operands(acc);   // the zeros are in the accumulator registers before the first wgmma_fence
#pragma unroll
            for (int p = 0; p < NP; ++p) {
                const uint32_t bb = take();
#pragma unroll
                for (int kb = 2 * p; kb < 2 * p + 2 && kb < KB; ++kb) mbar_wait(&abar[b * KB + kb], par);
                wgmma_fence();
#pragma unroll
                for (int kb = 2 * p; kb < 2 * p + 2 && kb < KB; ++kb) {
                    const uint32_t a = x1_base + kb * (FM_ROWS * 64), w = bb + (kb - 2 * p) * (C * 64);
#pragma unroll
                    for (int s = 0; s < 2; ++s)
#pragma unroll
                        for (int h = 0; h < NHALF; ++h)
                            wgmma_f16<96>(half96(acc, h), make_kmajor_desc<64>(a + 32 * s), make_kmajor_desc<64>(w + h * 96 * 64 + 32 * s), 1u);
                }
                commit();
                retire(1);
            }
            retire(0);
            wgmma_fence_operands(acc);
            mbar_wait(&xbar[b], par);
            // x1 over this warpgroup's own 64 rows of att, which its retired proj wgmma no longer reads
#pragma unroll
            for (int q = 0; q < C / 8; ++q) {
                const int col = 8 * q + cq;
                const float2 bq = __ldg(reinterpret_cast<const float2*>(bp + col));
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    const uint32_t off = sw64_off<FM_ROWS>(row0 + 8 * i, col);
                    const float2 xv = __half22float2(*reinterpret_cast<const __half2*>(sxin + off));
                    *reinterpret_cast<__half2*>(sx1 + off) =
                        __floats2half2_rn(xv.x + (acc[4 * q + 2 * i] + bq.x), xv.y + (acc[4 * q + 2 * i + 1] + bq.y));
                }
            }
            fence_async_smem();   // x1 (generic-proxy writes) -> A operand of this warpgroup's fc1 wgmma
            asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
            if (t == 0) mbar_arrive(xfree);   // this warpgroup no longer reads x
        } else {
            mbar_wait(&xbar[b], par);
        }

        float oacc[C / 2];
#pragma unroll
        for (int i = 0; i < C / 2; ++i) oacc[i] = 0.f;
        wgmma_fence_operands(oacc);
        float hacc[2][32];
        uint32_t af[4][4];   // k16 block kk of a chunk: {row g | g+8} x {cols 2t, 2t+8} as in the m16n8k16 A fragment
        // hidden chunk hc before GELU: x1 W1[64 hc : 64 hc + 64]^T, one stage of C/32 K-blocks
        auto fc1 = [&](float (&h)[32]) {
#pragma unroll
            for (int i = 0; i < 32; ++i) h[i] = 0.f;
            wgmma_fence_operands(h);
            const uint32_t bb = take();
            wgmma_fence();
#pragma unroll
            for (int kb = 0; kb < KB; ++kb) {
                const uint32_t a = x1_base + kb * (FM_ROWS * 64), w = bb + kb * (64 * 64);
                wgmma_f16<64>(h, make_kmajor_desc<64>(a), make_kmajor_desc<64>(w), 1u);
                wgmma_f16<64>(h, make_kmajor_desc<64>(a + 32), make_kmajor_desc<64>(w + 32), 1u);
            }
            commit();
        };
        fc1(hacc[0]);
#pragma unroll
        for (int hc = 0; hc < NH; ++hc) {
            const int hb = hc & 1;
            if (hc + 1 < NH) fc1(hacc[hb ^ 1]);
            // fc1(hc) and fc2(hc - 1), the last reader of af, retired; fc1(hc + 1), committed after them, stays in flight
            // during the GELU
            retire(hc + 1 < NH ? 1 : 0);
            wgmma_fence_operands(hacc[hb]);
            // gelu(. + b1) (:444), rounded to fp16 as the reference stores it
#pragma unroll
            for (int kk = 0; kk < 4; ++kk)
#pragma unroll
                for (int q = 0; q < 4; ++q) {
                    const int c8 = 2 * kk + (q >> 1), i = q & 1;
                    const float2 bq = __ldg(reinterpret_cast<const float2*>(b1 + 64 * hc + 8 * c8 + cq));
                    af[kk][q] = pack_half2(gelu_erf(hacc[hb][4 * c8 + 2 * i] + bq.x), gelu_erf(hacc[hb][4 * c8 + 2 * i + 1] + bq.y));
                }
            // out += hidden_chunk W2[:, 64 hc : 64 hc + 64]^T
            const uint32_t bb = take();
            wgmma_fence();
#pragma unroll
            for (int kb = 0; kb < 2; ++kb)
#pragma unroll
                for (int s = 0; s < 2; ++s)
#pragma unroll
                    for (int h = 0; h < NHALF; ++h)
                        wgmma_f16_rs96(half96(oacc, h), af[2 * kb + s], make_kmajor_desc<64>(bb + kb * (C * 64) + h * 96 * 64 + 32 * s), 1u);
            commit();
        }
        retire(0);
        wgmma_fence_operands(oacc);
        // x <- x1 + mlp(x1) (:454), in place over the x1 tile: stored with TMA (CS == 0) or the A operand of y
#pragma unroll
        for (int q = 0; q < C / 8; ++q) {
            const int col = 8 * q + cq;
            const float2 bq = __ldg(reinterpret_cast<const float2*>(b2 + col));
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                __half2* p = reinterpret_cast<__half2*>(sx1 + sw64_off<FM_ROWS>(row0 + 8 * i, col));
                const float2 xv = __half22float2(*p);
                *p = __floats2half2_rn(xv.x + (oacc[4 * q + 2 * i] + bq.x), xv.y + (oacc[4 * q + 2 * i + 1] + bq.y));
            }
        }
        fence_async_smem();
        if constexpr (CS > 0) {
            // y = x . Wy^T + by from this warpgroup's 64 rows of the tile, in the K order of a GEMM over the stored x, so y is
            // the same as to_image's Linear run on this block's output
            asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
            float yacc[CS / 2];
#pragma unroll
            for (int i = 0; i < CS / 2; ++i) yacc[i] = 0.f;
            wgmma_fence_operands(yacc);
            const uint32_t bb = take();
            wgmma_fence();
#pragma unroll
            for (int kb = 0; kb < KB; ++kb) {
                const uint32_t a = x1_base + kb * (FM_ROWS * 64), w = bb + kb * (CS * 64);
                wgmma_f16<CS>(yacc, make_kmajor_desc<64>(a), make_kmajor_desc<64>(w), 1u);
                wgmma_f16<CS>(yacc, make_kmajor_desc<64>(a + 32), make_kmajor_desc<64>(w + 32), 1u);
            }
            commit();
            retire(0);
            wgmma_fence_operands(yacc);
            // staged over the x tile as CS/16 boxes of [128][16] with the 32B swizzle, which overlaps the other warpgroup's
            // rows of x: both warpgroups' y wgmma must have retired first
            consumer_bar_sync();
#pragma unroll
            for (int q = 0; q < CS / 8; ++q) {
                const int col = 8 * q + cq;
                const float2 bq = __ldg(reinterpret_cast<const float2*>(by + col));
#pragma unroll
                for (int i = 0; i < 2; ++i) {
                    __half2* p = reinterpret_cast<__half2*>(sx1 + (col >> 4) * (FM_ROWS * 32) + stage_off<16>(row0 + 8 * i, (col & 15) >> 3) +
                                                            (col & 7) * 2);
                    *p = __floats2half2_rn(yacc[4 * q + 2 * i] + bq.x, yacc[4 * q + 2 * i + 1] + bq.y);
                }
            }
            fence_async_smem();
        }
        asm volatile("bar.sync %0, 128;" ::"r"(2 + wg) : "memory");
        if (t == 0) mbar_arrive(&outw[b]);   // this warpgroup's rows are written: warp 9 may store the tile
    }
}

static int map2d(CUtensorMap* m, const void* base, int cols, long long rows, int box_rows) {
    const cuuint64_t dims[2] = {(cuuint64_t)cols, (cuuint64_t)rows};
    const cuuint64_t strides[1] = {(cuuint64_t)cols * 2};
    const cuuint32_t box[2] = {32, (cuuint32_t)box_rows};
    return encode(m, base, 2, dims, strides, box, 64);
}

template <int C, bool PROJ, int CS = 0>
static int launch_mlp(cudaStream_t st, int ntiles, const FmMaps& maps, const float* bp, const float* b1, const float* b2,
                      const float* by = nullptr) {
    if (ensure_dyn_smem((const void*)swin_mlp_fused_kernel<C, PROJ, CS>, FmCfg<C>::SMEM)) return 1;
    // programmatic dependent launch (as gemm.cu): the producer's set-up and first weight stages overlap the head's last wave
    cudaLaunchConfig_t cfg = {};
    // persistent: one CTA per SM (g_tune[10] > 0 caps the grid, for tests; a tile's result does not depend on its CTA)
    int grid = std::min(ntiles, device_sm_count());
    if (g_tune[10] > 0) grid = std::min(grid, g_tune[10]);
    cfg.gridDim = dim3((unsigned)grid); cfg.blockDim = dim3(FM_THREADS); cfg.dynamicSmemBytes = FmCfg<C>::SMEM;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    NB_CUDA(cudaLaunchKernelEx(&cfg, swin_mlp_fused_kernel<C, PROJ, CS>, maps, bp, b1, b2, by, ntiles));
    NB_LAUNCHED();
    return 0;
}

int swin_mlp_fused(cudaStream_t st, __half* x, const __half* att, long long T, int C, const __half* wp, const float* bp,
                   const __half* w1, const float* b1, const __half* w2, const float* b2, __half* y, int cs, const __half* wy,
                   const float* by) {
    NB_CHECK(x && w1 && b1 && w2 && b2 && (!att || (wp && bp)) && (!y || (att && wy && by)), "null pointer");
    NB_CHECK(C == 96 || C == 192, "C must be 96 or 192");
    NB_CHECK(!y || (C == 192 && cs == 48) || (C == 96 && cs == 16), "y: cs must be 48 at C = 192 and 16 at C = 96");
    NB_CHECK(T > 0 && T < (1LL << 31), "token count out of range");
    FmMaps maps;
    memset(&maps, 0, sizeof(maps));
    if (map2d(&maps.x, x, C, T, FM_ROWS)) return 1;
    if (att && (map2d(&maps.att, att, C, T, FM_ROWS) || map2d(&maps.wp, wp, C, C, C))) return 1;
    if (map2d(&maps.w1, w1, C, 2 * C, 64) || map2d(&maps.w2, w2, 2 * C, C, C)) return 1;
    if (y) {
        if (map2d(&maps.wy, wy, C, cs, cs)) return 1;
        const cuuint64_t dims[2] = {(cuuint64_t)cs, (cuuint64_t)T};
        const cuuint64_t strides[1] = {(cuuint64_t)cs * 2};
        const cuuint32_t box[2] = {16, FM_ROWS};
        if (encode(&maps.y, y, 2, dims, strides, box, 32)) return 1;
    }
    const double Td = (double)T;
    ProfScope ps(st, PC_FUSED_MLP, Td * C * 2 * (C * ((att ? 1 : 0) + 4) + (y ? cs : 0)), Td * C * 2 * (att ? 2 : 1),
                 Td * (y ? cs : C) * 2);
    const int ntiles = (int)((T + FM_ROWS - 1) / FM_ROWS);
    if (rec_on()) rec_launch("swin_mlp", {{"T", T}, {"C", C}, {"proj", att ? 1 : 0}, {"cs", y ? cs : 0}});
    if (y) return C == 96 ? launch_mlp<96, true, 16>(st, ntiles, maps, bp, b1, b2, by) : launch_mlp<192, true, 48>(st, ntiles, maps, bp, b1, b2, by);
    if (C == 96) return att ? launch_mlp<96, true>(st, ntiles, maps, bp, b1, b2) : launch_mlp<96, false>(st, ntiles, maps, bp, b1, b2);
    return att ? launch_mlp<192, true>(st, ntiles, maps, bp, b1, b2) : launch_mlp<192, false>(st, ntiles, maps, bp, b1, b2);
}

}  // namespace nb200

using namespace nb200;

extern "C" int nb200_swin_mlp_fused_f16(void* x, const void* att, long long T, int C, const void* wp, const float* bp,
                                        const void* w1, const float* b1, const void* w2, const float* b2, void* stream) {
    return swin_mlp_fused((cudaStream_t)stream, (__half*)x, (const __half*)att, T, C, (const __half*)wp, bp, (const __half*)w1, b1,
                          (const __half*)w2, b2, nullptr, 0, nullptr, nullptr);
}

// The tail of the network's last block, which also runs to_image's Linear (the CS instantiations): x is left unchanged
extern "C" int nb200_swin_mlp_fused_y_f16(void* x, const void* att, long long T, int C, const void* wp, const float* bp,
                                          const void* w1, const float* b1, const void* w2, const float* b2, void* y, int cs,
                                          const void* wy, const float* by, void* stream) {
    NB_CHECK(y, "null pointer");
    return swin_mlp_fused((cudaStream_t)stream, (__half*)x, (const __half*)att, T, C, (const __half*)wp, bp, (const __half*)w1, b1,
                          (const __half*)w2, b2, (__half*)y, cs, (const __half*)wy, by);
}
