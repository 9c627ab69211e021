// Shifted-window attention core on tensor cores (mma.sync m16n8k16, fp16 in / fp32 accumulate).
//
// One CTA per 6x6 window, one warp per head (6 warps), 4 CTAs per SM (6 for d = 16).  q/k/v rows are staged with
// cp.async (16-byte LDGSTS, no register round trip).  The 36 tokens are padded to 48 MMA rows by clamping
// the row index (padded keys are masked by select, padded probabilities are exactly 0):
//   S = (Q*scale) K^T : M=48 (3 m16 tiles), N=48 (6 n8 tiles), K=d (d/16 steps)
//   softmax on the accumulator fragments (quad shuffles), relative-position bias and the
//   shift mask added per element, padded keys masked out
//   O = P V           : the S fragments are re-packed in registers as the A operand (no smem trip),
//                       V fragments come from ldmatrix.trans
// torchvision swin_transformer.py:166-221 (roll, partition, bias :190, mask :193-209, softmax :211,
// attn@v :214, un-roll) - everything but the qkv / proj Linears, which run on the wgmma GEMM.
//
// The 36x36 problem per head is far too small for a 64-row wgmma tile, and the op moves
// 8*C bytes/token for ~144*C FLOP/token: it is HBM/L2-bound, so the warp-level HMMA path is the
// right instrument here (DESIGN.md 4.2).
#include "common.cuh"
#include "gemm_wgmma.cuh"
#include "swin_kernels.h"
#include "tmap.h"
#include <map>
#include <mutex>

namespace nb200 {

extern int g_tune[16];  // gemm.cu (nb200_tune_set)

namespace {
constexpr int WS = 6, WTOK = 36, WPAD = 48, HEADS = 6;
}  // namespace

constexpr int NKT = 5;   // key tiles of 8 columns covering the 36 keys (columns 36..39 are masked by the bias table)

template <int D>
struct AttnCtx {
    __half* sq;
    const int* sreg;
    const float4* bf;
    const __half* kbase[NKT];
    const __half* vbase[3];
    int hc, g, t4;
    float scale;
    bool boundary;
};

// One 16-row query tile of one head: S = Q K^T, bias/mask, base-2 softmax numerators, O = P V, normalise, stage.
// LD: row stride (halves) of the q/k/v tiles.  LAST: query rows 32..35 only (accumulator rows g+8 are padding and are not
// evaluated).
template <int D, int LD, bool LAST>
__device__ __forceinline__ void attn_mtile(const AttnCtx<D>& cx, int mt) {
    constexpr uint32_t ONES = 0x3C003C00u;   // half2(1, 1)
    constexpr int HL = LAST ? 1 : 2;         // accumulator row halves in use
    const int g = cx.g, t4 = cx.t4, hc = cx.hc;
    const int row0 = min(mt * 16 + g, WTOK - 1), row1 = min(mt * 16 + g + 8, WTOK - 1);
    // ---- S = Q K^T
    float s[NKT][4];
#pragma unroll
    for (int nt = 0; nt < NKT; ++nt)
#pragma unroll
        for (int r = 0; r < 4; ++r) s[nt][r] = 0.f;
#pragma unroll
    for (int kt = 0; kt < D / 16; ++kt) {
        uint32_t a[4];
        const __half* p0 = cx.sq + row0 * LD + hc + kt * 16 + 2 * t4;
        const __half* p1 = cx.sq + row1 * LD + hc + kt * 16 + 2 * t4;
        a[0] = *reinterpret_cast<const uint32_t*>(p0);
        a[1] = *reinterpret_cast<const uint32_t*>(p1);
        a[2] = *reinterpret_cast<const uint32_t*>(p0 + 8);
        a[3] = *reinterpret_cast<const uint32_t*>(p1 + 8);
#pragma unroll
        for (int nt = 0; nt < NKT; ++nt) {
            const __half* pk = cx.kbase[nt] + kt * 16;
            mma16816(s[nt], a, *reinterpret_cast<const uint32_t*>(pk), *reinterpret_cast<const uint32_t*>(pk + 8));
        }
    }
    // ---- scale + bias (+ mask).  element r of tile nt: row = mt*16 + g + 8*(r>>1), col = nt*8 + 2*t4 + (r&1).
    // bias_frag holds log2(e)*relative_position_bias in exactly this fragment order (padded keys = -1e30), so
    // scale + bias + key padding is one FMA per element and the softmax runs in base 2.
#pragma unroll
    for (int nt = 0; nt < NKT; ++nt) {
        const float4 bv = __ldg(cx.bf + (mt * 6 + nt) * 32);
        s[nt][0] = fmaf(s[nt][0], cx.scale, bv.x);
        s[nt][1] = fmaf(s[nt][1], cx.scale, bv.y);
        if (!LAST) {
            s[nt][2] = fmaf(s[nt][2], cx.scale, bv.z);
            s[nt][3] = fmaf(s[nt][3], cx.scale, bv.w);
        }
    }
    if (cx.boundary) {  // -100 across regions (:193-209)
        const int q0 = cx.sreg[row0], q1 = cx.sreg[row1];
#pragma unroll
        for (int nt = 0; nt < NKT; ++nt)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                const int cr = cx.sreg[min(nt * 8 + 2 * t4 + e, WTOK - 1)];
                if (cr != q0) s[nt][e] += -100.0f * 1.4426950408889634f;
                if (!LAST && cr != q1) s[nt][2 + e] += -100.0f * 1.4426950408889634f;
            }
    }
    // ---- softmax numerators (base 2).  The row sums come out of the P V product itself (a ones column appended to V),
    // i.e. they are the sums of exactly the fp16 probabilities that multiply V; 1/sum is applied to the output rows.
#pragma unroll
    for (int hlf = 0; hlf < HL; ++hlf) {
        float mx = -1e30f;
#pragma unroll
        for (int nt = 0; nt < NKT; ++nt) mx = fmaxf(mx, fmaxf(s[nt][2 * hlf], s[nt][2 * hlf + 1]));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 1));
        mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, 2));
#pragma unroll
        for (int nt = 0; nt < NKT; ++nt)
#pragma unroll
            for (int e = 0; e < 2; ++e) {
                s[nt][2 * hlf + e] = ex2(s[nt][2 * hlf + e] - mx);
            }
    }
    if (LAST) {
#pragma unroll
        for (int nt = 0; nt < NKT; ++nt) s[nt][2] = s[nt][3] = 0.f;
    }
    // ---- O = P V  (P in fp16, un-normalised: values in [0, 1]); osum = P 1
    float o[D / 8][4], osum[4] = {0.f, 0.f, 0.f, 0.f};
#pragma unroll
    for (int nt = 0; nt < D / 8; ++nt)
#pragma unroll
        for (int r = 0; r < 4; ++r) o[nt][r] = 0.f;
#pragma unroll
    for (int kt = 0; kt < 2; ++kt) {
        uint32_t a[4];
        a[0] = pack_half2(s[2 * kt][0], s[2 * kt][1]);
        a[1] = pack_half2(s[2 * kt][2], s[2 * kt][3]);
        a[2] = pack_half2(s[2 * kt + 1][0], s[2 * kt + 1][1]);
        a[3] = pack_half2(s[2 * kt + 1][2], s[2 * kt + 1][3]);
        mma16816(osum, a, ONES, ONES);
#pragma unroll
        for (int nt = 0; nt < D / 8; ++nt) {
            uint32_t b[2];
            ldmatrix_x2_trans(b, smem_u32(cx.vbase[kt] + nt * 8));
            mma16816(o[nt], a, b[0], b[1]);
        }
    }
    {
        const uint32_t a0 = pack_half2(s[4][0], s[4][1]), a1 = pack_half2(s[4][2], s[4][3]);
        mma1688(osum, a0, a1, ONES);
#pragma unroll
        for (int nt = 0; nt < D / 8; ++nt) {
            mma1688(o[nt], a0, a1, ldmatrix_x1_trans(smem_u32(cx.vbase[2] + nt * 8)));
        }
    }
    const float inv0 = __fdividef(1.f, osum[0]);
    const float inv1 = LAST ? 0.f : __fdividef(1.f, osum[2]);
    // ---- stage this head's output columns into sq.  Each warp only ever reads and writes its own columns of
    // rows [16*mt, 16*mt+16) here, and those q rows are dead once this m-tile's S is done.
    __syncwarp();
    const int r0 = mt * 16 + g, r1 = r0 + 8;
#pragma unroll
    for (int nt = 0; nt < D / 8; ++nt) {
        if (!LAST || r0 < WTOK) *reinterpret_cast<uint32_t*>(cx.sq + r0 * LD + hc + nt * 8 + 2 * t4) = pack_half2(o[nt][0] * inv0, o[nt][1] * inv0);
        if (!LAST) *reinterpret_cast<uint32_t*>(cx.sq + r1 * LD + hc + nt * 8 + 2 * t4) = pack_half2(o[nt][2] * inv1, o[nt][3] * inv1);
    }
}

template <int D>
__global__ void __launch_bounds__(192, D == 16 ? 6 : 4) window_attention_mma_kernel(const __half* __restrict__ qkv, const float4* __restrict__ bias_frag,
                                                                   __half* __restrict__ out, int H, int W, int shift,
                                                                   size_t plane) {
    if (threadIdx.x == 0) NB_PDL_TRIGGER();
    constexpr int C = D * HEADS;
    constexpr int LD = C + 8;  // padded row: (C+8)*2 bytes = 4 words mod 32 banks -> conflict-free fragment loads
    extern __shared__ __align__(16) unsigned char smem_raw[];
    __half* sq = reinterpret_cast<__half*>(smem_raw);  // [WTOK][LD]  q, later the output tile
    __half* sk = sq + WTOK * LD;
    __half* sv = sk + WTOK * LD;
    int* stok = reinterpret_cast<int*>(sv + WTOK * LD);      // [WTOK]
    int* sreg = stok + WTOK;                                 // [WPAD]
    const int nww = W / WS;
    const int wx = blockIdx.x % nww, wy = blockIdx.x / nww, b = blockIdx.y;
    const int tid = threadIdx.x;
    if (tid < WPAD) {
        int reg = -1;
        if (tid < WTOK) {
            const int ry = wy * WS + tid / WS, rx = wx * WS + tid % WS;  // rolled coordinates
            const int y = (ry + shift) % H, x = (rx + shift) % W;        // torch.roll(-shift) :166-167
            stok[tid] = (b * H + y) * W + x;
            int hr = 0, wr = 0;
            if (shift > 0) {
                hr = ry < H - WS ? 0 : (ry < H - shift ? 1 : 2);
                wr = rx < W - WS ? 0 : (rx < W - shift ? 1 : 2);
            }
            reg = hr * 3 + wr;
        }
        sreg[tid] = reg;
    }
    __syncthreads();
    // ---- stage q, k, v: three dense [T][C] planes (the qkv GEMM writes them split, OUT_SPLIT), 16-byte cp.async each.
    // thread -> (16-byte column vv, row group rg); it walks tokens rg, rg+RG, ... of all three planes
    constexpr int VPT = C / 8;         // 16-byte columns per token row: 24 (C=192) or 12 (C=96)
    constexpr int RG = 192 / VPT;      // 8 or 16 row groups
    const int vv = tid % VPT, rg = tid / VPT;
    for (int t = rg; t < WTOK; t += RG) {
        const __half* src = qkv + (size_t)stok[t] * C + vv * 8;
        __half* dst = sq + t * LD + vv * 8;
        cp_async16(dst, src);
        cp_async16(dst + WTOK * LD, src + plane);
        cp_async16(dst + 2 * WTOK * LD, src + 2 * plane);
    }
    cp_async_commit();
    cp_async_wait<0>();
    __syncthreads();

    const int head = tid >> 5, lane = tid & 31, g = lane >> 2, t4 = lane & 3;
    const int hc = head * D;
    const float scale = ((D == 16) ? 0.25f : 0.17677669529663687f) * 1.4426950408889634f;  // (C//heads)**-0.5 (:187) * log2(e)
    const bool boundary = shift > 0 && (wy == gridDim.x / nww - 1 || wx == nww - 1);  // only these windows mix mask regions
    const float4* bf = bias_frag + (size_t)head * (3 * 6 * 32) + lane;
    AttnCtx<D> cx;
    cx.sq = sq; cx.sreg = sreg; cx.bf = bf; cx.hc = hc; cx.g = g; cx.t4 = t4; cx.scale = scale; cx.boundary = boundary;
    // per-thread fragment base pointers (row clamps and column offsets resolved once).  36 keys = 4.5 n8 tiles: S uses
    // 5 key tiles (40 columns), P V uses two k16 steps and one k8 step.
#pragma unroll
    for (int nt = 0; nt < NKT; ++nt) cx.kbase[nt] = sk + min(nt * 8 + g, WTOK - 1) * LD + hc + 2 * t4;
    cx.vbase[0] = sv + (lane & 15) * LD + hc;
    cx.vbase[1] = sv + (16 + (lane & 15)) * LD + hc;
    cx.vbase[2] = sv + min(32 + (lane & 7), WTOK - 1) * LD + hc;
    // One 16-row m-tile at a time (rows 0-15, 16-31, 32-47): keeps the live state at 20 + 4*D/8 (+4) accumulators so that
    // 4 CTAs fit per SM; K / V fragments are re-read from shared memory per m-tile (cheap, conflict-free).
    // The last tile holds query rows 32..35 only: its upper half (rows 40..47) is skipped.
#pragma unroll 1
    for (int mt = 0; mt < 2; ++mt) attn_mtile<D, LD, false>(cx, mt);
    attn_mtile<D, LD, true>(cx, 2);
    __syncthreads();
    for (int t = rg; t < WTOK; t += RG)
        *reinterpret_cast<uint4*>(out + (size_t)stok[t] * C + vv * 8) = *reinterpret_cast<const uint4*>(sq + t * LD + vv * 8);
}

// bias_frag[head][mt][nt][lane] (float4 = accumulator fragment order) = log2(e) * table[rel_index(row, col)][head];
// padded key columns (>= 36) hold -1e30 so they vanish in the softmax; padded query rows hold 0.
__global__ void build_bias_frag_kernel(const float* __restrict__ table, float4* __restrict__ frag) {
    const int i = blockIdx.x * blockDim.x + threadIdx.x;  // ((head*3 + mt)*6 + nt)*32 + lane
    if (i >= HEADS * 3 * 6 * 32) return;
    const int lane = i & 31, nt = (i >> 5) % 6, mt = (i / (32 * 6)) % 3, head = i / (32 * 6 * 3);
    const int g = lane >> 2, t4 = lane & 3;
    float v[4];
#pragma unroll
    for (int r = 0; r < 4; ++r) {
        const int row = mt * 16 + g + 8 * (r >> 1), col = nt * 8 + 2 * t4 + (r & 1);
        if (col >= WTOK) v[r] = -1e30f;
        else if (row >= WTOK) v[r] = 0.f;
        else {
            const int qy = row / WS, qx = row % WS, ky = col / WS, kx = col % WS;
            // relative_position_index (swin_transformer.py:267-279)
            v[r] = 1.4426950408889634f * table[((qy - ky + WS - 1) * (2 * WS - 1) + (qx - kx + WS - 1)) * HEADS + head];
        }
    }
    frag[i] = make_float4(v[0], v[1], v[2], v[3]);
}

int build_bias_frag(cudaStream_t st, const float* table, float* frag) {
    build_bias_frag_kernel<<<(HEADS * 3 * 6 * 32 + 255) / 256, 256, 0, st>>>(table, reinterpret_cast<float4*>(frag));
    NB_LAUNCHED();
    return 0;
}

template <int D>
static size_t attn_smem_bytes() {
    constexpr int C = D * HEADS, LD = C + 8;
    return (size_t)3 * WTOK * LD * 2 + (WTOK + WPAD) * 4 + 16;
}

// opt-in shared memory + carveout, per (device, kernel): both attributes are per-device state
static int set_attn_attrs(const void* func, size_t smem, int carveout) {
    static std::mutex mu;
    static std::map<std::pair<int, const void*>, int> done;
    int dev = 0;
    NB_CUDA(cudaGetDevice(&dev));
    std::lock_guard<std::mutex> lk(mu);
    int& have = done[{dev, func}];
    if (have != carveout) {
        NB_CUDA(cudaFuncSetAttribute(func, cudaFuncAttributeMaxDynamicSharedMemorySize, (int)smem));
        NB_CUDA(cudaFuncSetAttribute(func, cudaFuncAttributePreferredSharedMemoryCarveout, carveout));
        have = carveout;
    }
    return 0;
}

int window_attention(cudaStream_t st, const __half* qkv, const float* bias_frag_f, __half* out, int B, int H, int W, int C,
                     int shift, size_t plane) {
    const float4* bias_table = reinterpret_cast<const float4*>(bias_frag_f);
    NB_CHECK(H % WS == 0 && W % WS == 0, "feature map must be a multiple of the 6x6 window");
    NB_CHECK(C == 96 || C == 192, "window attention supports C=96 (d=16) and C=192 (d=32)");
    if (WS >= H) shift = 0;  // torchvision :151-155
    dim3 grid((H / WS) * (W / WS), B);
    ProfScope ps(st, PC_ATTN, (double)B * H * W * C * 4 * 2, (double)B * H * W * C * 3 * 2, (double)B * H * W * C * 2);  // q,k,v in; out
    // shared-memory carveout: just enough for the 4 resident CTAs, the rest stays L1 (the per-head bias fragments,
    // 55 KB per layer, are re-read by every window and should hit there).  g_tune[6] overrides the percentage.
    if (C == 96) {
        const int want = g_tune[6] > 0 ? g_tune[6] : 72;   // 6 CTAs x 23.6 KB
        if (set_attn_attrs((const void*)window_attention_mma_kernel<16>, attn_smem_bytes<16>(), want)) return 1;
        window_attention_mma_kernel<16><<<grid, 192, attn_smem_bytes<16>(), st>>>(qkv, bias_table, out, H, W, shift, plane);
    } else {
        const int want = g_tune[6] > 0 ? g_tune[6] : 86;
        if (set_attn_attrs((const void*)window_attention_mma_kernel<32>, attn_smem_bytes<32>(), want)) return 1;
        window_attention_mma_kernel<32><<<grid, 192, attn_smem_bytes<32>(), st>>>(qkv, bias_table, out, H, W, shift, plane);
    }
    NB_LAUNCHED();
    return 0;
}


// ---------------------------------------------------------------------------------------------
// Fused block head: att = window_attention_core(x . Wqkv^T + bqkv), q/k/v never leave shared memory.
// One CTA = 3 windows = 108 tokens (+20 zero rows) = the 128 rows of two wgmma warpgroups.
// q|k|v is computed head-major in C/32 chunks of 96 columns: chunk c holds columns [32c, 32c+32) of q, of k and of v, i.e.
// head c (d = 32) or heads 2c, 2c+1 (d = 16), so it is complete input of the attention core for those heads.
//   warp 8    : TMA producer of the weight blocks: per (chunk c, K-block) the rows 32c, C + 32c and 2C + 32c of Wqkv as three
//               [32][32] boxes (64B swizzle) stacked into one [96][32] operand, C/32 chunks x C/32 K-blocks
//   warps 0-7 : gather the rolled window tokens into a swizzled [128][C] A tile (cp.async); per chunk one wgmma
//               accumulation (M = 64 per warpgroup), bias, fp16 into the chunk's per-window q/k/v tiles; then the chunk's
//               (window, head, m-tile) items of the mma.sync attention core (attn_mtile, the same code as
//               window_attention_mma_kernel) on the 8 warps, each warp writing its un-rolled output rows back to HBM.
// Only one chunk of q/k/v is resident (25 KB instead of 127 KB for all heads at C = 192), so two CTAs share an SM at both C
// and one CTA's GEMM overlaps the other's attention.
// ---------------------------------------------------------------------------------------------
constexpr int FA_ROWS = 128, FA_WIN = 3, FA_THREADS = GEMM_CONSUMER_THREADS + 32, FA_SLOT = 96 * 64, FA_STAGES = 4;
constexpr int FA_LD = 32 + 8;   // chunk tile row: 80 B = 20 words, so fragment loads and ldmatrix rows are conflict-free
constexpr int FA_CHUNK_BYTES = FA_WIN * 3 * WTOK * FA_LD * 2;

template <int C>
struct FaCfg {
    static constexpr int X_BYTES = FA_ROWS * C * 2;
    static constexpr int SMEM = X_BYTES + FA_STAGES * FA_SLOT + FA_CHUNK_BYTES + FA_WIN * (WTOK + WPAD) * 4 + 2 * FA_STAGES * 8 + 1024;
};

template <int C>
__global__ void __launch_bounds__(FA_THREADS, 2) swin_attn_fused_kernel(const __grid_constant__ CUtensorMap wmap,
                                                                        const __half* __restrict__ x, const float* __restrict__ bqkv,
                                                                        const float4* __restrict__ bias_frag, __half* __restrict__ out,
                                                                        int H, int W, int shift, int nwin) {
    using Cfg = FaCfg<C>;
    constexpr int D = C / HEADS, KB = C / 32, NCH = C / 32, HPC = 32 / D;   // HPC: heads per chunk
    extern __shared__ uint8_t smem_dyn[];
    uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_dyn) + 1023) & ~(uintptr_t)1023);
    uint8_t* sx = smem;
    uint8_t* ring = smem + Cfg::X_BYTES;
    __half* sqkv = reinterpret_cast<__half*>(ring + FA_STAGES * FA_SLOT);   // [window][q|k|v][WTOK][FA_LD], one chunk
    int* stok = reinterpret_cast<int*>(reinterpret_cast<uint8_t*>(sqkv) + FA_CHUNK_BYTES);   // [window][WTOK], -1 = none
    int* sreg = stok + FA_WIN * WTOK;                                                         // [window][WPAD]
    uint64_t* full = reinterpret_cast<uint64_t*>(sreg + FA_WIN * WPAD);
    uint64_t* empty = full + FA_STAGES;
    const int tid = threadIdx.x, warp = tid >> 5;
    const int nww = W / WS, nwy = H / WS;
    if (tid < FA_WIN * WPAD) {
        const int w = tid / WPAD, t = tid % WPAD, gw = blockIdx.x * FA_WIN + w;
        int reg = -1;
        if (t < WTOK) {
            int tok = -1;
            if (gw < nwin) {
                const int b = gw / (nww * nwy), r = gw % (nww * nwy), wy = r / nww, wx = r % nww;
                const int ry = wy * WS + t / WS, rx = wx * WS + t % WS;       // rolled coordinates
                const int y = (ry + shift) % H, xx = (rx + shift) % W;        // torch.roll(-shift) :166-167
                tok = (b * H + y) * W + xx;
                int hr = 0, wr = 0;
                if (shift > 0) {
                    hr = ry < H - WS ? 0 : (ry < H - shift ? 1 : 2);
                    wr = rx < W - WS ? 0 : (rx < W - shift ? 1 : 2);
                }
                reg = hr * 3 + wr;
            }
            stok[w * WTOK + t] = tok;
        }
        sreg[w * WPAD + t] = reg;
    }
    if (tid == GEMM_CONSUMER_THREADS) {
        tma_prefetch_desc(&wmap);
        for (int s = 0; s < FA_STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 2);   // one arrival per consumer warpgroup
        }
        fence_barrier_init();
    }
    __syncthreads();
    // the block tail (swin_block.cu, a PDL launch) may start its prologue and weight loads once every CTA of this grid is resident
    if (tid == 0) NB_PDL_TRIGGER();

    if (warp == GEMM_CONSUMER_THREADS / 32) {
        // ===================== weight producer =====================
        if (elect_one()) {
            for (int i = 0; i < NCH * KB; ++i) {
                const int s = i % FA_STAGES, c = i / KB;
                mbar_wait(&empty[s], ((i / FA_STAGES) & 1) ^ 1);
                mbar_expect_tx(&full[s], FA_SLOT);
                // 32-row boxes at 2 KB offsets: the 64B swizzle repeats every 512 B, so the stack is laid out as one 96-row box
#pragma unroll
                for (int m = 0; m < 3; ++m)
                    tma_load_2d(&wmap, &full[s], ring + s * FA_SLOT + m * 32 * 64, (i % KB) * 32, m * C + 32 * c);
            }
        }
        return;
    }

    // ===================== gather: row r = window r/36, token r%36; rows >= 108 and missing windows are zero =====================
    // 16-byte cp.async copies: all of a thread's loads are in flight at once
    for (int i = tid; i < FA_ROWS * (C / 8); i += GEMM_CONSUMER_THREADS) {
        const int r = i / (C / 8), u = i % (C / 8);
        uint8_t* dst = sx + (u >> 2) * (FA_ROWS * 64) + stage_off<32>(r, u & 3);
        const int tok = r < FA_WIN * WTOK ? stok[r] : -1;
        if (tok >= 0) cp_async16(dst, x + (size_t)tok * C + u * 8);
        else *reinterpret_cast<uint4*>(dst) = make_uint4(0u, 0u, 0u, 0u);
    }
    cp_async_commit();
    cp_async_wait<0>();
    fence_async_smem();   // generic-proxy writes of the A tile -> visible to wgmma
    consumer_bar_sync();

    const int wg = tid >> 7, t = tid & 127;
    const int row0 = wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2);
    const int cq = 2 * (t & 3);
    const uint32_t a_base = smem_u32(sx) + wg * 64 * 64;
    const int lane = tid & 31, g = lane >> 2, t4 = lane & 3;
    const float scale = ((D == 16) ? 0.25f : 0.17677669529663687f) * 1.4426950408889634f;  // (C//heads)**-0.5 (:187) * log2(e)
#pragma unroll 1
    for (int c = 0; c < NCH; ++c) {
        // ===================== chunk c of q | k | v = x Wqkv^T + b =====================
        float acc[48];
#pragma unroll
        for (int j = 0; j < 48; ++j) acc[j] = 0.f;
#pragma unroll 1
        for (int kb = 0; kb < KB; ++kb) {
            const int it = c * KB + kb, s = it % FA_STAGES;
            mbar_wait(&full[s], (it / FA_STAGES) & 1);
            const uint32_t a = a_base + kb * (FA_ROWS * 64), bb = smem_u32(ring + s * FA_SLOT);
            wgmma_fence();
            wgmma_f16<96>(acc, make_kmajor_desc<64>(a), make_kmajor_desc<64>(bb), 1u);
            wgmma_f16<96>(acc, make_kmajor_desc<64>(a + 32), make_kmajor_desc<64>(bb + 32), 1u);
            wgmma_commit();
            // keep one group in flight: the stage read by the previous group is released once that group retired
            wgmma_wait<1>();
            if (kb > 0 && t == 0) mbar_arrive(&empty[(it - 1) % FA_STAGES]);
        }
        wgmma_wait<0>();
        if (t == 0) mbar_arrive(&empty[(c * KB + KB - 1) % FA_STAGES]);
        wgmma_fence_operands(acc);
        consumer_bar_sync();   // every warp is done with the previous chunk's q/k/v
#pragma unroll
        for (int j = 0; j < 12; ++j) {
            const int m = j >> 2, col = 8 * (j & 3) + cq;   // q|k|v, column within the chunk
            const float2 bq = __ldg(reinterpret_cast<const float2*>(bqkv + m * C + 32 * c + col));
#pragma unroll
            for (int i = 0; i < 2; ++i) {
                const int r = row0 + 8 * i;
                if (r < FA_WIN * WTOK) {
                    const int w = r / WTOK, tk = r - w * WTOK;
                    *reinterpret_cast<__half2*>(sqkv + ((w * 3 + m) * WTOK + tk) * FA_LD + col) =
                        __floats2half2_rn(acc[4 * j + 2 * i] + bq.x, acc[4 * j + 2 * i + 1] + bq.y);
                }
            }
        }
        consumer_bar_sync();

        // ===================== attention: the chunk's (window, head, m-tile) items on the 8 consumer warps =====================
        // m-tile-major order, so that the items left over for a last round are the cheap 4-row tiles
#pragma unroll 1
        for (int item = warp; item < 3 * FA_WIN * HPC; item += GEMM_CONSUMER_THREADS / 32) {
            const int mt = item / (FA_WIN * HPC), pr = item - mt * (FA_WIN * HPC), w = pr / HPC, hh = pr - w * HPC;
            const int gw = blockIdx.x * FA_WIN + w;
            if (gw >= nwin) continue;
            const int r = gw % (nww * nwy), wy = r / nww, wx = r % nww, head = c * HPC + hh;
            __half* sq = sqkv + w * 3 * WTOK * FA_LD;
            __half* sk = sq + WTOK * FA_LD;
            __half* sv = sk + WTOK * FA_LD;
            AttnCtx<D> cx;
            cx.sq = sq; cx.sreg = sreg + w * WPAD; cx.bf = bias_frag + (size_t)head * (3 * 6 * 32) + lane;
            cx.hc = hh * D; cx.g = g; cx.t4 = t4; cx.scale = scale;
            cx.boundary = shift > 0 && (wy == nwy - 1 || wx == nww - 1);   // only these windows mix mask regions
#pragma unroll
            for (int nt = 0; nt < NKT; ++nt) cx.kbase[nt] = sk + min(nt * 8 + g, WTOK - 1) * FA_LD + cx.hc + 2 * t4;
            cx.vbase[0] = sv + (lane & 15) * FA_LD + cx.hc;
            cx.vbase[1] = sv + (16 + (lane & 15)) * FA_LD + cx.hc;
            cx.vbase[2] = sv + min(32 + (lane & 7), WTOK - 1) * FA_LD + cx.hc;
            if (mt < 2) attn_mtile<D, FA_LD, false>(cx, mt);
            else attn_mtile<D, FA_LD, true>(cx, 2);
            // the m-tile's output rows (staged over its own q rows by this warp) -> HBM, D columns = D/8 16-byte pieces per row
            __syncwarp();
            const int nrow = mt < 2 ? 16 : WTOK - 32;
            for (int e = lane; e < nrow * (D / 8); e += 32) {
                const int tk = 16 * mt + e / (D / 8), u = e % (D / 8);
                *reinterpret_cast<uint4*>(out + (size_t)stok[w * WTOK + tk] * C + head * D + u * 8) =
                    *reinterpret_cast<const uint4*>(sq + tk * FA_LD + cx.hc + u * 8);
            }
        }
    }
}

int swin_attn_fused(cudaStream_t st, const __half* x, const __half* wqkv, const float* bqkv, const float* bias_frag_f, __half* att,
                    int B, int H, int W, int C, int shift) {
    NB_CHECK(x && wqkv && bqkv && bias_frag_f && att, "null pointer");
    NB_CHECK(H % WS == 0 && W % WS == 0, "feature map must be a multiple of the 6x6 window");
    NB_CHECK(C == 96 || C == 192, "fused window attention supports C=96 (d=16) and C=192 (d=32)");
    if (WS >= H) shift = 0;  // torchvision :151-155
    const long long nwin = (long long)B * (H / WS) * (W / WS);
    NB_CHECK(nwin > 0 && nwin < (1LL << 31), "window count out of range");
    CUtensorMap wmap;
    const cuuint64_t dims[2] = {(cuuint64_t)C, (cuuint64_t)(3 * C)};
    const cuuint64_t strides[1] = {(cuuint64_t)C * 2};
    const cuuint32_t box[2] = {32, 32};   // [32 rows][32]: one q, k or v block of a chunk
    if (encode(&wmap, wqkv, 2, dims, strides, box, 64)) return 1;
    const double T = (double)B * H * W;
    ProfScope ps(st, PC_FUSED_ATTN, T * 3.0 * C * C * 2 + T * C * 36 * 4, T * C * 2, T * C * 2);   // qkv GEMM + QK^T/PV; x in, att out
    const unsigned grid = (unsigned)((nwin + FA_WIN - 1) / FA_WIN);
    if (rec_on()) {
        char line[96];
        snprintf(line, sizeof(line), "swin_attn,%d,%d,%d,%d,%d", B, H, W, C, shift);
        rec_append(line);
    }
    const float4* bf = reinterpret_cast<const float4*>(bias_frag_f);
    if (C == 96) {
        if (ensure_dyn_smem((const void*)swin_attn_fused_kernel<96>, FaCfg<96>::SMEM)) return 1;
        swin_attn_fused_kernel<96><<<grid, FA_THREADS, FaCfg<96>::SMEM, st>>>(wmap, x, bqkv, bf, att, H, W, shift, (int)nwin);
    } else {
        if (ensure_dyn_smem((const void*)swin_attn_fused_kernel<192>, FaCfg<192>::SMEM)) return 1;
        swin_attn_fused_kernel<192><<<grid, FA_THREADS, FaCfg<192>::SMEM, st>>>(wmap, x, bqkv, bf, att, H, W, shift, (int)nwin);
    }
    NB_LAUNCHED();
    return 0;
}

}  // namespace nb200
