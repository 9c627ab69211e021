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

namespace nb200 {

extern int g_tune[16];  // gemm.cu (nb200_tune_set)

namespace {
constexpr int WS = 6, WTOK = 36, WPAD = 48, HEADS = 6;
// torchvision (:151-155) zeroes the shift of each axis the window covers, but the kernels take one shift for both axes: a
// shifted map with exactly one side of WS would be rolled along the wrong axes.  SwinUNet's maps are square.
constexpr const char* SHIFT_ONE_AXIS_MSG =
    "shifted window attention needs H and W both equal to the 6-token window or both larger (torchvision drops the shift per "
    "axis; these kernels shift both axes or neither)";
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
// evaluated).  BNT: key tiles per m-tile in cx.bf, 6 for the packed table in global memory, NKT for a copy in shared memory.
template <int D, int LD, bool LAST, int BNT = 6>
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
        const float4 bv = BNT == 6 ? __ldg(cx.bf + (mt * 6 + nt) * 32) : cx.bf[(mt * BNT + nt) * 32];
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
// padded key columns (>= 36) hold -1e30 so they vanish in the softmax; padded query rows hold 0.  The only definition of this
// layout: the model's loader (nb200_model_create) and the C entry points below both build the table with it.
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

// The geometry both head paths take (func: the caller, which the messages name): H and W multiples of the window, C = 96 or
// 192, and a shift on both axes or neither.  *shift is dropped where the window covers the map (torchvision :151-155).
static int check_window_geometry(const char* func, bool fused, int H, int W, int C, int* shift) {
    auto refuse = [&](const std::string& msg) { return fail(std::string(func) + ": " + msg); };
    if (H % WS != 0 || W % WS != 0) return refuse("feature map must be a multiple of the 6x6 window");
    if (C != 96 && C != 192) return refuse(std::string(fused ? "fused " : "") + "window attention supports C=96 (d=16) and C=192 (d=32)");
    if (*shift != 0 && (H == WS) != (W == WS)) return refuse(SHIFT_ONE_AXIS_MSG);
    if (WS >= H) *shift = 0;
    return 0;
}

int window_attention(cudaStream_t st, const __half* qkv, const float* bias_frag_f, __half* out, int B, int H, int W, int C,
                     int shift, size_t plane) {
    const float4* bias_table = reinterpret_cast<const float4*>(bias_frag_f);
    if (check_window_geometry(__func__, false, H, W, C, &shift)) return 1;
    dim3 grid((H / WS) * (W / WS), B);
    ProfScope ps(st, PC_ATTN, (double)B * H * W * C * 4 * 2, (double)B * H * W * C * 3 * 2, (double)B * H * W * C * 2);  // q,k,v in; out
    // shared-memory carveout: just enough for the 4 resident CTAs, the rest stays L1 (the per-head bias fragments,
    // 55 KB per layer, are re-read by every window and should hit there).  g_tune[6] overrides the percentage.
    if (C == 96) {
        const int want = g_tune[6] > 0 ? g_tune[6] : 72;   // 6 CTAs x 23.6 KB
        if (ensure_dyn_smem((const void*)window_attention_mma_kernel<16>, attn_smem_bytes<16>(), want)) return 1;
        window_attention_mma_kernel<16><<<grid, 192, attn_smem_bytes<16>(), st>>>(qkv, bias_table, out, H, W, shift, plane);
    } else {
        const int want = g_tune[6] > 0 ? g_tune[6] : 86;
        if (ensure_dyn_smem((const void*)window_attention_mma_kernel<32>, attn_smem_bytes<32>(), want)) return 1;
        window_attention_mma_kernel<32><<<grid, 192, attn_smem_bytes<32>(), st>>>(qkv, bias_table, out, H, W, shift, plane);
    }
    NB_LAUNCHED();
    return 0;
}


// ---------------------------------------------------------------------------------------------
// Fused block head: att = window_attention_core(x . Wqkv^T + bqkv), q/k/v never leave shared memory.
// The unit of work is a tile of 3 windows = 108 tokens (+20 zero rows) = the 128 rows of two wgmma warpgroups.
// q|k|v is computed head-major in C/32 chunks of 96 columns: chunk c holds columns [32c, 32c+32) of q, of k and of v, i.e.
// head c (d = 32) or heads 2c, 2c+1 (d = 16), so it is complete input of the attention core for those heads.
//
// Persistent and warp-specialised: one CTA per SM takes tiles blockIdx.x + k gridDim.x, and its three roles run concurrently
// through double-buffered shared memory.  20 warps: 5 per SM sub-partition share its 64 KB register file, 96 registers each
// (21 warps would put 6 on one sub-partition and cap every thread at 80).
//   warp 8      : producer (one lane).  Streams Wqkv through a 4-stage ring, tile after tile.  A stage is 3 K-blocks of one
//                 chunk; per K-block the rows 32c, C + 32c and 2C + 32c of chunk c as three [32][32] boxes (64B swizzle)
//                 stacked into one [96][32] operand.
//   warps 0-7   : two MMA warpgroups (64 rows each).  Per chunk the wgmma K loop into acc[48], then bias (bqkv, staged in
//                 shared memory once per CTA) + fp16 into chunk buffer g & 1 (g counts chunks across tiles) as per-window q/k/v
//                 tiles.
//   warps 9-19  : 11 attention warps.  Items (window, head, m-tile) run in one sequence over all of the CTA's tiles,
//                 chunk-major and m-tile-major within a chunk (54 per tile at both C); item n goes to attention warp n mod 11
//                 and is attn_mtile (the same code as window_attention_mma_kernel) plus the un-rolled store of its output rows.
//                 A warp may start on chunk g + 1 while others finish chunk g.  The attention warps also gather the NEXT tile's
//                 rolled window rows into the other A buffer (16-byte cp.async, zeros for missing windows; rows >= 108 are
//                 zeroed once at start-up): each warp issues its share at its first item of tile k and signals it at its
//                 second.  They wait on q|k|v most of the time, and a single producer warp issuing both the weights and the
//                 gather could not keep the MMA warps fed.
//
// Barriers (k: the CTA's tile counter, g: its chunk counter, q: its weight-stage counter; the parity of use u is u & 1):
//   barrier        count            arrivals                                             waiters
//   full[s]        1 (+ tx bytes)   producer expect_tx; TMA completes it                MMA warps, stage q: (q / 4) & 1
//   empty[s]       2                thread 0 of each MMA warpgroup once the stage's      producer before stage q:
//                                   wgmma group retired                                  ((q / 4) & 1) ^ 1
//   afull[b]       32 x 11          every attention lane after its cp.async.wait_all     MMA warps, tile k (b = k & 1):
//                                   and fence.proxy.async (wgmma reads the async proxy)  (k / 2) & 1
//   aempty[b]      2                thread 0 of each MMA warpgroup after the tile's      attention warps before gathering
//                                   last wgmma retired                                   tile k into b: ((k / 2) & 1) ^ 1
//   cfull[b]       8                lane 0 of each MMA warp after its epilogue stores   attention warps, chunk g (b = g & 1):
//                                                                                        (g / 2) & 1
//   cempty[b]      items per chunk  lane 0 of the warp that ran an item of the chunk     MMA warps before the epilogue of
//                  (9 or 18)        (items of windows past nwin arrive too)              chunk g: ((g / 2) & 1) ^ 1
// A parity wait is exact only if the waiter is at most one phase ahead.  The producer and the MMA warps wait on every phase
// of their barriers, and every attention warp gathers (waits on aempty) once per tile.  An attention warp waits only on the
// chunks of its own items, which are 11 apart in the sequence, so at most 2 chunks apart: when it waits for chunk g, either
// it waited for chunk g - 2 itself or it waited for chunk g - 1, which the MMA warps filled after chunk g - 2; and chunk
// g + 2 cannot be filled before its own item of chunk g is done.  No wait can deadlock: a warp's first two items of tile k
// lie in chunks the MMA warps fill from tile k alone, and at its first one the MMA warps have finished reading tile k - 1.
// The window tables are not per tile: the region pattern of a window (the shift mask) depends only on whether it is in the
// last window row and/or column, so the 4 patterns are built once; the token of a row is recomputed from the window index
// where it is needed (the gather, the output stores).  So nothing per tile outlives its A buffer.
// ---------------------------------------------------------------------------------------------
constexpr int FA_ROWS = 128, FA_WIN = 3, FA_SLOT = 96 * 64, FA_KPS = 3, FA_STAGES = 4;
constexpr int FA_MMA_THREADS = GEMM_CONSUMER_THREADS, FA_PRODUCER_WARP = FA_MMA_THREADS / 32, FA_ATTN_WARPS = 11;
constexpr int FA_THREADS = FA_MMA_THREADS + 32 + 32 * FA_ATTN_WARPS;   // 640
constexpr int FA_LD = 32 + 8;   // chunk tile row: 80 B = 20 words, so fragment loads and ldmatrix rows are conflict-free
constexpr int FA_CHUNK_BYTES = FA_WIN * 3 * WTOK * FA_LD * 2;
constexpr int FA_STAGE = FA_KPS * FA_SLOT;   // a ring stage: FA_KPS K-blocks of one chunk's [96][32] weight operand

template <int C>
struct FaCfg {
    static constexpr int X_BYTES = FA_ROWS * C * 2;
    // The attention warps read the relative-position-bias fragments of every item.  Where they fit (C = 96) the NKT key tiles
    // of each (head, m-tile) are copied to shared memory once per CTA; at C = 192 (4.3 KB left) they are read from L1/L2.
    static constexpr bool SBF = C == 96;
    static constexpr int SBF_BYTES = SBF ? HEADS * 3 * NKT * 32 * 16 : 0;
    static constexpr int SBF_OFF = 2 * X_BYTES + FA_STAGES * FA_STAGE + 2 * FA_CHUNK_BYTES + 4 * WPAD * 4 + (2 * FA_STAGES + 8) * 8 +
                                   3 * C * 4;
    static constexpr int SMEM = SBF_OFF + SBF_BYTES + 1024;
    static_assert(SBF_OFF % 16 == 0, "float4 bias fragments");
    static_assert(SMEM <= 232448, "over the 227 KB opt-in shared memory of an H100 CTA");
};

// token of row t of window (b, wy, wx) (torch.roll(-shift) :166-167); shift < H, W
__device__ __forceinline__ int fa_token(int b, int wy, int wx, int t, int H, int W, int shift) {
    int y = wy * WS + t / WS + shift, xx = wx * WS + t % WS + shift;
    if (y >= H) y -= H;
    if (xx >= W) xx -= W;
    return (b * H + y) * W + xx;
}

template <int C>
__global__ void __launch_bounds__(FA_THREADS, 1) swin_attn_fused_kernel(const __grid_constant__ CUtensorMap wmap,
                                                                        const __half* __restrict__ x, const float* __restrict__ bqkv,
                                                                        const float4* __restrict__ bias_frag, __half* __restrict__ out,
                                                                        int H, int W, int shift, int nwin) {
    using Cfg = FaCfg<C>;
    constexpr int D = C / HEADS, KB = C / 32, NCH = C / 32, HPC = 32 / D;   // HPC: heads per chunk
    constexpr int IPC = 3 * FA_WIN * HPC, IPT = NCH * IPC;                  // attention items per chunk / per tile
    constexpr int SPC = KB / FA_KPS;                                        // ring stages per chunk
    constexpr int VPR = C / 8;                                              // 16-byte pieces per row
    static_assert(KB % FA_KPS == 0, "a ring stage holds FA_KPS K-blocks of one chunk");
    static_assert(FA_WIN == 3, "the gather selects among 3 windows");
    extern __shared__ uint8_t smem_dyn[];
    // aligned by an offset from smem_dyn, not by integer arithmetic on its address: the compiler then knows every pointer
    // below is a shared-memory one and emits LDS/STS instead of generic loads and stores
    uint8_t* smem = smem_dyn + ((1024u - (smem_u32(smem_dyn) & 1023u)) & 1023u);
    uint8_t* sx = smem;                                                      // [2][128][C] A tiles
    uint8_t* ring = smem + 2 * Cfg::X_BYTES;
    __half* schunk = reinterpret_cast<__half*>(ring + FA_STAGES * FA_STAGE);  // [2][window][q|k|v][WTOK][FA_LD]
    int* sreg = reinterpret_cast<int*>(reinterpret_cast<uint8_t*>(schunk) + 2 * FA_CHUNK_BYTES);  // [last row][last col][WPAD]
    uint64_t* full = reinterpret_cast<uint64_t*>(sreg + 4 * WPAD);
    uint64_t* empty = full + FA_STAGES;
    uint64_t* afull = empty + FA_STAGES;
    uint64_t* aempty = afull + 2;
    uint64_t* cfull = aempty + 2;
    uint64_t* cempty = cfull + 2;
    float* sbias = reinterpret_cast<float*>(cempty + 2);   // [3C] bqkv
    float4* sbf = reinterpret_cast<float4*>(smem + Cfg::SBF_OFF);   // [head][m-tile][NKT][32] bias fragments (Cfg::SBF)
    const int tid = threadIdx.x, warp = tid >> 5, lane = tid & 31;
    const int nww = W / WS, nwy = H / WS;
    const int ntiles = (nwin + FA_WIN - 1) / FA_WIN;
    const int ntl = (ntiles - (int)blockIdx.x + (int)gridDim.x - 1) / (int)gridDim.x;   // this CTA's tiles (>= 1)

    if (tid < 4 * WPAD) {
        // region of token t (:193-209) in a window of the last window row (p & 2) and/or column (p & 1); only read when
        // shift > 0 and the window is in one of them
        const int p = tid / WPAD, t = tid % WPAD;
        int reg = -1;
        if (t < WTOK) {
            const int hr = (p & 2) ? (t / WS < WS - shift ? 1 : 2) : 0;
            const int wr = (p & 1) ? (t % WS < WS - shift ? 1 : 2) : 0;
            reg = hr * 3 + wr;
        }
        sreg[tid] = reg;
    }
    for (int i = tid; i < 3 * C; i += FA_THREADS) sbias[i] = bqkv[i];
    if (Cfg::SBF)   // from the packed [head][m-tile][6][32] table
        for (int i = tid; i < HEADS * 3 * NKT * 32; i += FA_THREADS)
            sbf[i] = __ldg(bias_frag + ((i >> 5) / NKT * 6 + (i >> 5) % NKT) * 32 + (i & 31));
    // rows 108..127 of both A tiles are zero for good
    for (int i = tid; i < 2 * (FA_ROWS - FA_WIN * WTOK) * VPR; i += FA_THREADS) {
        const int bsel = i / ((FA_ROWS - FA_WIN * WTOK) * VPR), j = i % ((FA_ROWS - FA_WIN * WTOK) * VPR);
        const int r = FA_WIN * WTOK + j / VPR, u = j % VPR;
        *reinterpret_cast<uint4*>(sx + bsel * Cfg::X_BYTES + (u >> 2) * (FA_ROWS * 64) + stage_off<32>(r, u & 3)) =
            make_uint4(0u, 0u, 0u, 0u);
    }
    if (tid == FA_MMA_THREADS) {
        tma_prefetch_desc(&wmap);
        for (int s = 0; s < FA_STAGES; ++s) {
            mbar_init(&full[s], 1);
            mbar_init(&empty[s], 2);   // one arrival per MMA warpgroup
        }
        for (int b = 0; b < 2; ++b) {
            mbar_init(&afull[b], 32 * FA_ATTN_WARPS);
            mbar_init(&aempty[b], 2);
            mbar_init(&cfull[b], FA_MMA_THREADS / 32);
            mbar_init(&cempty[b], IPC);
        }
        fence_barrier_init();
    }
    fence_async_smem();   // the zero rows (generic-proxy writes) -> visible to wgmma
    __syncthreads();
    // the block tail (swin_block.cu, a PDL launch) may start its prologue and weight loads once every CTA of this grid is resident
    if (tid == 0) NB_PDL_TRIGGER();

    if (warp == FA_PRODUCER_WARP) {
        // ===================== producer: the weight ring, tile after tile =====================
        if (elect_one()) {
            int q = 0;
#pragma unroll 1
            for (int k = 0; k < ntl; ++k) {
#pragma unroll 1
                for (int i = 0; i < NCH * SPC; ++i, ++q) {
                    const int s = q % FA_STAGES, c = i / SPC, kb0 = (i % SPC) * FA_KPS;
                    mbar_wait(&empty[s], ((q / FA_STAGES) & 1) ^ 1);
                    mbar_expect_tx(&full[s], FA_STAGE);
                    // 32-row boxes at 2 KB offsets: the 64B swizzle repeats every 512 B, so the stack is laid out as one 96-row box
#pragma unroll
                    for (int kk = 0; kk < FA_KPS; ++kk)
#pragma unroll
                        for (int m = 0; m < 3; ++m)
                            tma_load_2d(&wmap, &full[s], ring + s * FA_STAGE + kk * FA_SLOT + m * 32 * 64, (kb0 + kk) * 32, m * C + 32 * c);
                }
            }
        }
        return;
    }

    const float scale = ((D == 16) ? 0.25f : 0.17677669529663687f) * 1.4426950408889634f;  // (C//heads)**-0.5 (:187) * log2(e)
    const int g = lane >> 2, t4 = lane & 3;
    if (warp > FA_PRODUCER_WARP) {
        // ===================== attention: item n of the CTA's sequence on warp 9 + n mod 11 =====================
        const int aw = warp - FA_PRODUCER_WARP - 1;
        // this warp's share of the gather of tile `tile` into A tile sa: row r = window r/36, token r%36; 16-byte cp.async
        auto gather = [&](int tile, uint8_t* sa) {
            int wb[FA_WIN], wwy[FA_WIN], wwx[FA_WIN];   // (image, window row, window column) of the tile's windows; wb < 0: none
#pragma unroll
            for (int w = 0; w < FA_WIN; ++w) {
                const int gw = tile * FA_WIN + w, b = gw / (nww * nwy), rw = gw - b * (nww * nwy);
                wb[w] = gw < nwin ? b : -1;
                wwy[w] = rw / nww;
                wwx[w] = rw - wwy[w] * nww;
            }
            for (int i = aw * 32 + lane; i < FA_WIN * WTOK * VPR; i += 32 * FA_ATTN_WARPS) {
                const int r = i / VPR, u = i % VPR, w = r / WTOK;
                const int b = w == 0 ? wb[0] : (w == 1 ? wb[1] : wb[2]);
                const int wy = w == 0 ? wwy[0] : (w == 1 ? wwy[1] : wwy[2]), wx = w == 0 ? wwx[0] : (w == 1 ? wwx[1] : wwx[2]);
                uint8_t* dst = sa + (u >> 2) * (FA_ROWS * 64) + stage_off<32>(r, u & 3);
                if (b >= 0) cp_async16(dst, x + (size_t)fa_token(b, wy, wx, r - w * WTOK, H, W, shift) * C + u * 8);
                else *reinterpret_cast<uint4*>(dst) = make_uint4(0u, 0u, 0u, 0u);
            }
            cp_async_commit();
        };
        // the A tile is read by wgmma (the async proxy): every lane fences its own writes before it arrives
        auto gathered = [&](int kt) {
            cp_async_wait<0>();
            fence_async_smem();
            mbar_arrive(&afull[kt & 1]);
        };
        gather(blockIdx.x, sx);
        gathered(0);
        int kcur = -1, nth = 0;   // nth: this warp's items so far in tile kcur
#pragma unroll 1
        for (int n = aw; n < ntl * IPT; n += FA_ATTN_WARPS) {
            const int gc = n / IPC, item = n - gc * IPC, c = gc % NCH;   // gc: chunk counter, c: chunk of the tile
            const int kt = n / IPT, tile = blockIdx.x + kt * gridDim.x;
            mbar_wait(&cfull[gc & 1], (gc >> 1) & 1);
            if (kt != kcur) {
                kcur = kt;
                nth = 0;
            }
            // tile kt + 1 is gathered at this warp's first item of tile kt (chunk gc of tile kt is filled, so the MMA warps
            // have released A buffer (kt + 1) & 1, tile kt - 1) and signalled at its second (every warp has >= 4 items per
            // tile, both in the first 3 chunks, which the MMA warps fill without tile kt + 1)
            if (kt + 1 < ntl && nth == 0) {
                mbar_wait(&aempty[(kt + 1) & 1], (((kt + 1) >> 1) & 1) ^ 1);
                gather(tile + gridDim.x, sx + ((kt + 1) & 1) * Cfg::X_BYTES);
            }
            if (kt + 1 < ntl && nth == 1) gathered(kt + 1);
            ++nth;
            // m-tile-major within the chunk, so that the cheap 4-row tiles come last
            const int mt = item / (FA_WIN * HPC), pr = item - mt * (FA_WIN * HPC), w = pr / HPC, hh = pr - w * HPC;
            const int gw = tile * FA_WIN + w;
            if (gw < nwin) {
                const int b = gw / (nww * nwy), r = gw % (nww * nwy), wy = r / nww, wx = r % nww, head = c * HPC + hh;
                const bool lrow = wy == nwy - 1, lcol = wx == nww - 1;
                __half* sq = schunk + (gc & 1) * (FA_CHUNK_BYTES / 2) + w * 3 * WTOK * FA_LD;
                __half* sk = sq + WTOK * FA_LD;
                __half* sv = sk + WTOK * FA_LD;
                AttnCtx<D> cx;
                cx.sq = sq; cx.sreg = sreg + (2 * lrow + lcol) * WPAD;
                cx.bf = Cfg::SBF ? sbf + head * (3 * NKT * 32) + lane : bias_frag + (size_t)head * (3 * 6 * 32) + lane;
                cx.hc = hh * D; cx.g = g; cx.t4 = t4; cx.scale = scale;
                cx.boundary = shift > 0 && (lrow || lcol);   // only these windows mix mask regions
#pragma unroll
                for (int nt = 0; nt < NKT; ++nt) cx.kbase[nt] = sk + min(nt * 8 + g, WTOK - 1) * FA_LD + cx.hc + 2 * t4;
                cx.vbase[0] = sv + (lane & 15) * FA_LD + cx.hc;
                cx.vbase[1] = sv + (16 + (lane & 15)) * FA_LD + cx.hc;
                cx.vbase[2] = sv + min(32 + (lane & 7), WTOK - 1) * FA_LD + cx.hc;
                constexpr int BNT = Cfg::SBF ? NKT : 6;
                if (mt < 2) attn_mtile<D, FA_LD, false, BNT>(cx, mt);
                else attn_mtile<D, FA_LD, true, BNT>(cx, 2);
                // the m-tile's output rows (staged over its own q rows by this warp) -> HBM, D columns = D/8 16-byte pieces per row
                __syncwarp();
                const int nrow = mt < 2 ? 16 : WTOK - 32;
                for (int e = lane; e < nrow * (D / 8); e += 32) {
                    const int tk = 16 * mt + e / (D / 8), u = e % (D / 8);
                    *reinterpret_cast<uint4*>(out + (size_t)fa_token(b, wy, wx, tk, H, W, shift) * C + head * D + u * 8) =
                        *reinterpret_cast<const uint4*>(sq + tk * FA_LD + cx.hc + u * 8);
                }
            }
            __syncwarp();
            if (lane == 0) mbar_arrive(&cempty[gc & 1]);
        }
        return;
    }

    // ===================== MMA warps: q | k | v = x Wqkv^T + b, chunk by chunk =====================
    const int wg = tid >> 7, t = tid & 127;
    const int row0 = wg * 64 + (t >> 5) * 16 + ((t & 31) >> 2);
    const int cq = 2 * (t & 3);
    int q = 0, gc = 0;
#pragma unroll 1
    for (int k = 0; k < ntl; ++k) {
        mbar_wait(&afull[k & 1], (k >> 1) & 1);
        const uint32_t a_base = smem_u32(sx + (k & 1) * Cfg::X_BYTES) + wg * 64 * 64;
#pragma unroll 1
        for (int c = 0; c < NCH; ++c, ++gc) {
            float acc[48];
#pragma unroll
            for (int j = 0; j < 48; ++j) acc[j] = 0.f;
#pragma unroll 1
            for (int j = 0; j < SPC; ++j, ++q) {
                const int s = q % FA_STAGES;
                mbar_wait(&full[s], (q / FA_STAGES) & 1);
                wgmma_fence();
#pragma unroll
                for (int kk = 0; kk < FA_KPS; ++kk) {
                    const uint32_t a = a_base + (j * FA_KPS + kk) * (FA_ROWS * 64), bb = smem_u32(ring + s * FA_STAGE + kk * FA_SLOT);
                    wgmma_f16<96>(acc, make_kmajor_desc<64>(a), make_kmajor_desc<64>(bb), 1u);
                    wgmma_f16<96>(acc, make_kmajor_desc<64>(a + 32), make_kmajor_desc<64>(bb + 32), 1u);
                }
                wgmma_commit();
                // keep one group in flight: the stage read by the previous group is released once that group retired
                wgmma_wait<1>();
                if (j > 0 && t == 0) mbar_arrive(&empty[(q - 1) % FA_STAGES]);
            }
            wgmma_wait<0>();
            if (t == 0) {
                mbar_arrive(&empty[(q - 1) % FA_STAGES]);
                if (c == NCH - 1) mbar_arrive(&aempty[k & 1]);   // the tile's last wgmma has read A
            }
            wgmma_fence_operands(acc);
            mbar_wait(&cempty[gc & 1], ((gc >> 1) & 1) ^ 1);   // every item of chunk gc - 2 is done with the buffer
            __half* sqkv = schunk + (gc & 1) * (FA_CHUNK_BYTES / 2);
#pragma unroll
            for (int j = 0; j < 12; ++j) {
                const int m = j >> 2, col = 8 * (j & 3) + cq;   // q|k|v, column within the chunk
                const float2 bq = *reinterpret_cast<const float2*>(sbias + m * C + 32 * c + col);
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
            // one arrival per warp: __syncwarp orders the other lanes' stores before lane 0's (release) arrive; 256 arrivals on
            // one barrier cost about a microsecond per chunk
            __syncwarp();
            if (lane == 0) mbar_arrive(&cfull[gc & 1]);
        }
    }
}

int swin_attn_fused(cudaStream_t st, const __half* x, const __half* wqkv, const float* bqkv, const float* bias_frag_f, __half* att,
                    int B, int H, int W, int C, int shift) {
    NB_CHECK(x && wqkv && bqkv && bias_frag_f && att, "null pointer");
    if (check_window_geometry(__func__, true, H, W, C, &shift)) return 1;
    const long long nwin = (long long)B * (H / WS) * (W / WS);
    NB_CHECK(nwin > 0 && nwin < (1LL << 31), "window count out of range");
    CUtensorMap wmap;
    const cuuint64_t dims[2] = {(cuuint64_t)C, (cuuint64_t)(3 * C)};
    const cuuint64_t strides[1] = {(cuuint64_t)C * 2};
    const cuuint32_t box[2] = {32, 32};   // [32 rows][32]: one q, k or v block of a chunk
    if (encode(&wmap, wqkv, 2, dims, strides, box, 64)) return 1;
    const double T = (double)B * H * W;
    ProfScope ps(st, PC_FUSED_ATTN, T * 3.0 * C * C * 2 + T * C * 36 * 4, T * C * 2, T * C * 2);   // qkv GEMM + QK^T/PV; x in, att out
    // persistent: one CTA per SM, each taking every gridDim.x-th tile (g_tune[11] > 0 caps the grid, for tests; a tile's result
    // does not depend on its CTA)
    const long long ntiles = (nwin + FA_WIN - 1) / FA_WIN;
    long long grid = std::min<long long>(ntiles, device_sm_count());
    if (g_tune[11] > 0) grid = std::min<long long>(grid, g_tune[11]);
    if (rec_on()) rec_launch("swin_attn", {{"B", B}, {"H", H}, {"W", W}, {"C", C}, {"shift", shift}});
    const float4* bf = reinterpret_cast<const float4*>(bias_frag_f);
    if (C == 96) {
        if (ensure_dyn_smem((const void*)swin_attn_fused_kernel<96>, FaCfg<96>::SMEM)) return 1;
        swin_attn_fused_kernel<96><<<(unsigned)grid, FA_THREADS, FaCfg<96>::SMEM, st>>>(wmap, x, bqkv, bf, att, H, W, shift, (int)nwin);
    } else {
        if (ensure_dyn_smem((const void*)swin_attn_fused_kernel<192>, FaCfg<192>::SMEM)) return 1;
        swin_attn_fused_kernel<192><<<(unsigned)grid, FA_THREADS, FaCfg<192>::SMEM, st>>>(wmap, x, bqkv, bf, att, H, W, shift, (int)nwin);
    }
    NB_LAUNCHED();
    return 0;
}

// The C entry points take the raw [121][6] table and expand it into a stream-ordered temporary for the call
template <typename F>
static int with_bias_frag(void* stream, const float* table, F call) {
    cudaStream_t st = (cudaStream_t)stream;
    float* frag = nullptr;
    NB_CUDA(cudaMallocAsync((void**)&frag, BIAS_FRAG_FLOATS * sizeof(float), st));
    int rc = build_bias_frag(st, table, frag);
    if (!rc) rc = call(st, frag);
    cudaFreeAsync(frag, st);
    return rc;
}

}  // namespace nb200

using namespace nb200;

extern "C" int nb200_window_attention_f16(const void* qkv, const float* bias_table, void* out, int B, int H, int W, int C,
                                          int heads, int shift, void* stream) {
    NB_CHECK(qkv && bias_table && out, "null pointer");
    NB_CHECK(heads == 6, "only 6 heads are supported");
    return with_bias_frag(stream, bias_table, [&](cudaStream_t st, const float* frag) {
        return window_attention(st, (const __half*)qkv, frag, (__half*)out, B, H, W, C, shift, (size_t)B * H * W * C);
    });
}

extern "C" int nb200_swin_attn_fused_f16(const void* x, const void* wqkv, const float* bqkv, const float* bias_table, void* att,
                                         int B, int H, int W, int C, int shift, void* stream) {
    NB_CHECK(bias_table, "null pointer");
    return with_bias_frag(stream, bias_table, [&](cudaStream_t st, const float* frag) {
        return swin_attn_fused(st, (const __half*)x, (const __half*)wqkv, bqkv, frag, (__half*)att, B, H, W, C, shift);
    });
}
