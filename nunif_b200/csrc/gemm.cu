// Host side of the wgmma implicit-GEMM: tensor-map construction and dispatch.
#include "gemm.h"
#include "gemm_wgmma.cuh"
#include "tmap.h"
#include <mutex>
#include <cstdlib>

namespace nb200 {

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*, CUtensorMapInterleave,
                                  CUtensorMapSwizzle, CUtensorMapL2promotion, CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode() {
    // libcuda is resolved through the runtime so the library itself has no link-time
    // dependency on the driver (it must load on a CPU-only box for the symbol checks).
    static EncodeTiledFn fn = nullptr;
    static std::once_flag once;
    std::call_once(once, [] {
        void* p = nullptr;
        cudaDriverEntryPointQueryResult q;
        if (cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &q) == cudaSuccess &&
            q == cudaDriverEntryPointSuccess)
            fn = (EncodeTiledFn)p;
    });
    return fn;
}

int encode(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
                  const cuuint32_t* box, int swizzle_bytes) {
    EncodeTiledFn fn = get_encode();
    if (!fn) return fail("cuTensorMapEncodeTiled is not available (no CUDA driver?)");
    cuuint32_t estr[5] = {1, 1, 1, 1, 1};
    CUtensorMapSwizzle sw = swizzle_bytes == 128 ? CU_TENSOR_MAP_SWIZZLE_128B
                                                 : (swizzle_bytes == 64 ? CU_TENSOR_MAP_SWIZZLE_64B : CU_TENSOR_MAP_SWIZZLE_32B);
    CUresult r = fn(m, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, (cuuint32_t)rank, const_cast<void*>(base), dims, strides_bytes, box,
                    estr, CU_TENSOR_MAP_INTERLEAVE_NONE, sw, CU_TENSOR_MAP_L2_PROMOTION_L2_256B,
                    CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
    if (r != CUDA_SUCCESS) return fail("cuTensorMapEncodeTiled failed with CUresult " + std::to_string((int)r));
    return 0;
}

template <int BN, int BK>
static int launch_t(cudaStream_t st, const GemmMaps& maps, const GemmParams& p, int m_tiles, int n_tiles) {
    using Cfg = GemmCfg<BN, BK>;
    if (ensure_dyn_smem((const void*)gemm_conv_kernel<BN, BK>, Cfg::SMEM_BYTES)) return 1;
    // programmatic dependent launch: this grid may be scheduled while the previous kernel of the stream drains (that kernel
    // executes griddepcontrol.launch_dependents); barrier set-up and tensor-map prefetch then overlap the predecessor's tail,
    // and the producer warp blocks in griddepcontrol.wait before the first load.
    cudaLaunchConfig_t cfg = {};
    cfg.gridDim = dim3((unsigned)m_tiles * n_tiles); cfg.blockDim = dim3(GEMM_THREADS); cfg.dynamicSmemBytes = Cfg::SMEM_BYTES;
    cfg.stream = st;
    cudaLaunchAttribute at[1];
    at[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
    at[0].val.programmaticStreamSerializationAllowed = 1;
    cfg.attrs = at; cfg.numAttrs = 1;
    NB_CUDA(cudaLaunchKernelEx(&cfg, gemm_conv_kernel<BN, BK>, maps, p));
    NB_LAUNCHED();
    return 0;
}

template <int BK>
static int launch_bn(int bn, cudaStream_t st, const GemmMaps& maps, const GemmParams& p, int m_tiles, int n_tiles) {
    switch (bn) {
        case 16: return launch_t<16, BK>(st, maps, p, m_tiles, n_tiles);
        case 32: return launch_t<32, BK>(st, maps, p, m_tiles, n_tiles);
        case 48: return launch_t<48, BK>(st, maps, p, m_tiles, n_tiles);
        case 64: return launch_t<64, BK>(st, maps, p, m_tiles, n_tiles);
        case 96: return launch_t<96, BK>(st, maps, p, m_tiles, n_tiles);
        case 128: return launch_t<128, BK>(st, maps, p, m_tiles, n_tiles);
    }
    return fail("unsupported BLOCK_N");
}

static int num_sms() { return device_sm_count(); }

// knobs of nb200_tune_set, read by the kernels' host code; defaults are the shipped configuration
std::atomic<int> g_tune_epoch{0};
int g_tune[16] = {0, 0, 0, /*3 force gather backward warp*/ 0, 0, 0, /*6 attention smem carveout %*/ 0,
                  /*7 SIMT stem / tail convs*/ 0, 0, /*9 CUDA-graph replay of nb200_model_forward*/ 0, 0, 0, 0, 0, 0, 0};

// 4-D NHWC view (c, x, y, b) of an fp16 tensor for the epilogue's TMA stores / residual loads
static int encode_nhwc4(CUtensorMap* m, const __half* base, int C, int X, int Y, int B, long long sx, long long sy, long long sb,
                        int cw, int tw, int th) {
    cuuint64_t dims[4] = {(cuuint64_t)C, (cuuint64_t)X, (cuuint64_t)Y, (cuuint64_t)B};
    cuuint64_t strides[3] = {(cuuint64_t)sx * 2, (cuuint64_t)sy * 2, (cuuint64_t)sb * 2};
    cuuint32_t box[4] = {(cuuint32_t)cw, (cuuint32_t)tw, (cuuint32_t)th, 1};
    return encode(m, base, 4, dims, strides, box, cw * 2);
}

int conv_gemm(cudaStream_t st, const ConvGemm& g) {
    NB_CHECK(g.A && g.Wt && g.out, "null pointer");
    NB_CHECK(g.Ci % 8 == 0, "input channel stride must be a multiple of 8");
    NB_CHECK(g.N % 16 == 0, "N must be a multiple of 16 (pad the weights)");
    GemmParams p;
    memset(&p, 0, sizeof(p));
    int ktap;          // K per tap
    cuuint64_t dims[5], strides[4];
    cuuint32_t box[5];
    const cuuint64_t e = 2;  // bytes per element
    const cuuint64_t rs = (g.a_row_stride ? (cuuint64_t)g.a_row_stride : (cuuint64_t)g.Wi * g.Ci) * e;
    const cuuint64_t is = (g.a_img_stride ? (cuuint64_t)g.a_img_stride * e : (cuuint64_t)g.Hi * rs);
    switch (g.kind) {
        case CG_LINEAR_FLAT: {
            const long long M = (long long)g.B * g.Hi * g.Wi;
            p.B = 1; p.Ho = 1; p.Wo = (int)M; p.TH = 1; p.TW = 128;
            p.taps = g.a_planes; ktap = g.Cin;
            NB_CHECK(g.a_planes >= 1 && g.a_planes <= 16, "bad plane count");
            for (int t = 0; t < p.taps; ++t) { p.tap_dy[t] = 0; p.tap_dx[t] = 0; p.tap_dyi[t] = (int8_t)t; }
            dims[0] = g.Cin; dims[1] = M; dims[2] = g.a_planes; dims[3] = 1; dims[4] = 1;
            strides[0] = g.Ci * e; strides[1] = (g.a_planes > 1 ? (cuuint64_t)g.a_plane_stride : (cuuint64_t)M * g.Ci) * e;
            strides[2] = (cuuint64_t)M * g.Ci * e * g.a_planes; strides[3] = strides[2];
            break;
        }
        case CG_LINEAR_2D:
        case CG_CONV3: {
            const int kk = g.kind == CG_CONV3 ? 3 : 1;
            const int pad = g.kind == CG_CONV3 ? g.pad : 0;
            NB_CHECK(pad == 0 || pad == 1, "conv3x3 padding must be 0 or 1");
            p.B = g.B; p.Ho = g.Hi - (kk - 1) + 2 * pad; p.Wo = g.Wi - (kk - 1) + 2 * pad; p.TH = 8; p.TW = 16;
            p.taps = kk * kk; ktap = g.Cin;
            // pad: tap coordinates start at -1; tensor-map loads zero-fill everything outside [0, Wi) x [0, Hi)
            for (int t = 0; t < p.taps; ++t) { p.tap_dy[t] = (int8_t)(t / kk - pad); p.tap_dx[t] = (int8_t)(t % kk - pad); p.tap_dyi[t] = 0; }
            dims[0] = g.Cin; dims[1] = g.Wi; dims[2] = 1; dims[3] = g.Hi; dims[4] = g.B;
            strides[0] = g.Ci * e; strides[1] = rs; strides[2] = rs;
            strides[3] = is;
            break;
        }
        case CG_TCONV3: {
            NB_CHECK(g.dil >= 1 && g.dil <= 127, "temporal dilation must be in [1, 127]");
            p.B = g.B; p.Ho = g.Hi; p.Wo = g.Wi; p.TH = 8; p.TW = 16;
            p.taps = 3; ktap = g.Cin;
            for (int t = 0; t < 3; ++t) { p.tap_dy[t] = (int8_t)((t - 1) * g.dil); p.tap_dx[t] = 0; p.tap_dyi[t] = 0; }
            dims[0] = g.Cin; dims[1] = g.Wi; dims[2] = 1; dims[3] = g.Hi; dims[4] = g.B;
            strides[0] = g.Ci * e; strides[1] = rs; strides[2] = rs;
            strides[3] = is;
            break;
        }
        case CG_DOWN2: {
            NB_CHECK(g.Hi % 2 == 0 && g.Wi % 2 == 0, "2x2 stride-2 conv needs even H and W");
            NB_CHECK(g.Cin == g.Ci, "2x2 stride-2 conv needs a dense channel dimension");
            p.B = g.B; p.Ho = g.Hi / 2; p.Wo = g.Wi / 2; p.TH = 8; p.TW = 16;
            p.taps = 2; ktap = 2 * g.Cin;
            for (int t = 0; t < 2; ++t) { p.tap_dy[t] = 0; p.tap_dx[t] = 0; p.tap_dyi[t] = t; }
            dims[0] = 2 * g.Cin; dims[1] = g.Wi / 2; dims[2] = 2; dims[3] = g.Hi / 2; dims[4] = g.B;
            strides[0] = 2 * g.Ci * e; strides[1] = rs; strides[2] = 2 * rs;
            strides[3] = is;
            break;
        }
        default: return fail("conv_gemm: unknown kind");
    }
    NB_CHECK(ktap % 32 == 0, "K per tap must be a multiple of 32");
    const int BK = (ktap % 64 == 0) ? 64 : 32;
    p.cpt = ktap / BK;
    p.tiles_x = cdiv(p.Wo, p.TW);
    p.tiles_y = cdiv(p.Ho, p.TH);
    p.N = g.N;
    p.bias = g.bias; p.act = g.act; p.out_mode = g.out_mode; p.cout = g.cout;
    p.has_res = g.res ? 1 : 0;
    p.res_before_act = g.res_before_act;
    const bool shuf = g.out_mode == OUT_PIXSHUF2;
    const bool split = g.out_mode == OUT_SPLIT;
    if (split) {
        NB_CHECK(g.cout % 16 == 0 && g.N % g.cout == 0 && g.N / g.cout <= 4, "split output: N must be 1..4 blocks of cout");
        NB_CHECK(!g.res, "split output does not take a residual");
    }
    if (shuf) {
        NB_CHECK(g.kind != CG_LINEAR_FLAT, "pixel-shuffle output needs 2-D tiling");
        NB_CHECK(g.cout % 16 == 0 && g.N == 4 * g.cout, "pixel-shuffle: N must be 4*cout, cout % 16 == 0");
    }
    NB_CHECK(g.ldo % 8 == 0 && (!g.res || g.ldr % 8 == 0), "channel strides must be multiples of 8");
    // largest BLOCK_N (<= 128: the accumulators live in registers) dividing N whose store chunk (64/32/16 columns) does not
    // straddle a pixel-shuffle group or a split plane
    int bn = 0, cw = 0;
    static const int cands[] = {128, 96, 64, 48, 32, 16};
    for (int c : cands) {
        const int w = (c % 64 == 0) ? 64 : ((c % 32 == 0) ? 32 : 16);
        if (g.N % c == 0 && (!shuf || g.cout % w == 0) && (!split || g.cout % c == 0)) { bn = c; cw = w; break; }
    }
    NB_CHECK(bn > 0, "no BLOCK_N divides N");
    if (!shuf) {
        // small-M launches (ViT tokens of a few frames, coarse DPT levels): prefer narrower tiles until the grid
        // (m-tiles x n-tiles) covers most SMs; the activation tile is then re-read from L2 by the extra n-tiles
        const long long m_tiles_est = (long long)p.tiles_x * p.tiles_y * p.B;
        static const int narrower[] = {96, 64};
        for (int c : narrower) {
            if ((long long)(g.N / bn) * m_tiles_est >= (long long)num_sms() * 3 / 4) break;
            if (c >= bn || g.N % c) continue;
            const int w = (c % 64 == 0) ? 64 : 32;
            if (split && g.cout % w) continue;
            bn = c; cw = w;
        }
    }
    p.n_tiles = g.N / bn;
    box[0] = BK; box[1] = p.TW; box[2] = 1; box[3] = p.TH; box[4] = 1;
    GemmMaps maps;
    memset(&maps, 0, sizeof(maps));
    if (encode(&maps.a, g.A, 5, dims, strides, box, BK * 2)) return 1;
    const int K = p.taps * ktap;
    cuuint64_t bdims[2] = {(cuuint64_t)K, (cuuint64_t)g.N};
    cuuint64_t bstr[1] = {(cuuint64_t)K * e};
    cuuint32_t bbox[2] = {(cuuint32_t)BK, (cuuint32_t)bn};
    if (encode(&maps.b, g.Wt, 2, bdims, bstr, bbox, BK * 2)) return 1;
    // ---- output / residual views
    if (split) {
        for (int q = 0; q < g.N / g.cout; ++q)
            if (encode_nhwc4(&maps.o[q], g.out + (size_t)q * g.split_stride, g.cout, p.Wo, p.Ho, p.B, g.ldo, (long long)p.Wo * g.ldo,
                             (long long)p.Ho * p.Wo * g.ldo, cw, p.TW, p.TH)) return 1;
    } else if (!shuf) {
        if (encode_nhwc4(&maps.o[0], g.out, g.N, p.Wo, p.Ho, p.B, g.ldo, (long long)p.Wo * g.ldo, (long long)p.Ho * p.Wo * g.ldo,
                         cw, p.TW, p.TH)) return 1;
        if (g.res) {
            const int rW = g.kind == CG_LINEAR_FLAT ? p.Wo : g.res_W, rH = g.kind == CG_LINEAR_FLAT ? 1 : g.res_H;
            p.res_cx = g.kind == CG_LINEAR_FLAT ? 0 : g.res_cx;
            p.res_cy = g.kind == CG_LINEAR_FLAT ? 0 : g.res_cy;
            if (encode_nhwc4(&maps.r[0], g.res, g.N, rW, rH, p.B, g.ldr, (long long)rW * g.ldr, (long long)rH * rW * g.ldr, cw,
                             p.TW, p.TH)) return 1;
        }
    } else {
        const int OW = 2 * p.Wo, OH = 2 * p.Ho;
        for (int q = 0; q < 4; ++q) {
            const int dy = q >> 1, dx = q & 1;
            if (encode_nhwc4(&maps.o[q], g.out + ((size_t)dy * OW + dx) * g.ldo, g.cout, p.Wo, p.Ho, p.B, 2LL * g.ldo,
                             2LL * OW * g.ldo, (long long)OH * OW * g.ldo, cw, p.TW, p.TH)) return 1;
            if (g.res) {
                // crop folded into the base: position (2y+dy+cy, 2x+dx+cx) of the residual tensor
                const int oy = dy + g.res_cy, ox = dx + g.res_cx;
                NB_CHECK(oy + 2 * (p.Ho - 1) < g.res_H && ox + 2 * (p.Wo - 1) < g.res_W, "residual tensor too small");
                if (encode_nhwc4(&maps.r[q], g.res + ((size_t)oy * g.res_W + ox) * g.ldr, g.cout, p.Wo, p.Ho, p.B, 2LL * g.ldr,
                                 2LL * g.res_W * g.ldr, (long long)g.res_H * g.res_W * g.ldr, cw, p.TW, p.TH)) return 1;
            }
        }
        p.res_cx = p.res_cy = 0;
    }
    const int m_tiles = p.tiles_x * p.tiles_y * p.B;
    const double Mrows = (double)p.B * p.Ho * p.Wo;
    // algorithmic HBM traffic: the input region once (taps re-read from L2), the residual, the output
    const double in_px = g.kind == CG_DOWN2 ? 4.0 * Mrows : ((g.kind == CG_CONV3 || g.kind == CG_TCONV3) ? (double)p.B * g.Hi * g.Wi : Mrows);
    ProfScope ps(st, PC_GEMM, 2.0 * Mrows * (double)g.N * (double)K,
                 in_px * (g.kind == CG_LINEAR_FLAT ? g.Cin * g.a_planes : g.Cin) * 2.0 + (g.res ? Mrows * g.N * 2.0 : 0.0) + (double)g.N * K * 2.0,
                 Mrows * (double)g.N * 2.0);
    return BK == 64 ? launch_bn<64>(bn, st, maps, p, m_tiles, p.n_tiles) : launch_bn<32>(bn, st, maps, p, m_tiles, p.n_tiles);
}

}  // namespace nb200

using namespace nb200;

// Low-level op exposed for unit tests and micro-benchmarks (see include/nunif_b200.h).
extern "C" int nb200_conv_gemm_f16(const void* A, int B, int Hi, int Wi, int Ci, int Cin, int kind, const void* Wt, int N,
                                   const float* bias, int act, void* out, int ldo, int out_mode, int cout,
                                   const void* res, int ldr, int res_H, int res_W, int res_cy, int res_cx,
                                   int res_before_act, void* stream) {
    ConvGemm g;
    g.A = (const __half*)A; g.B = B; g.Hi = Hi; g.Wi = Wi; g.Ci = Ci; g.Cin = Cin;
    g.kind = kind == 4 ? CG_CONV3 : kind;   // 4 = 3x3 conv with zero padding 1
    g.pad = kind == 4 ? 1 : 0;
    g.Wt = (const __half*)Wt; g.N = N; g.bias = bias; g.act = act; g.out = (__half*)out; g.ldo = ldo;
    g.out_mode = out_mode; g.cout = cout; g.res = (const __half*)res; g.ldr = ldr; g.res_H = res_H; g.res_W = res_W;
    g.res_cy = res_cy; g.res_cx = res_cx; g.res_before_act = res_before_act;
    return conv_gemm((cudaStream_t)stream, g);
}

// profiling knobs (see g_tune in this file); not part of the reference-facing API
extern "C" int nb200_tune_set(int key, int value) {
    NB_CHECK(key >= 0 && key < 16, "bad key");
    g_tune[key] = value;
    g_tune_epoch.fetch_add(1);   // models drop their captured CUDA graphs (model.cu)
    return 0;
}
