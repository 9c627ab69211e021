// Model containers: weight packing from the reference's state_dict keys and the
// forward passes of SwinUNet (swin_unet.py:119-199), CUNet/UpCUNet (cunet.py:10-203) and UpConv7/VGG7
// (upconv_7.py, vgg_7.py) expressed as sequences of the sm_90a kernels.  Also the whole-image tiled render.
#include "common.cuh"
#include "gemm.h"
#include "gemm_wgmma.cuh"
#include "swin_kernels.h"
#include "cunet_kernels.h"
#include "legacy_kernels.h"
#include "depth_kernels.h"
#include "rowflow_kernels.h"
#include "depth_aa_kernels.h"
#include "mlbw_kernels.h"
#include "zoe_kernels.h"
#include "inpaint_kernels.h"
#include "window_mha.h"
#include "sod_kernels.h"
#include "transnet_kernels.h"
#include "../../include/nunif_b200.h"
#include <map>
#include <vector>
#include <string>
#include <cstring>
#include <cmath>
#include <memory>
#include <tuple>
#include <algorithm>

namespace nb200 {

extern int g_tune[16];                 // gemm.cu (nb200_tune_set)
extern std::atomic<int> g_tune_epoch;  // gemm.cu: bumped by every nb200_tune_set (captured graphs bake the knobs in)

// ---------------------------------------------------------------------------------------------
// weight packing
// ---------------------------------------------------------------------------------------------
struct HostTensor {
    const float* data;
    int64_t numel;
    bool used;
};

struct Packer {
    std::map<std::string, HostTensor> src;
    std::vector<uint8_t> blob;
    std::string err;

    const float* get(const std::string& name, int64_t numel) {
        auto it = src.find(name);
        if (it == src.end()) {
            if (err.empty()) err = "missing key in state_dict: " + name;
            return nullptr;
        }
        if (it->second.numel != numel) {
            if (err.empty())
                err = "size mismatch for " + name + ": expected " + std::to_string(numel) + " elements, got " +
                      std::to_string(it->second.numel);
            return nullptr;
        }
        it->second.used = true;
        return it->second.data;
    }
    void mark(const std::string& name) {
        auto it = src.find(name);
        if (it != src.end()) it->second.used = true;
    }
    size_t reserve(size_t bytes) {
        size_t off = (blob.size() + 255) & ~(size_t)255;
        blob.resize(off + bytes, 0);
        return off;
    }
    size_t add_f16(const std::vector<float>& v) {
        size_t off = reserve(v.size() * 2);
        __half* d = reinterpret_cast<__half*>(blob.data() + off);
        for (size_t i = 0; i < v.size(); ++i) d[i] = __float2half_rn(v[i]);
        return off;
    }
    size_t add_f32(const std::vector<float>& v) {
        size_t off = reserve(v.size() * 4);
        memcpy(blob.data() + off, v.data(), v.size() * 4);
        return off;
    }
};

struct Lin {  // a packed GEMM operand: Wt [N][K] fp16 + bias [N] fp32
    size_t w = 0, b = 0;
    int N = 0, K = 0;
};

// Linear: weight [N][K]
static Lin pack_linear(Packer& pk, const std::string& name, int N, int K, int n_pad = 0) {
    Lin l;
    l.N = n_pad ? n_pad : N;
    l.K = K;
    const float* w = pk.get(name + ".weight", (int64_t)N * K);
    const float* b = pk.get(name + ".bias", N);
    if (!w || !b) return l;
    std::vector<float> wv((size_t)l.N * K, 0.f), bv(l.N, 0.f);
    memcpy(wv.data(), w, (size_t)N * K * 4);
    memcpy(bv.data(), b, (size_t)N * 4);
    l.w = pk.add_f16(wv);
    l.b = pk.add_f32(bv);
    return l;
}
// Linear followed by pixel_shuffle(2): rows reordered so n = (dy*2+dx)*cout + co  (F.pixel_shuffle: c*4 + dy*2 + dx)
// With `skip`, the Linear [cout][Ks] of the skip tensor that is added to the result is appended to every row (the GEMM's
// second A operand, ConvGemm::A2): row n = [up row | skip row co], K + Ks columns, bias = both biases summed in fp32.
static Lin pack_linear_pixshuf2(Packer& pk, const std::string& name, int cout, int K, const std::string& skip = "", int Ks = 0) {
    Lin l;
    l.N = 4 * cout;
    l.K = K + Ks;
    const float* w = pk.get(name + ".weight", (int64_t)4 * cout * K);
    const float* b = pk.get(name + ".bias", 4 * cout);
    const float* ws = Ks ? pk.get(skip + ".weight", (int64_t)cout * Ks) : nullptr;
    const float* bs = Ks ? pk.get(skip + ".bias", cout) : nullptr;
    if (!w || !b || (Ks && (!ws || !bs))) return l;
    std::vector<float> wv((size_t)l.N * l.K), bv(l.N);
    for (int co = 0; co < cout; ++co)
        for (int g = 0; g < 4; ++g) {
            float* row = &wv[((size_t)g * cout + co) * l.K];
            memcpy(row, &w[((size_t)co * 4 + g) * K], (size_t)K * 4);
            if (Ks) memcpy(row + K, &ws[(size_t)co * Ks], (size_t)Ks * 4);
            bv[g * cout + co] = b[co * 4 + g] + (Ks ? bs[co] : 0.f);
        }
    l.w = pk.add_f16(wv);
    l.b = pk.add_f32(bv);
    return l;
}
// Conv2d weight [Cout][Cin][kh][kw] -> [Cout][kh][kw][cin_pad]
static Lin pack_conv(Packer& pk, const std::string& name, int cout, int cin, int kh, int kw, int cin_pad = 0, int cout_pad = 0) {
    Lin l;
    if (!cin_pad) cin_pad = cin;
    l.N = cout_pad ? cout_pad : cout;
    l.K = kh * kw * cin_pad;
    const float* w = pk.get(name + ".weight", (int64_t)cout * cin * kh * kw);
    const float* b = pk.get(name + ".bias", cout);
    if (!w || !b) return l;
    std::vector<float> wv((size_t)l.N * l.K, 0.f), bv(l.N, 0.f);
    for (int co = 0; co < cout; ++co)
        for (int ci = 0; ci < cin; ++ci)
            for (int y = 0; y < kh; ++y)
                for (int x = 0; x < kw; ++x)
                    wv[(size_t)co * l.K + ((size_t)y * kw + x) * cin_pad + ci] = w[(((size_t)co * cin + ci) * kh + y) * kw + x];
    memcpy(bv.data(), b, (size_t)cout * 4);
    l.w = pk.add_f16(wv);
    l.b = pk.add_f32(bv);
    return l;
}
// ConvTranspose2d(k=2, s=2) weight [Cin][Cout][2][2] -> rows n = (dy*2+dx)*cout + co, K = cin
static Lin pack_convT2(Packer& pk, const std::string& name, int cin, int cout) {
    Lin l;
    l.N = 4 * cout;
    l.K = cin;
    const float* w = pk.get(name + ".weight", (int64_t)cin * cout * 4);
    const float* b = pk.get(name + ".bias", cout);
    if (!w || !b) return l;
    std::vector<float> wv((size_t)l.N * cin), bv(l.N);
    for (int g = 0; g < 4; ++g)
        for (int co = 0; co < cout; ++co) {
            for (int ci = 0; ci < cin; ++ci) wv[((size_t)g * cout + co) * cin + ci] = w[((size_t)ci * cout + co) * 4 + g];
            bv[g * cout + co] = b[co];
        }
    l.w = pk.add_f16(wv);
    l.b = pk.add_f32(bv);
    return l;
}
// first 3x3 conv from 3 channels: Conv2d weight [cout][3][3][3] and bias [cout] -> wv = fp32 [27][cout_pad] with
// k = (ky*3+kx)*3 + ci, then the mma.sync B fragments; bv = bias [cout_pad] (both zero padded)
static void pack_stem_w(const float* w, const float* b, int cout, int cout_pad, std::vector<float>& wv, std::vector<float>& bv) {
    wv.assign((size_t)27 * cout_pad, 0.f);
    bv.assign(cout_pad, 0.f);
    for (int co = 0; co < cout; ++co)
        for (int ci = 0; ci < 3; ++ci)
            for (int k = 0; k < 9; ++k) {
                // the stem reads fp16 inputs and the reference runs this conv in fp16 with fp32 accumulate:
                // keep the weights at fp16 precision
                wv[(size_t)(k * 3 + ci) * cout_pad + co] = round_f16(w[((size_t)co * 3 + ci) * 9 + k]);
            }
    memcpy(bv.data(), b, (size_t)cout * 4);
    // ... followed by the same weights as fp16 mma.sync B fragments for stem_conv_mma_kernel:
    // [ks (3)][nt (cout_pad/8)][n (8)][k (16)] with k -> tap = ks*4 + k/4, ci = k%4 (ci == 3 and taps >= 9 are zero)
    const size_t nf = wv.size();
    wv.resize(nf + (size_t)24 * cout_pad, 0.f);
    __half* frag = reinterpret_cast<__half*>(wv.data() + nf);
    for (int ks = 0; ks < 3; ++ks)
        for (int nt = 0; nt < cout_pad / 8; ++nt)
            for (int nn = 0; nn < 8; ++nn)
                for (int k = 0; k < 16; ++k) {
                    const int tap = ks * 4 + k / 4, ci = k % 4;
                    const float v = (tap < 9 && ci < 3) ? wv[(size_t)(tap * 3 + ci) * cout_pad + nt * 8 + nn] : 0.f;
                    frag[(((size_t)ks * (cout_pad / 8) + nt) * 8 + nn) * 16 + k] = __float2half_rn(v);
                }
}
static Lin pack_stem(Packer& pk, const std::string& name, int cout, int cout_pad) {
    Lin l;
    l.N = cout_pad;
    l.K = 27;
    const float* w = pk.get(name + ".weight", (int64_t)cout * 27);
    const float* b = pk.get(name + ".bias", cout);
    if (!w || !b) return l;
    std::vector<float> wv, bv;
    pack_stem_w(w, b, cout, cout_pad, wv, bv);
    l.w = pk.add_f32(wv);
    l.b = pk.add_f32(bv);
    return l;
}

struct SwinBlockW {
    Lin qkv, proj, fc1, fc2;
    size_t rpb = 0;       // relative_position_bias_table [121][6] fp32, as in the state_dict
    // rpb in the attention core's accumulator-fragment order, built on the device at load by build_bias_frag_kernel
    // (swin_attention_mma.cu), the only definition of that layout
    size_t table = 0;
    int C = 0, shift = 0;
};

struct SwinW {
    int C = 96, r = 4, cs = 48;
    Lin stem, conv2, down1, down2, up2, up1, toimg;   // 4x: up1 carries proj2 (pack_linear_pixshuf2 with a skip)
    std::vector<SwinBlockW> s1, s2, s3, s4, s5;
};

// Bump allocator over a model's workspace: every take() starts on a 256-byte boundary.  With a null base it hands out
// null pointers and only advances `off`, which is how a forward's plan sizes its workspace (nb200_model::carve).
struct Arena {
    uint8_t* base = nullptr;
    size_t off = 0;
    template <typename T>
    T* take(size_t count) {
        off = (off + 255) & ~(size_t)255;
        T* p = base ? reinterpret_cast<T*>(base + off) : nullptr;
        off += count * sizeof(T);
        return p;
    }
};

struct CUNetW;  // cunet_model.inl
struct LegacyW; // legacy_model.inl
struct DaW;     // depth_model.inl
struct RfW;     // rowflow_model.inl
struct AaW;     // depth_aa_model.inl
struct MlW;     // mlbw_model.inl
struct ZoeW;    // zoe_model.inl
struct InpW;    // inpaint_model.inl
struct Rf2W;    // rowflow_v2_model.inl

}  // namespace nb200

using namespace nb200;

struct nb200_model {
    int kind = 0, no_clip = 0, device = 0;
    int scale = 1, offset = 0, blend = 0;
    uint8_t* blob = nullptr;
    size_t blob_bytes = 0;
    SwinW sw;
    std::shared_ptr<CUNetW> cu;
    std::shared_ptr<LegacyW> lg;
    std::shared_ptr<DaW> da;
    std::shared_ptr<RfW> rf;
    std::shared_ptr<AaW> aa;
    std::shared_ptr<MlW> ml;
    std::shared_ptr<ZoeW> zoe;
    std::shared_ptr<InpW> inp;
    std::shared_ptr<Rf2W> rf2;
    std::shared_ptr<SodW> sod;
    std::shared_ptr<TnW> tn;
    uint8_t* ws = nullptr;
    size_t ws_bytes = 0;
    cudaStream_t copy_stream = nullptr;   // D2H side stream of nb200_tiled_render_host
    // CUDA-graph cache of nb200_model_forward, keyed by (input ptr, output ptr, n, tile, downscale); nullptr = capture failed
    struct GraphKey {
        const void* x; void* z; int n, T, down;
        bool operator<(const GraphKey& o) const {
            return std::tie(x, z, n, T, down) < std::tie(o.x, o.z, o.n, o.T, o.down);
        }
    };
    std::map<GraphKey, cudaGraphExec_t> graphs;
    std::map<GraphKey, int> graph_seen;
    std::map<GraphKey, uint64_t> graph_launches;   // kernel launches one replay stands for (nb200_launch_count)
    int graph_epoch = 0;                            // g_tune_epoch the cached graphs were captured under
    void clear_graphs() {
        for (auto& kv : graphs) if (kv.second) cudaGraphExecDestroy(kv.second);
        graphs.clear();
        graph_seen.clear();
        graph_launches.clear();
    }
    // frame-level buffers of nb200_tiled_render (persistent so that the captured graphs see stable pointers)
    __half* frame_xb = nullptr; size_t frame_xb_bytes = 0;
    __half* frame_z = nullptr; size_t frame_z_bytes = 0;
    int ensure_frame(size_t xb_bytes, size_t z_bytes) {
        if (xb_bytes > frame_xb_bytes) {
            clear_graphs();
            if (frame_xb) cudaFree(frame_xb);
            frame_xb = nullptr; frame_xb_bytes = 0;
            NB_CUDA(cudaMalloc((void**)&frame_xb, xb_bytes));
            frame_xb_bytes = xb_bytes;
        }
        if (z_bytes > frame_z_bytes) {
            clear_graphs();
            if (frame_z) cudaFree(frame_z);
            frame_z = nullptr; frame_z_bytes = 0;
            NB_CUDA(cudaMalloc((void**)&frame_z, z_bytes));
            frame_z_bytes = z_bytes;
        }
        return 0;
    }
    template <typename T>
    T* at(size_t off) const { return reinterpret_cast<T*>(blob + off); }
    int ensure_ws(size_t bytes) {
        if (bytes <= ws_bytes) return 0;
        clear_graphs();   // captured graphs hold pointers into the old workspace
        if (ws) cudaFree(ws);
        ws = nullptr;
        ws_bytes = 0;
        NB_CUDA(cudaMalloc((void**)&ws, bytes));
        ws_bytes = bytes;
        return 0;
    }
    // A forward lists its workspace buffers once, as plan(Arena&): the first run over a null base sizes the workspace
    // (plus a 4 KB tail guard), the second hands out the pointers into it.
    template <typename F>
    int carve(F plan) {
        Arena size;
        plan(size);
        if (ensure_ws(size.off + 4096)) return 1;
        Arena a{ws};
        plan(a);
        return 0;
    }
};

namespace nb200 {

static void pack_swin_blocks(Packer& pk, std::vector<SwinBlockW>& out, const std::string& prefix, int C, int layers) {
    for (int i = 0; i < layers; ++i) {
        SwinBlockW b;
        const std::string p = prefix + ".block." + std::to_string(i);
        b.C = C;
        b.shift = (i % 2 == 0) ? 0 : 3;  // swin_unet.py:30
        b.qkv = pack_linear(pk, p + ".attn.qkv", 3 * C, C);
        b.proj = pack_linear(pk, p + ".attn.proj", C, C);
        b.fc1 = pack_linear(pk, p + ".mlp.0", 2 * C, C);
        b.fc2 = pack_linear(pk, p + ".mlp.3", C, 2 * C);
        const float* t = pk.get(p + ".attn.relative_position_bias_table", 121 * 6);
        if (t) {
            b.rpb = pk.add_f32(std::vector<float>(t, t + 121 * 6));
            b.table = pk.add_f32(std::vector<float>(BIAS_FRAG_FLOATS));   // filled by nb200_model_create
        }
        pk.mark(p + ".attn.relative_position_index");  // buffer; the kernel recomputes the index (swin_transformer.py:267-279)
        out.push_back(b);
    }
}

static void pack_swin(Packer& pk, SwinW& w, int r) {
    const int C = 96;
    w.C = C;
    w.r = r;
    w.cs = (3 * r * r + 15) / 16 * 16;
    w.stem = pack_stem(pk, "unet.patch.0", C / 2, 64);
    w.conv2 = pack_conv(pk, "unet.patch.2", C, C / 2, 3, 3, /*cin_pad=*/64);
    pack_swin_blocks(pk, w.s1, "unet.swin1", C, 2);
    w.down1 = pack_conv(pk, "unet.down1.conv", 2 * C, C, 2, 2);
    pack_swin_blocks(pk, w.s2, "unet.swin2", 2 * C, 2);
    w.down2 = pack_conv(pk, "unet.down2.conv", 2 * C, 2 * C, 2, 2);
    pack_swin_blocks(pk, w.s3, "unet.swin3", 2 * C, 6);
    w.up2 = pack_linear_pixshuf2(pk, "unet.up2.proj", 2 * C, 2 * C);
    pack_swin_blocks(pk, w.s4, "unet.swin4", 2 * C, 2);
    if (r == 4) {
        w.up1 = pack_linear_pixshuf2(pk, "unet.up1.proj", 2 * C, 2 * C, "unet.proj2", C);
        pack_swin_blocks(pk, w.s5, "unet.swin5", 2 * C, 2);
        w.toimg = pack_linear(pk, "unet.to_image.proj", 3 * r * r, 2 * C, w.cs);
    } else {
        w.up1 = pack_linear_pixshuf2(pk, "unet.up1.proj", C, 2 * C);
        pack_swin_blocks(pk, w.s5, "unet.swin5", C, 2);
        w.toimg = pack_linear(pk, "unet.to_image.proj", 3 * r * r, C, w.cs);
    }
}

// ---------------------------------------------------------------------------------------------
// forward helpers
// ---------------------------------------------------------------------------------------------
// split > 0: the N outputs are written as N/split dense [M][split] planes (OUT_SPLIT); a_planes > 1: A is given as planes
static int linear_flat(cudaStream_t st, const nb200_model* m, const Lin& l, const __half* A, long long M, int lda, __half* out,
                       int ldo, int act, const __half* res = nullptr, int ldr = 0, int split = 0, int a_planes = 1) {
    ConvGemm g;
    g.A = A; g.B = 1; g.Hi = 1; g.Wi = (int)M; g.Ci = lda; g.Cin = l.K / a_planes; g.kind = CG_LINEAR_FLAT;
    g.a_planes = a_planes; g.a_plane_stride = (long long)M * lda;
    g.Wt = m->at<__half>(l.w); g.N = l.N; g.bias = m->at<float>(l.b); g.act = act; g.out = out; g.ldo = ldo;
    g.res = res; g.ldr = ldr;
    if (split) { g.out_mode = OUT_SPLIT; g.cout = split; g.split_stride = (long long)M * split; g.ldo = split; }
    return conv_gemm(st, g);
}

// toimg != nullptr: the block's output is not written to X; Y = output . Wtoimg^T + b ([T][toimg->N]) is, by the tail kernel
static int swin_block(cudaStream_t st, const nb200_model* m, const SwinBlockW& w, __half* X, int n, int H, __half* ATT,
                      const Lin* toimg = nullptr, __half* Y = nullptr) {
    const int C = w.C;
    const long long T = (long long)n * H * H;
    // two launches per block: q/k/v, x1 and the hidden tensor stay in shared memory / registers
    if (swin_attn_fused(st, X, m->at<__half>(w.qkv.w), m->at<float>(w.qkv.b), m->at<float>(w.table), ATT, n, H, H, C, w.shift)) return 1;
    return swin_mlp_fused(st, X, ATT, T, C, m->at<__half>(w.proj.w), m->at<float>(w.proj.b), m->at<__half>(w.fc1.w), m->at<float>(w.fc1.b),
                          m->at<__half>(w.fc2.w), m->at<float>(w.fc2.b), toimg ? Y : nullptr, toimg ? toimg->N : 0,
                          toimg ? m->at<__half>(toimg->w) : nullptr, toimg ? m->at<float>(toimg->b) : nullptr);
}

static int swin_forward(nb200_model* m, cudaStream_t st, const __half* x, int n, int T, int down, void* z) {
    const SwinW& w = m->sw;
    NB_CHECK(T > 16 && (T - 16) % 12 == 0 && (T - 16) % 16 == 0, "invalid tile size for swin_unet (swin_unet.py:202-205)");
    const int C = w.C, Hc = T - 16, H2 = Hc / 2, H3 = Hc / 4, S1w = T - 2;
    const int C5 = w.r == 4 ? 2 * C : C;
    const size_t t1 = (size_t)n * Hc * Hc;
    __half *S1, *X1, *ATT, *X2, *X3, *X4, *X5, *Y;
    if (m->carve([&](Arena& a) {
            S1 = a.take<__half>((size_t)n * S1w * S1w * 64);
            X1 = a.take<__half>(t1 * C);
            ATT = a.take<__half>(t1 * C5);
            X2 = a.take<__half>(t1 / 4 * 2 * C);
            X3 = a.take<__half>(t1 / 16 * 2 * C);
            X4 = a.take<__half>(t1 / 4 * 2 * C);
            X5 = a.take<__half>(t1 * C5);
            Y = a.take<__half>(t1 * w.cs);
        })) return 1;

    // patch stem (swin_unet.py:133-137) + crop 6 (:182) folded into the second conv's addressing
    if (stem_conv3x3(st, x, m->at<float>(w.stem.w), m->at<float>(w.stem.b), S1, n, T, T, 64, 64)) return 1;
    {
        ConvGemm g;
        g.A = S1 + ((size_t)6 * S1w + 6) * 64; g.B = n; g.Hi = Hc + 2; g.Wi = Hc + 2; g.Ci = 64; g.Cin = 64;
        g.a_row_stride = (long long)S1w * 64; g.a_img_stride = (long long)S1w * S1w * 64; g.kind = CG_CONV3;
        g.Wt = m->at<__half>(w.conv2.w); g.N = C; g.bias = m->at<float>(w.conv2.b); g.act = ACT_LRELU01; g.out = X1; g.ldo = C;
        if (conv_gemm(st, g)) return 1;
    }
    for (const auto& b : w.s1) if (swin_block(st, m, b, X1, n, Hc, ATT)) return 1;   // x3
    {   // down1 (swin_unet.py:45-62)
        ConvGemm g;
        g.A = X1; g.B = n; g.Hi = Hc; g.Wi = Hc; g.Ci = C; g.Cin = C; g.kind = CG_DOWN2;
        g.Wt = m->at<__half>(w.down1.w); g.N = 2 * C; g.bias = m->at<float>(w.down1.b); g.out = X2; g.ldo = 2 * C;
        if (conv_gemm(st, g)) return 1;
    }
    for (const auto& b : w.s2) if (swin_block(st, m, b, X2, n, H2, ATT)) return 1;   // x4
    {   // down2
        ConvGemm g;
        g.A = X2; g.B = n; g.Hi = H2; g.Wi = H2; g.Ci = 2 * C; g.Cin = 2 * C; g.kind = CG_DOWN2;
        g.Wt = m->at<__half>(w.down2.w); g.N = 2 * C; g.bias = m->at<float>(w.down2.b); g.out = X3; g.ldo = 2 * C;
        if (conv_gemm(st, g)) return 1;
    }
    for (const auto& b : w.s3) if (swin_block(st, m, b, X3, n, H3, ATT)) return 1;   // x5
    {   // up2 + skip: x = up2(x5) + x4   (swin_unet.py:190-191)
        ConvGemm g;
        g.A = X3; g.B = n; g.Hi = H3; g.Wi = H3; g.Ci = 2 * C; g.Cin = 2 * C; g.kind = CG_LINEAR_2D;
        g.Wt = m->at<__half>(w.up2.w); g.N = w.up2.N; g.bias = m->at<float>(w.up2.b); g.out = X4; g.ldo = 2 * C;
        g.out_mode = OUT_PIXSHUF2; g.cout = 2 * C; g.res = X2; g.ldr = 2 * C; g.res_H = H2; g.res_W = H2;
        if (conv_gemm(st, g)) return 1;
    }
    for (const auto& b : w.s4) if (swin_block(st, m, b, X4, n, H2, ATT)) return 1;
    {   // up1 + skip; 4x: the skip is proj2(x3) (swin_unet.py:159,195), the GEMM's second A operand
        ConvGemm g;
        g.A = X4; g.B = n; g.Hi = H2; g.Wi = H2; g.Ci = 2 * C; g.Cin = 2 * C; g.kind = CG_LINEAR_2D;
        g.Wt = m->at<__half>(w.up1.w); g.N = w.up1.N; g.bias = m->at<float>(w.up1.b); g.out = X5; g.ldo = C5;
        g.out_mode = OUT_PIXSHUF2; g.cout = C5;
        if (w.r == 4) { g.A2 = X1; g.Cin2 = C; g.ld2 = C; }
        else { g.res = X1; g.ldr = C5; g.res_H = Hc; g.res_W = Hc; }
        if (conv_gemm(st, g)) return 1;
    }
    // the last block's tail also runs ToImage.proj (:109) and writes only its result Y
    for (size_t i = 0; i < w.s5.size(); ++i)
        if (swin_block(st, m, w.s5[i], X5, n, Hc, ATT, i + 1 == w.s5.size() ? &w.toimg : nullptr, Y)) return 1;
    return to_image(st, Y, z, n, Hc, Hc, w.cs, w.r, down);
}

}  // namespace nb200

#include "cunet_model.inl"
#include "legacy_model.inl"
// debug tap (nb200_debug_tap): stage `g_tap_id` of the next ZoeDepth, light_inpaint_v1 or TransNetV2 forward is copied to
// `g_tap_buf` (ZoeDepth ids 0..15 in zoe_model.inl; light_inpaint_v1 ids 100..173, table in DESIGN.md §5; TransNetV2 ids
// 200..205 in transnet_model.inl); the forward warp's kernel writes id 300 itself (warp_forward.cu)
static int g_tap_id = -1;
static void* g_tap_buf = nullptr;
static size_t g_tap_cap = 0;
static int tap_copy(cudaStream_t st, int id, const void* src, size_t bytes) {
    if (id != g_tap_id || !g_tap_buf) return 0;
    NB_CHECK(bytes <= g_tap_cap, "debug tap buffer too small: need " + std::to_string(bytes) + " bytes");
    NB_CUDA(cudaMemcpyAsync(g_tap_buf, src, bytes, cudaMemcpyDeviceToDevice, st));
    return 0;
}

int nb200::debug_tap_target(int id, size_t bytes, void** buf) {
    *buf = nullptr;
    if (id != g_tap_id || !g_tap_buf) return 0;
    NB_CHECK(bytes <= g_tap_cap, "debug tap buffer too small: need " + std::to_string(bytes) + " bytes");
    *buf = g_tap_buf;
    return 0;
}

#include "depth_model.inl"
#include "wa_block.inl"
#include "rowflow_model.inl"
#include "rowflow_v2_model.inl"
#include "depth_aa_model.inl"
#include "mlbw_model.inl"
#include "zoe_model.inl"
#include "inpaint_model.inl"
#include "sod_model.inl"
#include "transnet_model.inl"

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
extern "C" int nb200_model_create(int kind, int n_tensors, const char* const* names, const float* const* data,
                                  const int64_t* numel, int no_clip, nb200_model** out) {
    NB_CHECK(out && names && data && numel, "null pointer");
    NB_CHECK(kind >= NB200_MODEL_UPCUNET && kind <= NB200_MODEL_TRANSNET_V2, "unknown model kind");
    int dev = 0;
    NB_CUDA(cudaGetDevice(&dev));
    if (nb200_check_device(dev)) return 1;
    {
        // frame-level scratch comes from cudaMallocAsync every render: keep freed blocks cached in the device pool
        // instead of returning them to the driver at each synchronisation
        cudaMemPool_t pool;
        if (cudaDeviceGetDefaultMemPool(&pool, dev) == cudaSuccess) {
            uint64_t keep = ~0ull;
            cudaMemPoolSetAttribute(pool, cudaMemPoolAttrReleaseThreshold, &keep);
        }
    }
    Packer pk;
    for (int i = 0; i < n_tensors; ++i) pk.src[names[i]] = HostTensor{data[i], numel[i], false};
    auto m = new nb200_model();
    m->kind = kind;
    m->no_clip = no_clip;
    m->device = dev;
    switch (kind) {
        case NB200_MODEL_SWIN_UNET_1X: pack_swin(pk, m->sw, 1); m->scale = 1; m->offset = 8; m->blend = 4; break;    // swin_unet.py:213
        case NB200_MODEL_SWIN_UNET_2X: pack_swin(pk, m->sw, 2); m->scale = 2; m->offset = 16; m->blend = 8; break;   // :234
        case NB200_MODEL_SWIN_UNET_4X: pack_swin(pk, m->sw, 4); m->scale = 4; m->offset = 32; m->blend = 16; break;  // :267
        case NB200_MODEL_UPCUNET: m->cu = pack_cunet(pk, true); m->scale = 2; m->offset = 36; m->blend = 0; break;   // cunet.py:144
        case NB200_MODEL_CUNET: m->cu = pack_cunet(pk, false); m->scale = 1; m->offset = 28; m->blend = 0; break;    // cunet.py:178
        case NB200_MODEL_DEPTH_ANYTHING_V2_S: m->da = pack_depth_anything(pk, 0); m->scale = 1; break;
        case NB200_MODEL_DEPTH_ANYTHING_V2_B: m->da = pack_depth_anything(pk, 1); m->scale = 1; break;
        case NB200_MODEL_DEPTH_ANYTHING_V2_L: m->da = pack_depth_anything(pk, 2); m->scale = 1; break;
        case NB200_MODEL_ZOEDEPTH_N: m->zoe = pack_zoedepth(pk); m->scale = 1; break;                                   // zoedepth_model.py:151-157
        case NB200_MODEL_MLBW: m->ml = pack_mlbw(pk); m->scale = 1; m->offset = 32; m->blend = 4; break;               // mlbw.py:41
        case NB200_MODEL_DEPTH_AA: m->aa = pack_depth_aa(pk); m->scale = 1; break;                                     // depth_aa.py:34
        case NB200_MODEL_ROW_FLOW_V3: m->rf = pack_row_flow(pk); m->scale = 1; m->offset = 32; m->blend = 4; break;   // row_flow_v3.py:37
        case NB200_MODEL_UPCONV_7: m->lg = pack_legacy(pk, true); m->scale = 2; m->offset = 14; m->blend = 0; break;  // upconv_7.py:11
        case NB200_MODEL_VGG_7: m->lg = pack_legacy(pk, false); m->scale = 1; m->offset = 7; m->blend = 0; break;     // vgg_7.py:11
        case NB200_MODEL_LIGHT_INPAINT_V1: m->inp = pack_light_inpaint(pk); m->scale = 1; m->offset = 16; m->blend = 8; break;  // light_inpaint_v1.py:56
        case NB200_MODEL_ROW_FLOW_V2: m->rf2 = pack_row_flow_v2(pk); m->scale = 1; m->offset = 28; m->blend = 4; break;   // row_flow_v2.py:14
        case NB200_MODEL_SOD_V1: m->sod = pack_sod(pk); m->scale = 1; break;                                           // sod_v1.py:15
        case NB200_MODEL_ZOEDEPTH_ANY_N: m->zoe = pack_zoedepth_any(pk, false); m->scale = 1; break;                    // zoedepth_model.py:20
        case NB200_MODEL_ZOEDEPTH_ANY_K: m->zoe = pack_zoedepth_any(pk, true); m->scale = 1; break;
        case NB200_MODEL_DEPTH_ANYTHING_V1_S: m->da = pack_depth_anything(pk, 0, "", true); m->scale = 1; break;     // depth_anything_model.py:36-38
        case NB200_MODEL_DEPTH_ANYTHING_V1_B: m->da = pack_depth_anything(pk, 1, "", true); m->scale = 1; break;
        case NB200_MODEL_DEPTH_ANYTHING_V1_L: m->da = pack_depth_anything(pk, 2, "", true); m->scale = 1; break;
        case NB200_MODEL_TRANSNET_V2: m->tn = pack_transnet(pk); m->scale = 1; break;                                    // transnetv2.py:7-47
    }
    if (pk.err.empty())
        for (auto& kv : pk.src)
            if (!kv.second.used) { pk.err = "unexpected key in state_dict: " + kv.first; break; }
    if (!pk.err.empty()) {
        delete m;
        return fail(pk.err);
    }
    m->blob_bytes = pk.blob.size();
    cudaError_t e = cudaMalloc((void**)&m->blob, m->blob_bytes);
    if (e == cudaSuccess) e = cudaMemcpy(m->blob, pk.blob.data(), m->blob_bytes, cudaMemcpyHostToDevice);
    // Swin blocks: each bias-fragment slot is built from the block's raw table, then synchronised, since forwards may run on
    // non-blocking streams
    int rc = 0;
    for (const auto* blocks : {&m->sw.s1, &m->sw.s2, &m->sw.s3, &m->sw.s4, &m->sw.s5})
        for (const SwinBlockW& b : *blocks)
            if (e == cudaSuccess && !rc) rc = build_bias_frag(0, m->at<float>(b.rpb), m->at<float>(b.table));
    if (e == cudaSuccess && !rc) e = cudaStreamSynchronize(0);
    if (e != cudaSuccess || rc) {
        nb200_model_destroy(m);
        return rc ? 1 : fail(std::string("weight upload failed: ") + cudaGetErrorString(e));
    }
    *out = m;
    return 0;
}

extern "C" void nb200_model_destroy(nb200_model* m) {
    if (!m) return;
    if (m->blob) cudaFree(m->blob);
    if (m->ws) cudaFree(m->ws);
    m->clear_graphs();
    if (m->frame_xb) cudaFree(m->frame_xb);
    if (m->frame_z) cudaFree(m->frame_z);
    if (m->copy_stream) cudaStreamDestroy(m->copy_stream);
    delete m;
}

extern "C" int nb200_model_info(const nb200_model* m, int* scale, int* offset, int* blend_size) {
    NB_CHECK(m, "null model");
    if (scale) *scale = m->scale;
    if (offset) *offset = m->offset;
    if (blend_size) *blend_size = m->blend;
    return 0;
}

extern "C" int nb200_model_weight_blob(nb200_model* m, void** dev_ptr, size_t* bytes) {
    NB_CHECK(m && dev_ptr && bytes, "null pointer");
    *dev_ptr = m->blob;
    *bytes = m->blob_bytes;
    return 0;
}

static int model_out_geometry(const nb200_model* m, int tile_size, int down, int* scale, int* offset, int* blend, int* S) {
    NB_CHECK(down == 1 || down == 2 || down == 4, "downscale must be 1, 2 or 4");
    NB_CHECK(down == 1 || m->kind == NB200_MODEL_SWIN_UNET_4X, "downscale is defined for swin_unet_4x only (swin_unet.py:339-387)");
    // SwinUNetDownscaled: offset = 32//f, scale = 4//f, blend = 4*f (swin_unet.py:345-350)
    *scale = down == 1 ? m->scale : 4 / down;
    *offset = down == 1 ? m->offset : 32 / down;
    *blend = down == 1 ? m->blend : 4 * down;
    *S = tile_size * (*scale) - 2 * (*offset);
    NB_CHECK(*S > 0, "tile_size too small");
    return 0;
}

extern "C" int nb200_model_forward(nb200_model* m, const void* x, int n, int tile_size, int downscale, void* z, void* stream) {
    NB_CHECK(m && x && z, "null pointer");
    NB_CHECK(n > 0, "empty batch");
    int scale, offset, blend, S;
    if (model_out_geometry(m, tile_size, downscale, &scale, &offset, &blend, &S)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    NB_CHECK(m->kind <= NB200_MODEL_SWIN_UNET_4X || m->lg, "not an image-to-image model");
    auto eager = [&]() {
        if (m->lg) return legacy_forward(m, st, (const __half*)x, n, tile_size, (__half*)z);
        if (m->kind >= NB200_MODEL_SWIN_UNET_1X) return swin_forward(m, st, (const __half*)x, n, tile_size, downscale, z);
        return cunet_forward(m, st, (const __half*)x, n, tile_size, (__half*)z);
    };
    // CUDA graphs (g_tune[9]): the ~80 launches of one tile batch are replayed as one graph launch once the same
    // (buffers, shape) has been seen twice; removes most of the inter-kernel launch latency.  Never while the event
    // profiler is on.
    if (!g_tune[9] || g_prof_enabled.load(std::memory_order_relaxed)) return eager();
    if (m->graph_epoch != g_tune_epoch.load()) {            // a tuning knob changed: the captured launch configurations are stale
        m->clear_graphs();
        m->graph_epoch = g_tune_epoch.load();
    }
    if (m->graph_seen.size() > 1024) m->graph_seen.clear();  // callers that never repeat a (buffers, shape) key
    const nb200_model::GraphKey key{x, z, n, tile_size, downscale};
    auto it = m->graphs.find(key);
    if (it != m->graphs.end()) {
        if (!it->second) return eager();
        NB_CUDA(cudaGraphLaunch(it->second, st));
        g_launches.fetch_add(m->graph_launches[key]);
        return 0;
    }
    if (++m->graph_seen[key] < 2) return eager();           // first sighting: eager (also sizes the workspace, sets func attributes)
    if (m->graphs.size() > 256) m->clear_graphs();
    cudaGraph_t graph = nullptr;
    cudaError_t e = cudaStreamBeginCapture(st, cudaStreamCaptureModeThreadLocal);
    int rc = 1;
    const uint64_t l0 = g_launches.load();
    if (e == cudaSuccess) {
        rc = eager();
        e = cudaStreamEndCapture(st, &graph);
    }
    const uint64_t captured = g_launches.load() - l0;
    cudaGraphExec_t exec = nullptr;
    if (e == cudaSuccess && rc == 0 && graph) e = cudaGraphInstantiate(&exec, graph, 0);
    if (graph) cudaGraphDestroy(graph);
    if (e != cudaSuccess || rc != 0 || !exec) {
        cudaGetLastError();                                  // capture is not available for this sequence: stay eager
        m->graphs[key] = nullptr;
        return eager();
    }
    m->graphs[key] = exec;
    m->graph_launches[key] = captured;
    NB_CUDA(cudaGraphLaunch(exec, st));                      // (the launches counted during capture stand for this first replay)
    return 0;
}

extern "C" int nb200_tiled_render(nb200_model* m, const float* x, int C, int H, int W, int tile_size, int batch_size,
                                  int downscale, float* out, void* stream) {
    NB_CHECK(m && x && out, "null pointer");
    NB_CHECK(C == 3, "models take 3-channel input");
    NB_CHECK(batch_size > 0, "batch_size must be positive");
    int scale, offset, blend, S;
    if (model_out_geometry(m, tile_size, downscale, &scale, &offset, &blend, &S)) return 1;
    nb200_tile_config cfg;
    if (nb200_tile_config_create(H, W, scale, offset, tile_size, blend, &cfg)) return 1;
    const int ntiles = cfg.h_blocks * cfg.w_blocks;
    // frame-level buffers (stream-ordered): the unfolded tile batch and every tile's output
    // frame-level buffers: the unfolded tile batch and every tile's output (persistent per model; not re-entrant:
    // one render at a time per model handle, like the reference's module)
    const size_t xb_elems = (size_t)batch_size * tile_size * tile_size * 8, z_tile = (size_t)3 * S * S;
    const int z_f32 = downscale > 1;                      // the downscaled models return fp32 tiles (swin_unet.py:366-379)
    const size_t zsz = z_f32 ? 4 : 2;
    if (m->ensure_frame(xb_elems * 2, (size_t)ntiles * z_tile * zsz)) return 1;
    __half* xb = m->frame_xb;
    uint8_t* zall = reinterpret_cast<uint8_t*>(m->frame_z);
    int rc = 0;
    for (int t0 = 0; t0 < ntiles && !rc; t0 += batch_size) {
        const int nb = ntiles - t0 < batch_size ? ntiles - t0 : batch_size;
        rc = nb200_tile_unfold(x, C, H, W, &cfg, tile_size, t0, nb, xb, 8, stream);
        if (!rc) rc = nb200_model_forward(m, xb, nb, tile_size, downscale, zall + (size_t)t0 * z_tile * zsz, stream);
    }
    if (!rc) rc = tile_gather_blend_rows(zall, z_f32, C, &cfg, scale, offset, tile_size, blend, out, 0, cfg.y_h, stream);
    return rc;
}

// Same render with HOST buffers (the call a non-torch binding makes, and bench.py's e2e leg): the input is copied in once,
// and the output is blended and copied out in bands - as soon as every tile row covering a band of output rows has been
// computed, that band is blended on the compute stream and its D2H copy runs on a side stream under the remaining tile
// batches.  Only the last band's copy is exposed.  Pinned host buffers give the overlap; pageable ones still work.
extern "C" int nb200_tiled_render_host(nb200_model* m, const float* x_host, int C, int H, int W, int tile_size, int batch_size,
                                       int downscale, float* out_host, void* stream) {
    NB_CHECK(m && x_host && out_host, "null pointer");
    NB_CHECK(C == 3, "models take 3-channel input");
    NB_CHECK(batch_size > 0, "batch_size must be positive");
    int scale, offset, blend, S;
    if (model_out_geometry(m, tile_size, downscale, &scale, &offset, &blend, &S)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    nb200_tile_config cfg;
    if (nb200_tile_config_create(H, W, scale, offset, tile_size, blend, &cfg)) return 1;
    if (!m->copy_stream) NB_CUDA(cudaStreamCreateWithFlags(&m->copy_stream, cudaStreamNonBlocking));
    cudaStream_t cs = m->copy_stream;
    const int ntiles = cfg.h_blocks * cfg.w_blocks;
    __half* xb = nullptr;
    uint8_t* zall = nullptr;
    float *xd = nullptr, *od = nullptr;
    const size_t xb_elems = (size_t)batch_size * tile_size * tile_size * 8, z_tile = (size_t)3 * S * S;
    const int z_f32 = downscale > 1;
    const size_t zsz = z_f32 ? 4 : 2;
    const size_t oplane = (size_t)cfg.y_h * cfg.y_w;
    struct AsyncFree {   // the frame-level scratch goes back to the stream-ordered pool on every exit path
        cudaStream_t st; float** a; float** b;
        ~AsyncFree() { if (*a) cudaFreeAsync(*a, st); if (*b) cudaFreeAsync(*b, st); }
    } scratch_guard{st, &xd, &od};
    NB_CUDA(cudaMallocAsync((void**)&xd, (size_t)C * H * W * 4, st));
    NB_CUDA(cudaMallocAsync((void**)&od, (size_t)C * oplane * 4, st));
    if (m->ensure_frame(xb_elems * 2, (size_t)ntiles * z_tile * zsz)) return 1;
    xb = m->frame_xb; zall = reinterpret_cast<uint8_t*>(m->frame_z);
    NB_CUDA(cudaMemcpyAsync(xd, x_host, (size_t)C * H * W * 4, cudaMemcpyHostToDevice, st));
    int rc = 0, rows_done = 0;
    for (int t0 = 0; t0 < ntiles && !rc; t0 += batch_size) {
        const int nb = ntiles - t0 < batch_size ? ntiles - t0 : batch_size;
        rc = nb200_tile_unfold(xd, C, H, W, &cfg, tile_size, t0, nb, xb, 8, stream);
        if (!rc) rc = nb200_model_forward(m, xb, nb, tile_size, downscale, zall + (size_t)t0 * z_tile * zsz, stream);
        if (rc) break;
        // output rows below the first unfinished tile row are final
        const int rows_full = (t0 + nb) / cfg.w_blocks;
        int y1 = rows_full >= cfg.h_blocks ? cfg.y_h : rows_full * cfg.output_tile_step;
        if (y1 > cfg.y_h) y1 = cfg.y_h;
        if (y1 > rows_done) {
            rc = tile_gather_blend_rows(zall, z_f32, C, &cfg, scale, offset, tile_size, blend, od, rows_done, y1, stream);
            if (rc) break;
            cudaEvent_t ev;
            NB_CUDA(cudaEventCreateWithFlags(&ev, cudaEventDisableTiming));
            NB_CUDA(cudaEventRecord(ev, st));
            NB_CUDA(cudaStreamWaitEvent(cs, ev, 0));
            NB_CUDA(cudaEventDestroy(ev));   // released once the wait has been satisfied
            for (int c = 0; c < C; ++c) {
                const size_t o = (size_t)c * oplane + (size_t)rows_done * cfg.y_w;
                NB_CUDA(cudaMemcpyAsync(out_host + o, od + o, (size_t)(y1 - rows_done) * cfg.y_w * 4, cudaMemcpyDeviceToHost, cs));
            }
            rows_done = y1;
        }
    }
    // the caller's stream completes only after the last band has landed in host memory
    cudaEvent_t ev_end;
    NB_CUDA(cudaEventCreateWithFlags(&ev_end, cudaEventDisableTiming));
    NB_CUDA(cudaEventRecord(ev_end, cs));
    NB_CUDA(cudaStreamWaitEvent(st, ev_end, 0));
    NB_CUDA(cudaEventDestroy(ev_end));
    return rc;   // scratch_guard frees xd / od behind the last copy (stream-ordered)
}

// debug: copy intermediate `id` of the following nb200_zoedepth_forward / nb200_light_inpaint / nb200_transnetv2_forward calls,
// or the padded depth rows of the following nb200_forward_warp calls (id 300), into dev_buf (capacity bytes); id < 0 disables
extern "C" int nb200_debug_tap(int id, void* dev_buf, size_t capacity) {
    g_tap_id = id; g_tap_buf = dev_buf; g_tap_cap = capacity;
    return 0;
}

// Host-only: the relative-position table resample of the BEiT blocks (MiDaS beit.py _get_rel_pos_bias) for a ph x pw token grid.
// table [(2g-1)^2 + 3][heads] -> out [(2ph-1)(2pw-1) + 3][heads].  No GPU needed (tests/test_host_logic.py).
extern "C" int nb200_zoe_rel_pos_table(const float* table, int g, int heads, int ph, int pw, float* out) {
    NB_CHECK(table && out, "null pointer");
    NB_CHECK(g > 0 && heads > 0 && ph > 0 && pw > 0, "bad shape");
    const size_t n = ((size_t)(2 * g - 1) * (2 * g - 1) + 3) * heads;
    zoe_resample_table(std::vector<float>(table, table + n), g, heads, ph, pw, out);
    return 0;
}

// ZoeDepth.forward(x)['metric_depth'] (what zoedepth_model._forward calls, iw3/zoedepth_model.py:23-27)
extern "C" int nb200_zoedepth_forward(nb200_model* m, const float* x, int B, int H, int W, float* depth, void* stream) {
    NB_CHECK(m && x && depth, "null pointer");
    NB_CHECK(m->zoe, "model is not a ZoeDepth network");
    NB_CHECK(B > 0, "empty batch");
    return zoedepth_forward(m, (cudaStream_t)stream, x, B, H, W, depth);
}

// DepthAnythingV2.forward (what DepthAnythingModel._forward calls, iw3/depth_anything_model.py:113-119)
extern "C" int nb200_depth_anything_forward(nb200_model* m, const float* x, int B, int H, int W, float* depth, void* stream) {
    NB_CHECK(m && x && depth, "null pointer");
    NB_CHECK(m->da, "model is not a Depth-Anything network");
    NB_CHECK(B > 0, "empty batch");
    return depth_anything_forward(m, (cudaStream_t)stream, x, B, H, W, depth);
}

// MLBW.forward with delta_output=True (iw3/models/mlbw.py:96-127,237-245): the x components of the L flow layers and their weights
extern "C" int nb200_mlbw_delta(nb200_model* m, const float* x, int B, int h, int w, float* delta, float* layer_weight, void* stream) {
    NB_CHECK(m && x && delta && layer_weight, "null pointer");
    NB_CHECK(m->kind == NB200_MODEL_MLBW && m->ml, "model is not sbs.mlbw");
    NB_CHECK(!m->ml->hole, "this sbs.mlbw has a hole_mask head (sbs.mask_mlbw_l2): use nb200_mlbw_delta_hole");
    NB_CHECK(B > 0 && h > 0 && w > 0, "empty input");
    return mlbw_forward(m, (cudaStream_t)stream, x, B, h, w, delta, layer_weight, nullptr);
}
extern "C" int nb200_mlbw_num_layers(const nb200_model* m) { return (m && m->kind == NB200_MODEL_MLBW && m->ml) ? m->ml->L : 0; }
extern "C" int nb200_mlbw_has_hole_mask(const nb200_model* m) { return (m && m->kind == NB200_MODEL_MLBW && m->ml && m->ml->hole) ? 1 : 0; }

// MLBW._forward_delta_only of a hole_mask model (mlbw.py:232-240): delta, layer_weight and the hole logits
extern "C" int nb200_mlbw_delta_hole(nb200_model* m, const float* x, int B, int h, int w, float* delta, float* layer_weight,
                                     float* hole_logits, void* stream) {
    NB_CHECK(m && x && delta && layer_weight && hole_logits, "null pointer");
    NB_CHECK(m->kind == NB200_MODEL_MLBW && m->ml, "model is not sbs.mlbw");
    NB_CHECK(m->ml->hole, "this sbs.mlbw has no hole_mask head: use nb200_mlbw_delta");
    NB_CHECK(B > 0 && h > 0 && w > 0, "empty input");
    return mlbw_forward(m, (cudaStream_t)stream, x, B, h, w, delta, layer_weight, hole_logits);
}

// postprocess_hole_mask (iw3/backward_warp.py:382-393), steps 1-3: closing, align-corners resize, sigmoid > threshold
extern "C" int nb200_hole_mask(const float* logits, int B, int h, int w, int H, int W, float threshold, int mirror, float* out,
                               void* stream) {
    NB_CHECK(logits && out, "null pointer");
    NB_CHECK(B > 0 && h > 0 && w > 0 && H > 0 && W > 0, "empty mask");
    return hole_mask((cudaStream_t)stream, logits, B, h, w, H, W, threshold, mirror ? 1 : 0, out);
}

// DepthAA.forward / DepthAA.infer (iw3/models/depth_aa.py:46-87)
extern "C" int nb200_depth_aa(nb200_model* m, const float* x, int B, int H, int W, int mode, float* out, void* stream) {
    NB_CHECK(m && x && out, "null pointer");
    NB_CHECK(m->kind == NB200_MODEL_DEPTH_AA && m->aa, "model is not iw3.depth_aa");
    NB_CHECK(B > 0 && H > 0 && W > 0 && mode >= 0 && mode <= 2, "bad arguments");
    return depth_aa_forward(m, (cudaStream_t)stream, x, B, H, W, mode, out);
}

// RowFlowV3.forward with delta_output=True (iw3/models/row_flow_v3.py:111-116) - the x component of the returned delta
extern "C" int nb200_row_flow_delta(nb200_model* m, const float* x, int B, int h, int w, float* delta, void* stream) {
    NB_CHECK(m && x && delta, "null pointer");
    NB_CHECK(m->kind == NB200_MODEL_ROW_FLOW_V3 && m->rf, "model is not sbs.row_flow_v3");
    NB_CHECK(B > 0 && h > 0 && w > 0, "bad shape");
    return row_flow_forward(m, (cudaStream_t)stream, x, B, h, w, delta);
}

// RowFlowV2.forward with delta_output=True (iw3/models/row_flow_v2.py:80-86) - the x component of the returned delta
extern "C" int nb200_row_flow_v2_delta(nb200_model* m, const float* x, int B, int h, int w, float* delta, void* stream) {
    NB_CHECK(m && x && delta, "null pointer");
    NB_CHECK(m->kind == NB200_MODEL_ROW_FLOW_V2 && m->rf2, "model is not sbs.row_flow_v2");
    NB_CHECK(B > 0 && h > 0 && w > 0, "bad shape");
    return rf2_forward((cudaStream_t)stream, m->blob + m->rf2->params, x, B, h, w, delta);
}

// SODV1.infer (iw3/models/sod_v1.py:47-54) under autocast: sigmoid(U2NETP(cat(rgb, d, d ** 0.5, d ** 2))) at 192 x 192
extern "C" int nb200_sod_forward(nb200_model* m, const float* rgb, int B, int H, int W, const float* depth, int h, int w,
                                 float* saliency, float* depth192, void* stream) {
    NB_CHECK(m && rgb && depth && saliency && depth192, "null pointer");
    NB_CHECK(m->kind == NB200_MODEL_SOD_V1 && m->sod, "model is not iw3.sod_v1");
    NB_CHECK(B > 0 && H > 0 && W > 0 && h > 0 && w > 0, "bad shape");
    return sod_forward((cudaStream_t)stream, m->blob, *m->sod, rgb, B, H, W, depth, h, w, saliency, depth192);
}

// TransNetV2.forward (nunif/utils/transnetv2.py:49-87) on B windows of T frames: the one_hot and many_hot logits
extern "C" int nb200_transnetv2_forward(nb200_model* m, const float* x, int B, int T, float* one_hot, float* many_hot, void* stream) {
    NB_CHECK(m && x && one_hot && many_hot, "null pointer");
    NB_CHECK(m->kind == NB200_MODEL_TRANSNET_V2 && m->tn, "model is not TransNetV2");
    NB_CHECK(B > 0 && T > 0 && (long long)B * T <= (1 << 20), "bad shape");
    return transnet_forward(m, (cudaStream_t)stream, x, B, T, one_hot, many_hot);
}

// iw3/dilation.py:67-98: n = max(round(W / base_width * n_iter), 1) (Python's round: half to even), 0 when n_iter <= 0
static int dilation_run(int n_iter, int base_width, int W) {
    if (n_iter <= 0) return 0;
    if (base_width <= 0) return n_iter;
    const double n = std::nearbyint((double)W / base_width * n_iter);
    return n < 1 ? 1 : (int)n;
}

extern "C" int nb200_inpaint_mask(const float* mask, int B, int H, int W, int binarize, int closing, int outer_iter, int inner_iter,
                                  int base_width, int mirror, float* out, void* stream) {
    NB_CHECK(mask && out, "null pointer");
    NB_CHECK(B > 0 && H > 0 && W > 0, "empty mask");
    const int no = dilation_run(outer_iter, base_width, W), ni = dilation_run(inner_iter, base_width, W);
    cudaStream_t st = (cudaStream_t)stream;
    float* tmp = nullptr;
    if (closing) NB_CUDA(cudaMallocAsync((void**)&tmp, (size_t)B * H * W * 4, st));
    // in image coordinates the mirrored mask's right-hand runs (dilate_outer) grow to the left
    const int rc = inpaint_mask(st, mask, B, H, W, binarize, closing, mirror ? ni : no, mirror ? no : ni, tmp, out);
    if (tmp) cudaFreeAsync(tmp, st);
    return rc;
}

extern "C" int nb200_inpaint_blur(const float* mask, int B, int H, int W, float* out, void* stream) {
    NB_CHECK(mask && out, "null pointer");
    NB_CHECK(B > 0 && H > 0 && W > 0, "empty mask");
    cudaStream_t st = (cudaStream_t)stream;
    float* tmp = nullptr;
    NB_CUDA(cudaMallocAsync((void**)&tmp, (size_t)B * H * W * 4, st));
    const int rc = inpaint_blur(st, mask, B, H, W, 0, tmp, out);
    cudaFreeAsync(tmp, st);
    return rc;
}

extern "C" int nb200_light_inpaint(nb200_model* m, const float* x, const float* mask, int B, int H, int W, int mirror, float* out,
                                   void* stream) {
    NB_CHECK(m && x && mask && out, "null pointer");
    NB_CHECK(m->kind == NB200_MODEL_LIGHT_INPAINT_V1 && m->inp, "model is not inpaint.light_inpaint_v1");
    NB_CHECK(B > 0 && H > 0 && W > 0, "empty input");
    return light_inpaint_forward(m, (cudaStream_t)stream, x, mask, B, H, W, mirror, out);
}

// ---- test entry points of the waifu2x convolutions and the SE block: the weights are host fp32 tensors in the PyTorch layout,
// packed by the network's own packers and copied to a stream-ordered workspace that is freed behind the launch
static int upload_f32(cudaStream_t st, const std::vector<const std::vector<float>*>& parts, float** dev, std::vector<const float*>& ptrs) {
    std::vector<float> all;
    std::vector<size_t> off;
    for (const std::vector<float>* p : parts) {
        off.push_back(all.size());
        all.insert(all.end(), p->begin(), p->end());
        all.resize((all.size() + 63) & ~(size_t)63, 0.f);   // every part 256-byte aligned
    }
    NB_CUDA(cudaMallocAsync((void**)dev, all.size() * 4, st));
    const cudaError_t e = cudaMemcpyAsync(*dev, all.data(), all.size() * 4, cudaMemcpyHostToDevice, st);
    if (e != cudaSuccess) {
        cudaFreeAsync(*dev, st);
        return fail(std::string("upload_f32: ") + cudaGetErrorString(e));
    }
    ptrs.clear();
    for (size_t o : off) ptrs.push_back(*dev + o);
    return 0;
}

extern "C" int nb200_stem_conv_f16(const void* x, const float* w, const float* b, int cout, int cout_pad, int n, int Hi, int Wi,
                                   void* out, int ldo, void* stream) {
    NB_CHECK(x && w && b && out, "null pointer");
    NB_CHECK(cout > 0 && cout <= cout_pad && (cout_pad == 32 || cout_pad == 64), "cout_pad must be 32 or 64, cout at most cout_pad");
    NB_CHECK(n > 0 && Hi > 2 && Wi > 2, "input too small");
    std::vector<float> wv, bv;
    pack_stem_w(w, b, cout, cout_pad, wv, bv);
    cudaStream_t st = (cudaStream_t)stream;
    float* ws = nullptr;
    std::vector<const float*> p;
    if (upload_f32(st, {&wv, &bv}, &ws, p)) return 1;
    const int rc = stem_conv3x3(st, (const __half*)x, p[0], p[1], (__half*)out, n, Hi, Wi, cout_pad, ldo);
    cudaFreeAsync(ws, st);
    return rc;
}

extern "C" int nb200_tail_conv_f16(const void* x, const float* w, const float* b, int mode, int epi, int n, int Hi, int Wi, void* out,
                                   const void* z1, int z1H, int z1W, int clip, void* stream) {
    NB_CHECK(x && w && b && out && (epi == 0 || z1), "null pointer");
    NB_CHECK((mode == 0 && (epi == 0 || epi == 1)) || (mode == 1 && epi == 0), "unsupported (mode, epilogue)");
    const int Ho = mode == 0 ? Hi - 2 : 2 * Hi - 4, Wo = mode == 0 ? Wi - 2 : 2 * Wi - 4;
    NB_CHECK(n > 0 && Ho > 0 && Wo > 0, "input too small");
    NB_CHECK(epi == 0 || (z1H >= Ho + 40 && z1W >= Wo + 40), "z1 smaller than the output plus its 20-pixel crop");
    const std::vector<float> wv = pack_tail_w(w, mode == 1), bv(b, b + 3);
    cudaStream_t st = (cudaStream_t)stream;
    float* ws = nullptr;
    std::vector<const float*> p;
    if (upload_f32(st, {&wv, &bv}, &ws, p)) return 1;
    const int rc = tail_conv(st, mode, epi, (const __half*)x, p[0], p[1], (__half*)out, (const __half*)z1, n, Hi, Wi, z1H, z1W, clip);
    cudaFreeAsync(ws, st);
    return rc;
}

extern "C" int nb200_head_conv_f16(const void* x, const float* w, const float* b, int mode, int cin, int n, int Hi, int Wi, void* out,
                                   void* stream) {
    NB_CHECK(x && w && b && out, "null pointer");
    NB_CHECK((mode == 0 && cin == 128) || (mode == 1 && cin == 256), "unsupported (mode, input channels)");
    NB_CHECK(n > 0, "empty batch");
    const std::vector<float> wv = pack_head_w(w, mode == 1, cin), bv(b, b + 3);
    cudaStream_t st = (cudaStream_t)stream;
    float* ws = nullptr;
    std::vector<const float*> p;
    if (upload_f32(st, {&wv, &bv}, &ws, p)) return 1;
    const int rc = head_conv(st, mode, cin, (const __half*)x, p[0], p[1], (__half*)out, n, Hi, Wi);
    cudaFreeAsync(ws, st);
    return rc;
}

extern "C" int nb200_se_block_f16(void* x, const float* w1, const float* b1, const float* w2, const float* b2, int n, int H, int W, int C,
                                  void* stream) {
    NB_CHECK(x && w1 && b1 && w2 && b2, "null pointer");
    NB_CHECK(C == 64 || C == 128, "channels must be 64 or 128");
    NB_CHECK(n > 0 && n <= 65535 && H > 0 && W > 0, "bad geometry");
    const int R = C / 8;
    const std::vector<float> W1 = pack_se_w(w1, (size_t)R * C), B1 = pack_se_w(b1, R), W2 = pack_se_w(w2, (size_t)C * R),
                             B2 = pack_se_w(b2, C);
    const std::vector<float> scratch(se_partial_floats(n, H, W, C) + (size_t)n * C);   // partial sums, then the scales
    cudaStream_t st = (cudaStream_t)stream;
    float* ws = nullptr;
    std::vector<const float*> p;
    if (upload_f32(st, {&W1, &B1, &W2, &B2, &scratch}, &ws, p)) return 1;
    float* partial = const_cast<float*>(p[4]);
    const int rc = se_block(st, (__half*)x, n, H, W, C, p[0], p[1], p[2], p[3], partial, partial + se_partial_floats(n, H, W, C));
    cudaFreeAsync(ws, st);
    return rc;
}

// ---- test entry points of the learned stereo networks' input and output stages (the kernels a model forward launches between
// its window-attention blocks): the geometry is what the model's forward computes, the weights host fp32 tensors in the PyTorch
// layout.  Every check runs before the first CUDA call.
static int stereo_geometry(int B, int H, int W, int ph1, int pw1, int Hp, int Wp) {
    NB_CHECK(B > 0 && H > 0 && W > 0, "empty input");
    NB_CHECK(ph1 >= 0 && pw1 >= 0, "negative leading pad");
    NB_CHECK(ph1 + H <= Hp, "padded height < ph1 + H");
    NB_CHECK(pw1 + W <= Wp, "padded width < pw1 + W");
    return 0;
}

extern "C" int nb200_row_flow_prep_f16(const float* x, int B, int h, int w, int Hp, int Wt, void* out, void* stream) {
    NB_CHECK(x && out, "null pointer");
    if (stereo_geometry(B, h, w, 0, 0, Hp, 8 * Wt)) return 1;
    return rf_prep((cudaStream_t)stream, x, B, h, w, Hp, Wt, (__half*)out);
}

extern "C" int nb200_row_flow_last_conv_f32(const void* x, int B, int Hp, int Wt, int h, int w, const float* weight, const float* bias,
                                            float* delta, void* stream) {
    NB_CHECK(x && weight && bias && delta, "null pointer");
    if (stereo_geometry(B, h, w, 0, 0, Hp, 8 * Wt)) return 1;
    const std::vector<float> wv(weight, weight + 72);
    cudaStream_t st = (cudaStream_t)stream;
    float* ws = nullptr;
    std::vector<const float*> p;
    if (upload_f32(st, {&wv}, &ws, p)) return 1;
    const int rc = rf_last_conv(st, (const __half*)x, B, Hp, Wt, h, w, p[0], bias[0], delta);
    cudaFreeAsync(ws, st);
    return rc;
}

extern "C" int nb200_mlbw_prep_f16(const float* x, int B, int H, int W, int ph1, int pw1, int Hp, int Wt, int C1, const float* weight,
                                   const float* bias, void* out, void* stream) {
    NB_CHECK(x && weight && bias && out, "null pointer");
    if (stereo_geometry(B, H, W, ph1, pw1, Hp, 8 * Wt)) return 1;
    NB_CHECK(C1 > 0 && C1 <= 64, "C1 must be 1..64");
    const std::vector<float> wv(weight, weight + (size_t)C1 * 27), bv(bias, bias + C1);
    cudaStream_t st = (cudaStream_t)stream;
    float* ws = nullptr;
    std::vector<const float*> p;
    if (upload_f32(st, {&wv, &bv}, &ws, p)) return 1;
    const int rc = mlbw_prep(st, x, B, H, W, ph1, pw1, Hp, Wt, C1, p[0], p[1], (__half*)out);
    cudaFreeAsync(ws, st);
    return rc;
}

extern "C" int nb200_mlbw_out_f32(const void* t, const void* t0, int B, int H, int W, int ph1, int pw1, int Hp, int Wt, int C1, int L,
                                  const float* weight, const float* bias, float* delta, float* layer_weight, float* hole, void* stream) {
    NB_CHECK(t && t0 && weight && bias && delta && layer_weight, "null pointer");
    if (stereo_geometry(B, H, W, ph1, pw1, Hp, 8 * Wt)) return 1;
    NB_CHECK(C1 > 0 && C1 <= 64, "C1 must be 1..64");
    NB_CHECK(L == 2 || L == 4, "L must be 2 or 4 (the kernel's instantiations)");
    NB_CHECK(!hole || L == 2, "the hole head exists for L = 2 only");
    const int NO = 2 * L + (hole ? 1 : 0);
    // the kernel reads weights and biases as one [NO][C1][9] + [NO] block
    std::vector<float> all(weight, weight + (size_t)NO * C1 * 9);
    all.insert(all.end(), bias, bias + NO);
    cudaStream_t st = (cudaStream_t)stream;
    float* ws = nullptr;
    std::vector<const float*> p;
    if (upload_f32(st, {&all}, &ws, p)) return 1;
    const int rc = mlbw_out(st, (const __half*)t, (const __half*)t0, B, H, W, ph1, pw1, Hp, Wt, C1, L, p[0], p[0] + NO * C1 * 9, delta,
                            layer_weight, hole);
    cudaFreeAsync(ws, st);
    return rc;
}

extern "C" int nb200_depth_aa_minmax_f32(const float* x, long long n, float* minmax, void* stream) {
    NB_CHECK(x && minmax, "null pointer");
    NB_CHECK(n > 0, "empty input");
    return aa_minmax((cudaStream_t)stream, x, n, minmax);
}

extern "C" int nb200_depth_aa_prep_f16(const float* x, const float* minmax, int B, int H, int W, int ph1, int pw1, int Hh, int Wh,
                                       const float* weight, const float* bias, void* out, void* stream) {
    NB_CHECK(x && weight && bias && out, "null pointer");
    if (stereo_geometry(B, H, W, ph1, pw1, 2 * Hh, 2 * Wh)) return 1;
    const std::vector<float> wv(weight, weight + 128), bv(bias, bias + 32);
    cudaStream_t st = (cudaStream_t)stream;
    float* ws = nullptr;
    std::vector<const float*> p;
    if (upload_f32(st, {&wv, &bv}, &ws, p)) return 1;
    const int rc = aa_prep(st, x, minmax, B, H, W, ph1, pw1, Hh, Wh, p[0], p[1], (__half*)out);
    cudaFreeAsync(ws, st);
    return rc;
}

extern "C" int nb200_depth_aa_out_f32(const void* tok, const float* x, const float* minmax, int B, int H, int W, int ph1, int pw1, int Hh,
                                      int Wh, const float* weight, const float* bias, int clamp, float* out, void* stream) {
    NB_CHECK(tok && x && weight && bias && out, "null pointer");
    if (stereo_geometry(B, H, W, ph1, pw1, 2 * Hh, 2 * Wh)) return 1;
    const std::vector<float> wv(weight, weight + 128), bv(bias, bias + 4);
    cudaStream_t st = (cudaStream_t)stream;
    float* ws = nullptr;
    std::vector<const float*> p;
    if (upload_f32(st, {&wv, &bv}, &ws, p)) return 1;
    const int rc = aa_out(st, (const __half*)tok, x, minmax, B, H, W, ph1, pw1, Hh, Wh, p[0], p[1], clamp ? 1 : 0, out);
    cudaFreeAsync(ws, st);
    return rc;
}
