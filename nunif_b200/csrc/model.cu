// The model handle: the kind table that packs each NB200_MODEL_* network, create / destroy / info, nb200_model_forward with
// its CUDA-graph cache, the whole-image tiled renders and the debug tap.  Also the packers and forward helpers that several
// network families share (model.h).  Each family's weights, forward and entry points are in its own file (swin_model.cu,
// cunet_model.cu, ...).
#include "model.h"
#include "gemm.h"

namespace nb200 {

extern int g_tune[16];                 // gemm.cu (nb200_tune_set)
extern std::atomic<int> g_tune_epoch;  // gemm.cu: bumped by every nb200_tune_set (captured graphs bake the knobs in)

// ---------------------------------------------------------------------------------------------
// shared packers
// ---------------------------------------------------------------------------------------------
// Linear: weight [N][K]
Lin pack_linear(Packer& pk, const std::string& name, int N, int K, int n_pad) {
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
Lin pack_linear_pixshuf2(Packer& pk, const std::string& name, int cout, int K, const std::string& skip, int Ks) {
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
Lin pack_conv(Packer& pk, const std::string& name, int cout, int cin, int kh, int kw, int cin_pad, int cout_pad) {
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
// first 3x3 conv from 3 channels: Conv2d weight [cout][3][3][3] and bias [cout] -> wv = fp32 [27][cout_pad] with
// k = (ky*3+kx)*3 + ci, then the mma.sync B fragments; bv = bias [cout_pad] (both zero padded)
void pack_stem_w(const float* w, const float* b, int cout, int cout_pad, std::vector<float>& wv, std::vector<float>& bv) {
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
Lin pack_stem(Packer& pk, const std::string& name, int cout, int cout_pad) {
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
size_t pack_vec_f32(Packer& pk, const std::string& name, int n) {
    const float* v = pk.get(name, n);
    if (!v) return 0;
    return pk.add_f32(std::vector<float>(v, v + n));
}

// ---------------------------------------------------------------------------------------------
// forward helpers
// ---------------------------------------------------------------------------------------------
// split > 0: the N outputs are written as N/split dense [M][split] planes (OUT_SPLIT); a_planes > 1: A is given as planes
int linear_flat(cudaStream_t st, const nb200_model* m, const Lin& l, const __half* A, long long M, int lda, __half* out, int ldo,
                int act, const __half* res, int ldr, int split, int a_planes) {
    ConvGemm g;
    g.A = A; g.B = 1; g.Hi = 1; g.Wi = (int)M; g.Ci = lda; g.Cin = l.K / a_planes; g.kind = CG_LINEAR_FLAT;
    g.a_planes = a_planes; g.a_plane_stride = (long long)M * lda;
    g.Wt = m->at<__half>(l.w); g.N = l.N; g.bias = m->at<float>(l.b); g.act = act; g.out = out; g.ldo = ldo;
    g.res = res; g.ldr = ldr;
    if (split) { g.out_mode = OUT_SPLIT; g.cout = split; g.split_stride = (long long)M * split; g.ldo = split; }
    return conv_gemm(st, g);
}

// debug tap (nb200_debug_tap): stage `g_tap_id` of the next ZoeDepth, light_inpaint_v1 or TransNetV2 forward is copied to
// `g_tap_buf` (ZoeDepth ids 0..15 in zoe_model.cu; light_inpaint_v1 ids 100..173, table in DESIGN.md §5; TransNetV2 ids
// 200..205 in transnet_model.cu); the forward warp's kernel writes id 300 itself (warp_forward.cu)
static int g_tap_id = -1;
static void* g_tap_buf = nullptr;
static size_t g_tap_cap = 0;
int tap_copy(cudaStream_t st, int id, const void* src, size_t bytes) {
    if (id != g_tap_id || !g_tap_buf) return 0;
    NB_CHECK(bytes <= g_tap_cap, "debug tap buffer too small: need " + std::to_string(bytes) + " bytes");
    NB_CUDA(cudaMemcpyAsync(g_tap_buf, src, bytes, cudaMemcpyDeviceToDevice, st));
    return 0;
}

int debug_tap_target(int id, size_t bytes, void** buf) {
    *buf = nullptr;
    if (id != g_tap_id || !g_tap_buf) return 0;
    NB_CHECK(bytes <= g_tap_cap, "debug tap buffer too small: need " + std::to_string(bytes) + " bytes");
    *buf = g_tap_buf;
    return 0;
}

int upload_f32(cudaStream_t st, const std::vector<const std::vector<float>*>& parts, float** dev, std::vector<const float*>& ptrs) {
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

// ---------------------------------------------------------------------------------------------
// the kind table: one row per NB200_MODEL_* value
// ---------------------------------------------------------------------------------------------
struct ModelKind {
    int kind;
    std::unique_ptr<NetW> (*pack)(Packer& pk);
    int scale, offset, blend;              // nb200_model_info
    ImageForward forward;                  // nb200_model_forward and the tiled renders; null: not an image-to-image model
    int (*after_upload)(nb200_model* m);   // device-side setup once the weights are on the device, or null
};

static const ModelKind KINDS[] = {
    {NB200_MODEL_UPCUNET, [](Packer& pk) { return pack_cunet(pk, true); }, 2, 36, 0, cunet_forward, nullptr},            // cunet.py:144
    {NB200_MODEL_CUNET, [](Packer& pk) { return pack_cunet(pk, false); }, 1, 28, 0, cunet_forward, nullptr},             // cunet.py:178
    {NB200_MODEL_SWIN_UNET_1X, [](Packer& pk) { return pack_swin(pk, 1); }, 1, 8, 4, swin_forward, swin_build_bias_frags},    // swin_unet.py:213
    {NB200_MODEL_SWIN_UNET_2X, [](Packer& pk) { return pack_swin(pk, 2); }, 2, 16, 8, swin_forward, swin_build_bias_frags},   // :234
    {NB200_MODEL_SWIN_UNET_4X, [](Packer& pk) { return pack_swin(pk, 4); }, 4, 32, 16, swin_forward, swin_build_bias_frags},  // :267
    {NB200_MODEL_UPCONV_7, [](Packer& pk) { return pack_legacy(pk, true); }, 2, 14, 0, legacy_forward, nullptr},         // upconv_7.py:11
    {NB200_MODEL_VGG_7, [](Packer& pk) { return pack_legacy(pk, false); }, 1, 7, 0, legacy_forward, nullptr},            // vgg_7.py:11
    {NB200_MODEL_DEPTH_ANYTHING_V2_S, [](Packer& pk) { return pack_depth_anything(pk, 0, false); }, 1, 0, 0, nullptr, nullptr},
    {NB200_MODEL_DEPTH_ANYTHING_V2_B, [](Packer& pk) { return pack_depth_anything(pk, 1, false); }, 1, 0, 0, nullptr, nullptr},
    {NB200_MODEL_DEPTH_ANYTHING_V2_L, [](Packer& pk) { return pack_depth_anything(pk, 2, false); }, 1, 0, 0, nullptr, nullptr},
    // depth_anything_model.py:36-38
    {NB200_MODEL_DEPTH_ANYTHING_V1_S, [](Packer& pk) { return pack_depth_anything(pk, 0, true); }, 1, 0, 0, nullptr, nullptr},
    {NB200_MODEL_DEPTH_ANYTHING_V1_B, [](Packer& pk) { return pack_depth_anything(pk, 1, true); }, 1, 0, 0, nullptr, nullptr},
    {NB200_MODEL_DEPTH_ANYTHING_V1_L, [](Packer& pk) { return pack_depth_anything(pk, 2, true); }, 1, 0, 0, nullptr, nullptr},
    {NB200_MODEL_ZOEDEPTH_N, pack_zoedepth, 1, 0, 0, nullptr, nullptr},                                                   // zoedepth_model.py:151-157
    {NB200_MODEL_ZOEDEPTH_ANY_N, [](Packer& pk) { return pack_zoedepth_any(pk, false); }, 1, 0, 0, nullptr, nullptr},    // zoedepth_model.py:20
    {NB200_MODEL_ZOEDEPTH_ANY_K, [](Packer& pk) { return pack_zoedepth_any(pk, true); }, 1, 0, 0, nullptr, nullptr},
    {NB200_MODEL_DEPTH_AA, pack_depth_aa, 1, 0, 0, nullptr, nullptr},                                                     // depth_aa.py:34
    {NB200_MODEL_ROW_FLOW_V3, pack_row_flow, 1, 32, 4, nullptr, nullptr},                                                 // row_flow_v3.py:37
    {NB200_MODEL_ROW_FLOW_V2, pack_row_flow_v2, 1, 28, 4, nullptr, nullptr},                                              // row_flow_v2.py:14
    {NB200_MODEL_MLBW, pack_mlbw, 1, 32, 4, nullptr, nullptr},                                                            // mlbw.py:41
    {NB200_MODEL_LIGHT_INPAINT_V1, pack_light_inpaint, 1, 16, 8, nullptr, nullptr},                                       // light_inpaint_v1.py:56
    {NB200_MODEL_SOD_V1, pack_sod, 1, 0, 0, nullptr, nullptr},                                                            // sod_v1.py:15
    {NB200_MODEL_TRANSNET_V2, pack_transnet, 1, 0, 0, nullptr, nullptr},                                                  // transnetv2.py:7-47
};

static const ModelKind* model_kind(int kind) {
    for (const ModelKind& k : KINDS)
        if (k.kind == kind) return &k;
    return nullptr;
}

}  // namespace nb200

using namespace nb200;

// ---------------------------------------------------------------------------------------------
// C ABI
// ---------------------------------------------------------------------------------------------
extern "C" int nb200_model_create(int kind, int n_tensors, const char* const* names, const float* const* data,
                                  const int64_t* numel, int no_clip, nb200_model** out) {
    NB_CHECK(out && names && data && numel, "null pointer");
    const ModelKind* k = model_kind(kind);
    NB_CHECK(k, "unknown model kind");
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
    m->scale = k->scale;
    m->offset = k->offset;
    m->blend = k->blend;
    m->net = k->pack(pk);
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
    // the family's device-side setup (Swin: the bias fragments), then synchronised, since forwards may run on non-blocking
    // streams
    int rc = 0;
    if (e == cudaSuccess && k->after_upload) rc = k->after_upload(m);
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

// the output geometry of an image-to-image handle; every image entry point calls this before its first CUDA call
static int model_out_geometry(const nb200_model* m, int tile_size, int down, int* scale, int* offset, int* blend, int* S) {
    NB_CHECK(model_kind(m->kind)->forward, "not an image-to-image model");
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
    const ImageForward forward = model_kind(m->kind)->forward;
    auto eager = [&]() { return forward(m, st, (const __half*)x, n, tile_size, downscale, z); };
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
