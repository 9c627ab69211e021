// The model handle (nb200_model) and what the network families' source files share: the state_dict packer, the shared
// packers, the workspace arena and the family entry points that the kind table in model.cu calls.  Host code only.
// The functions declared here, and the families' weights types, have hidden visibility (NB_HIDDEN), so that they do not
// add to the library's dynamic symbol table.
#pragma once
#include "common.cuh"
#include "../../include/nunif_b200.h"
#include <map>
#include <memory>
#include <string>
#include <tuple>
#include <vector>
#include <cstring>

#define NB_HIDDEN __attribute__((visibility("hidden")))

namespace nb200 {

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
NB_HIDDEN Lin pack_linear(Packer& pk, const std::string& name, int N, int K, int n_pad = 0);
// Linear followed by pixel_shuffle(2): rows reordered so n = (dy*2+dx)*cout + co  (F.pixel_shuffle: c*4 + dy*2 + dx)
// With `skip`, the Linear [cout][Ks] of the skip tensor that is added to the result is appended to every row (the GEMM's
// second A operand, ConvGemm::A2): row n = [up row | skip row co], K + Ks columns, bias = both biases summed in fp32.
NB_HIDDEN Lin pack_linear_pixshuf2(Packer& pk, const std::string& name, int cout, int K, const std::string& skip = "", int Ks = 0);
// Conv2d weight [Cout][Cin][kh][kw] -> [Cout][kh][kw][cin_pad]
NB_HIDDEN Lin pack_conv(Packer& pk, const std::string& name, int cout, int cin, int kh, int kw, int cin_pad = 0, int cout_pad = 0);
// first 3x3 conv from 3 channels (the stem kernel's fp32 weights and their mma.sync B fragments)
NB_HIDDEN void pack_stem_w(const float* w, const float* b, int cout, int cout_pad, std::vector<float>& wv, std::vector<float>& bv);
NB_HIDDEN Lin pack_stem(Packer& pk, const std::string& name, int cout, int cout_pad);
// a tensor as stored, fp32
NB_HIDDEN size_t pack_vec_f32(Packer& pk, const std::string& name, int n);

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

// The packed weights of one network family: each family's weights struct derives from this, and a handle owns exactly one.
struct NetW {
    virtual ~NetW() = default;
};

}  // namespace nb200

struct nb200_model {
    int kind = 0, no_clip = 0, device = 0;
    int scale = 1, offset = 0, blend = 0;
    uint8_t* blob = nullptr;
    size_t blob_bytes = 0;
    std::unique_ptr<nb200::NetW> net;      // the network's weights (offsets into blob) and host-side state
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
        nb200::Arena size;
        plan(size);
        if (ensure_ws(size.off + 4096)) return 1;
        nb200::Arena a{ws};
        plan(a);
        return 0;
    }
};

namespace nb200 {

// The weights of a handle of family W, or null for a null handle or one of another family.
template <class W>
W* net_as(const nb200_model* m) {
    return m ? dynamic_cast<W*>(m->net.get()) : nullptr;
}

// ---------------------------------------------------------------------------------------------
// forward helpers
// ---------------------------------------------------------------------------------------------
// split > 0: the N outputs are written as N/split dense [M][split] planes (OUT_SPLIT); a_planes > 1: A is given as planes
NB_HIDDEN int linear_flat(cudaStream_t st, const nb200_model* m, const Lin& l, const __half* A, long long M, int lda, __half* out,
                          int ldo, int act, const __half* res = nullptr, int ldr = 0, int split = 0, int a_planes = 1);

// debug tap (nb200_debug_tap): copies `bytes` of `src` to the armed buffer when stage `id` is the armed one
NB_HIDDEN int tap_copy(cudaStream_t st, int id, const void* src, size_t bytes);

// The test entry points of single stages take host fp32 weights: with_uploaded copies `parts` to one stream-ordered device
// block (each part 256-byte aligned), calls launch(pointers to the parts) and frees the block behind it, also when the
// launch fails.
NB_HIDDEN int upload_f32(cudaStream_t st, const std::vector<const std::vector<float>*>& parts, float** dev,
                         std::vector<const float*>& ptrs);
template <typename F>
int with_uploaded(cudaStream_t st, const std::vector<const std::vector<float>*>& parts, F launch) {
    float* dev = nullptr;
    std::vector<const float*> p;
    if (upload_f32(st, parts, &dev, p)) return 1;
    const int rc = launch(p);
    cudaFreeAsync(dev, st);
    return rc;
}

// ---------------------------------------------------------------------------------------------
// the network families (one source file each): the packers and forwards that the kind table in model.cu names
// ---------------------------------------------------------------------------------------------
// an image-to-image forward: x [n][T][T][8] fp16 tiles -> z [n][3][S][S] (fp16, or fp32 when downscaled)
using ImageForward = int (*)(nb200_model* m, cudaStream_t st, const __half* x, int n, int T, int down, void* z);

NB_HIDDEN std::unique_ptr<NetW> pack_swin(Packer& pk, int r);                                 // swin_model.cu
NB_HIDDEN int swin_forward(nb200_model* m, cudaStream_t st, const __half* x, int n, int T, int down, void* z);
NB_HIDDEN int swin_build_bias_frags(nb200_model* m);
NB_HIDDEN std::unique_ptr<NetW> pack_cunet(Packer& pk, bool up);                              // cunet_model.cu
NB_HIDDEN int cunet_forward(nb200_model* m, cudaStream_t st, const __half* x, int n, int T, int down, void* z);
NB_HIDDEN std::unique_ptr<NetW> pack_legacy(Packer& pk, bool up);                             // legacy_model.cu
NB_HIDDEN int legacy_forward(nb200_model* m, cudaStream_t st, const __half* x, int n, int T, int down, void* z);
NB_HIDDEN std::unique_ptr<NetW> pack_depth_anything(Packer& pk, int encoder, bool v1);        // depth_model.cu
NB_HIDDEN std::unique_ptr<NetW> pack_zoedepth(Packer& pk);                                    // zoe_model.cu
NB_HIDDEN std::unique_ptr<NetW> pack_zoedepth_any(Packer& pk, bool normed);
NB_HIDDEN std::unique_ptr<NetW> pack_row_flow(Packer& pk);                                    // rowflow_model.cu
NB_HIDDEN std::unique_ptr<NetW> pack_row_flow_v2(Packer& pk);                                 // rowflow_v2_model.cu
NB_HIDDEN std::unique_ptr<NetW> pack_depth_aa(Packer& pk);                                    // depth_aa_model.cu
NB_HIDDEN std::unique_ptr<NetW> pack_mlbw(Packer& pk);                                        // mlbw_model.cu
NB_HIDDEN std::unique_ptr<NetW> pack_light_inpaint(Packer& pk);                               // inpaint_model.cu
NB_HIDDEN std::unique_ptr<NetW> pack_sod(Packer& pk);                                         // sod_model.cu
NB_HIDDEN std::unique_ptr<NetW> pack_transnet(Packer& pk);                                    // transnet_model.cu

}  // namespace nb200
