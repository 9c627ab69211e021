// iw3.depth_aa container (iw3/models/depth_aa.py:30-87, state_dict keys `proj_in.*`, `blocks.N.*`, `proj_out.*`): the learned
// anti-aliasing filter of Depth-Anything's output, and the test entry points of its input and output stages.  The
// window-attention blocks are wa_block.cu's.
#include "wa_block.h"
#include "depth_aa_kernels.h"

namespace nb200 {

struct NB_HIDDEN AaW : NetW {
    size_t win = 0, bin = 0;     // proj_in  fp32 [32][4], [32]
    size_t wout = 0, bout = 0;   // proj_out fp32 [4][32], [4]
    std::vector<WaBlockW> blk;
};

std::unique_ptr<NetW> pack_depth_aa(Packer& pk) {
    auto r = std::make_unique<AaW>();
    if (const float* w = pk.get("proj_in.weight", 32 * 4)) r->win = pk.add_f32(std::vector<float>(w, w + 128));
    if (const float* b = pk.get("proj_in.bias", 32)) r->bin = pk.add_f32(std::vector<float>(b, b + 32));
    if (const float* w = pk.get("proj_out.weight", 4 * 32)) r->wout = pk.add_f32(std::vector<float>(w, w + 128));
    if (const float* b = pk.get("proj_out.bias", 4)) r->bout = pk.add_f32(std::vector<float>(b, b + 4));
    for (int i = 0; i < 3; ++i) {
        const int pad = i != 1 ? 4 : 0;                                     // depth_aa.py:38-42: blocks 0 and 2 are shifted
        r->blk.push_back(pack_wa_block(pk, "blocks." + std::to_string(i) + ".", 32, 8, 2, pad, pad, ACT_LRELU01));
    }
    return r;
}

// DepthAA.forward (mode 0: eval clamp, mode 2: no clamp) / DepthAA.infer (mode 1: whole-tensor min/max normalisation, :46-55)
static int depth_aa_forward(nb200_model* m, const AaW& r, cudaStream_t st, const float* x, int B, int H, int W, int mode, float* out) {
    const int pad_w = 16 - W % 16, pad_h = 16 - H % 16;                     // always pads, also when already aligned (:61-62)
    const int pw1 = pad_w / 2, ph1 = pad_h / 2;
    const int Hh = (H + pad_h) / 2, Wh = (W + pad_w) / 2;
    float* mm;
    WaBufs wb;
    if (m->carve([&](Arena& a) {
            mm = a.take<float>(64);
            wa_plan(a, wb, B, Hh, Wh, 32);
        })) return 1;
    const float* mmp = nullptr;
    if (mode == 1) {
        if (aa_minmax(st, x, (long long)B * H * W, mm)) return 1;
        mmp = mm;
    }
    if (aa_prep(st, x, mmp, B, H, W, ph1, pw1, Hh, Wh, m->at<float>(r.win), m->at<float>(r.bin), wb.X)) return 1;
    for (const WaBlockW& b : r.blk)
        if (wa_block(st, m, b, wb, B, Hh, Wh)) return 1;
    return aa_out(st, wb.X, x, mmp, B, H, W, ph1, pw1, Hh, Wh, m->at<float>(r.wout), m->at<float>(r.bout), mode == 0, out);
}

}  // namespace nb200

using namespace nb200;

// DepthAA.forward / DepthAA.infer (iw3/models/depth_aa.py:46-87)
extern "C" int nb200_depth_aa(nb200_model* m, const float* x, int B, int H, int W, int mode, float* out, void* stream) {
    NB_CHECK(m && x && out, "null pointer");
    const AaW* r = net_as<AaW>(m);
    NB_CHECK(r, "model is not iw3.depth_aa");
    NB_CHECK(B > 0 && H > 0 && W > 0 && mode >= 0 && mode <= 2, "bad arguments");
    return depth_aa_forward(m, *r, (cudaStream_t)stream, x, B, H, W, mode, out);
}

// ---- test entry points of the input and output stages: the geometry is what the forward computes, the weights host fp32
// tensors in the PyTorch layout.  Every check runs before the first CUDA call.
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
    return with_uploaded(st, {&wv, &bv}, [&](const std::vector<const float*>& p) {
        return aa_prep(st, x, minmax, B, H, W, ph1, pw1, Hh, Wh, p[0], p[1], (__half*)out);
    });
}

extern "C" int nb200_depth_aa_out_f32(const void* tok, const float* x, const float* minmax, int B, int H, int W, int ph1, int pw1, int Hh,
                                      int Wh, const float* weight, const float* bias, int clamp, float* out, void* stream) {
    NB_CHECK(tok && x && weight && bias && out, "null pointer");
    if (stereo_geometry(B, H, W, ph1, pw1, 2 * Hh, 2 * Wh)) return 1;
    const std::vector<float> wv(weight, weight + 128), bv(bias, bias + 4);
    cudaStream_t st = (cudaStream_t)stream;
    return with_uploaded(st, {&wv, &bv}, [&](const std::vector<const float*>& p) {
        return aa_out(st, (const __half*)tok, x, minmax, B, H, W, ph1, pw1, Hh, Wh, p[0], p[1], clamp ? 1 : 0, out);
    });
}
