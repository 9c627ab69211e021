// sbs.row_flow_v3 container (iw3/models/row_flow_v3.py:32-68, state_dict keys `blocks.*`, `last_layer.1.*`): the learned
// delta network of iw3's default stereo method, and the test entry points of its input and output stages.  The two
// window-attention blocks are wa_block.cu's.
#include "wa_block.h"
#include "rowflow_kernels.h"

namespace nb200 {

struct NB_HIDDEN RfW : NetW {
    Lin c0;            // Conv2d(24, 64, 1) as a Linear over K = 32 (zero padded)
    std::vector<WaBlockW> blk;
    size_t lastw = 0;  // fp32 [8][3][3]
    float lastb = 0.f;
};

std::unique_ptr<NetW> pack_row_flow(Packer& pk) {
    auto r = std::make_unique<RfW>();
    r->c0 = pack_conv(pk, "blocks.0", 64, 24, 1, 1, /*cin_pad=*/32);
    r->blk.push_back(pack_wa_block(pk, "blocks.1.", 64, 4, 2, 0, 0, ACT_LRELU01));     // row_flow_v3.py:41-45
    r->blk.push_back(pack_wa_block(pk, "blocks.2.", 64, 3, 2, 0, 0, ACT_LRELU01));
    if (const float* w = pk.get("last_layer.1.weight", 72)) r->lastw = pk.add_f32(std::vector<float>(w, w + 72));
    if (const float* b = pk.get("last_layer.1.bias", 1)) r->lastb = b[0];
    pk.mark("delta_scale");
    return r;
}

// RowFlowV3._forward (delta_output mode): x fp32 [B][3][h][w] (depth, divergence feature, convergence feature) -> delta [B][1][h][w]
static int row_flow_forward(nb200_model* m, const RfW& r, cudaStream_t st, const float* x, int B, int h, int w, float* delta) {
    const int pad1 = 96 - w % 96, pad2 = 12 - h % 12;          // row_flow_v3.py:59-60 (always pads, also when already aligned)
    const int Hp = h + pad2, Wp = w + pad1, Wt = Wp / 8;
    const long long M = (long long)B * Hp * Wt;
    __half* A0;
    WaBufs wb;
    if (m->carve([&](Arena& a) {
            A0 = a.take<__half>((size_t)M * 32);
            wa_plan(a, wb, B, Hp, Wt, 64);
        })) return 1;
    if (rf_prep(st, x, B, h, w, Hp, Wt, A0)) return 1;
    if (linear_flat(st, m, r.c0, A0, M, 32, wb.X, 64, ACT_NONE)) return 1;
    for (const WaBlockW& b : r.blk)
        if (wa_block(st, m, b, wb, B, Hp, Wt)) return 1;
    return rf_last_conv(st, wb.X, B, Hp, Wt, h, w, m->at<float>(r.lastw), r.lastb, delta);
}

}  // namespace nb200

using namespace nb200;

// RowFlowV3.forward with delta_output=True (iw3/models/row_flow_v3.py:111-116) - the x component of the returned delta
extern "C" int nb200_row_flow_delta(nb200_model* m, const float* x, int B, int h, int w, float* delta, void* stream) {
    NB_CHECK(m && x && delta, "null pointer");
    const RfW* r = net_as<RfW>(m);
    NB_CHECK(r, "model is not sbs.row_flow_v3");
    NB_CHECK(B > 0 && h > 0 && w > 0, "bad shape");
    return row_flow_forward(m, *r, (cudaStream_t)stream, x, B, h, w, delta);
}

// ---- test entry points of the input and output stages: the geometry is what the forward computes, the weights host fp32
// tensors in the PyTorch layout.  Every check runs before the first CUDA call.
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
    return with_uploaded(st, {&wv}, [&](const std::vector<const float*>& p) {
        return rf_last_conv(st, (const __half*)x, B, Hp, Wt, h, w, p[0], bias[0], delta);
    });
}
