// sbs.mlbw container (iw3/models/mlbw.py:36-127; MLBW(num_layers = 2 | 4, base_dim = 32, small, hole_mask); state_dict keys
// `lv1_in.1.*`, `lv2.N.*`, `lv1_out.1.*`), its hole-mask post-processing and the test entry points of its input and output
// stages.  The window-attention blocks lv2.N are wa_block.cu's.  num_layers and hole_mask are read off lv1_out.1.bias (2 L
// outputs, + 1 hole logit with hole_mask, :70-74), `small` (two blocks, shifted along x only, :53-57) off the absence of lv2.2.
#include "wa_block.h"
#include "mlbw_kernels.h"

namespace nb200 {

struct NB_HIDDEN MlW : NetW {
    int L = 2, C = 64, C1 = 8;
    bool hole = false;                              // hole_mask head: lv1_out has 2 L + 1 outputs (sbs.mask_mlbw_l2)
    size_t win = 0, bin = 0, wout = 0, bout = 0;   // fp32 conv (1, 9) weights as stored
    std::vector<WaBlockW> blk;
};

std::unique_ptr<NetW> pack_mlbw(Packer& pk) {
    auto r = std::make_unique<MlW>();
    auto it = pk.src.find("lv1_out.1.bias");
    // upstream registers one hole_mask model, sbs.mask_mlbw_l2 (num_layers 2): 5 outputs
    if (it == pk.src.end() || (it->second.numel != 4 && it->second.numel != 8 && it->second.numel != 5)) {
        pk.err = "sbs.mlbw: lv1_out.1.bias must have 2 * num_layers elements (num_layers 2 or 4), or 5 for the hole_mask model "
                 "(sbs.mask_mlbw_l2: num_layers 2 + 1 hole logit)";
        return r;
    }
    r->hole = it->second.numel == 5;
    r->L = (int)it->second.numel / 2;
    r->C = 32 * r->L;
    r->C1 = r->C / 8;
    const bool small = pk.src.find("lv2.2.conv_mlp.0.bias") == pk.src.end();
    const int C = r->C, C1 = r->C1, L = r->L, NO = 2 * L + (r->hole ? 1 : 0);
    if (const float* w = pk.get("lv1_in.1.weight", (int64_t)C1 * 27)) r->win = pk.add_f32(std::vector<float>(w, w + C1 * 27));
    if (const float* b = pk.get("lv1_in.1.bias", C1)) r->bin = pk.add_f32(std::vector<float>(b, b + C1));
    if (const float* w = pk.get("lv1_out.1.weight", (int64_t)NO * C1 * 9)) r->wout = pk.add_f32(std::vector<float>(w, w + NO * C1 * 9));
    if (const float* b = pk.get("lv1_out.1.bias", NO)) r->bout = pk.add_f32(std::vector<float>(b, b + NO));
    for (int i = 0; i < (small ? 2 : 4); ++i) {
        const bool shifted = i % 2 == 0;                                    // :53-64
        r->blk.push_back(pack_wa_block(pk, "lv2." + std::to_string(i) + ".", C, 4, L, shifted && !small ? 2 : 0, shifted ? 2 : 0, ACT_NONE));
    }
    return r;
}

// MLBW._forward in eval mode (:96-127): x fp32 [B][3][h][w] -> delta [B][L][h][w], layer_weight [B][L][h][w] (softmax over L) and,
// for a hole_mask model, the hole logits [B][1][h][w] (hole must then be non-null)
static int mlbw_forward(nb200_model* m, const MlW& r, cudaStream_t st, const float* x, int B, int h, int w, float* delta, float* lw,
                        float* hole) {
    const int C = r.C;
    const int pad_w = 32 - w % 32, pad_h = 4 - h % 4;                       // _calc_pad :72-88 (always pads)
    const int pw1 = pad_w / 2, ph1 = pad_h / 2;
    const int Hp = h + pad_h, Wt = (w + pad_w) / 8;
    const long long M = (long long)B * Hp * Wt;
    __half* T0;
    WaBufs wb;
    if (m->carve([&](Arena& a) {
            T0 = a.take<__half>((size_t)M * C);
            wa_plan(a, wb, B, Hp, Wt, C);
        })) return 1;
    if (mlbw_prep(st, x, B, h, w, ph1, pw1, Hp, Wt, r.C1, m->at<float>(r.win), m->at<float>(r.bin), T0)) return 1;
    NB_CUDA(cudaMemcpyAsync(wb.X, T0, (size_t)M * C * 2, cudaMemcpyDeviceToDevice, st));
    for (const WaBlockW& b : r.blk)
        if (wa_block(st, m, b, wb, B, Hp, Wt)) return 1;
    return mlbw_out(st, wb.X, T0, B, h, w, ph1, pw1, Hp, Wt, r.C1, r.L, m->at<float>(r.wout), m->at<float>(r.bout), delta, lw,
                    r.hole ? hole : nullptr);
}

}  // namespace nb200

using namespace nb200;

// MLBW.forward with delta_output=True (iw3/models/mlbw.py:96-127,237-245): the x components of the L flow layers and their weights
extern "C" int nb200_mlbw_delta(nb200_model* m, const float* x, int B, int h, int w, float* delta, float* layer_weight, void* stream) {
    NB_CHECK(m && x && delta && layer_weight, "null pointer");
    const MlW* r = net_as<MlW>(m);
    NB_CHECK(r, "model is not sbs.mlbw");
    NB_CHECK(!r->hole, "this sbs.mlbw has a hole_mask head (sbs.mask_mlbw_l2): use nb200_mlbw_delta_hole");
    NB_CHECK(B > 0 && h > 0 && w > 0, "empty input");
    return mlbw_forward(m, *r, (cudaStream_t)stream, x, B, h, w, delta, layer_weight, nullptr);
}
extern "C" int nb200_mlbw_num_layers(const nb200_model* m) {
    const MlW* r = net_as<MlW>(m);
    return r ? r->L : 0;
}
extern "C" int nb200_mlbw_has_hole_mask(const nb200_model* m) {
    const MlW* r = net_as<MlW>(m);
    return r && r->hole ? 1 : 0;
}

// MLBW._forward_delta_only of a hole_mask model (mlbw.py:232-240): delta, layer_weight and the hole logits
extern "C" int nb200_mlbw_delta_hole(nb200_model* m, const float* x, int B, int h, int w, float* delta, float* layer_weight,
                                     float* hole_logits, void* stream) {
    NB_CHECK(m && x && delta && layer_weight && hole_logits, "null pointer");
    const MlW* r = net_as<MlW>(m);
    NB_CHECK(r, "model is not sbs.mlbw");
    NB_CHECK(r->hole, "this sbs.mlbw has no hole_mask head: use nb200_mlbw_delta");
    NB_CHECK(B > 0 && h > 0 && w > 0, "empty input");
    return mlbw_forward(m, *r, (cudaStream_t)stream, x, B, h, w, delta, layer_weight, hole_logits);
}

// postprocess_hole_mask (iw3/backward_warp.py:382-393), steps 1-3: closing, align-corners resize, sigmoid > threshold
extern "C" int nb200_hole_mask(const float* logits, int B, int h, int w, int H, int W, float threshold, int mirror, float* out,
                               void* stream) {
    NB_CHECK(logits && out, "null pointer");
    NB_CHECK(B > 0 && h > 0 && w > 0 && H > 0 && W > 0, "empty mask");
    return hole_mask((cudaStream_t)stream, logits, B, h, w, H, W, threshold, mirror ? 1 : 0, out);
}

// ---- test entry points of the input and output stages: the geometry is what the forward computes, the weights host fp32
// tensors in the PyTorch layout.  Every check runs before the first CUDA call.
extern "C" int nb200_mlbw_prep_f16(const float* x, int B, int H, int W, int ph1, int pw1, int Hp, int Wt, int C1, const float* weight,
                                   const float* bias, void* out, void* stream) {
    NB_CHECK(x && weight && bias && out, "null pointer");
    if (stereo_geometry(B, H, W, ph1, pw1, Hp, 8 * Wt)) return 1;
    NB_CHECK(C1 > 0 && C1 <= 64, "C1 must be 1..64");
    const std::vector<float> wv(weight, weight + (size_t)C1 * 27), bv(bias, bias + C1);
    cudaStream_t st = (cudaStream_t)stream;
    return with_uploaded(st, {&wv, &bv}, [&](const std::vector<const float*>& p) {
        return mlbw_prep(st, x, B, H, W, ph1, pw1, Hp, Wt, C1, p[0], p[1], (__half*)out);
    });
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
    return with_uploaded(st, {&all}, [&](const std::vector<const float*>& p) {
        return mlbw_out(st, (const __half*)t, (const __half*)t0, B, H, W, ph1, pw1, Hp, Wt, C1, L, p[0], p[0] + NO * C1 * 9, delta,
                        layer_weight, hole);
    });
}
