// iw3.sod_v1 container (iw3/models/sod_v1.py; state_dict keys `u2netp.stageN.rebnconv*.conv_s1.*`, `.bn_s1.*`,
// `u2netp.side1..6.*`, `u2netp.outconv.*`) and its entry point; the forward is sod.cu's.  Every REBNCONV's BatchNorm is folded
// into its conv in fp32, as U2NETP.fuse() does with torch.nn.utils.fuse_conv_bn_eval, then rounded to fp16 (autocast runs the
// fused conv with fp16 weights and bias).
#include "model.h"
#include "sod_kernels.h"
#include <cmath>

namespace nb200 {

struct NB_HIDDEN SodNet : NetW {
    SodW w;
};

std::unique_ptr<NetW> pack_sod(Packer& pk) {
    auto net = std::make_unique<SodNet>();
    SodW* r = &net->w;
    sod_layer_list(r->convs);
    const float eps = 1e-5f;   // BatchNorm2d default
    for (SodConv& c : r->convs) {
        const std::string p = c.name;
        const int K = c.cin * 9;
        const float* w = pk.get(p + ".conv_s1.weight", (int64_t)c.cout * K);
        const float* b = pk.get(p + ".conv_s1.bias", c.cout);
        const float* g = pk.get(p + ".bn_s1.weight", c.cout);
        const float* be = pk.get(p + ".bn_s1.bias", c.cout);
        const float* rm = pk.get(p + ".bn_s1.running_mean", c.cout);
        const float* rv = pk.get(p + ".bn_s1.running_var", c.cout);
        pk.mark(p + ".bn_s1.num_batches_tracked");
        if (!w || !b || !g || !be || !rm || !rv) return net;
        std::vector<float> wt((size_t)c.cout * 9 * c.cin_pad, 0.f), bias(c.cout);
        for (int co = 0; co < c.cout; ++co) {
            // fuse_conv_bn_eval: w * (gamma * rsqrt(var + eps)), (b - mean) * rsqrt(var + eps) * gamma + beta
            const float rs = 1.f / std::sqrt(rv[co] + eps);
            const float s = g[co] * rs;
            for (int ci = 0; ci < c.cin; ++ci)
                for (int tap = 0; tap < 9; ++tap)
                    wt[((size_t)co * 9 + tap) * c.cin_pad + ci] = w[((size_t)co * c.cin + ci) * 9 + tap] * s;
            bias[co] = round_f16((b[co] - rm[co]) * rs * g[co] + be[co]);
        }
        c.w = pk.add_f16(wt);
        c.b = pk.add_f32(bias);
    }
    std::vector<float> side(6 * 9 * 64 + 6);
    for (int l = 0; l < 6; ++l) {
        const std::string p = "u2netp.side" + std::to_string(l + 1);
        const float* w = pk.get(p + ".weight", 64 * 9);
        const float* b = pk.get(p + ".bias", 1);
        if (!w || !b) return net;
        for (int ci = 0; ci < 64; ++ci)
            for (int tap = 0; tap < 9; ++tap) side[(l * 9 + tap) * 64 + ci] = round_f16(w[ci * 9 + tap]);
        side[6 * 9 * 64 + l] = round_f16(b[0]);
    }
    const float* ow = pk.get("u2netp.outconv.weight", 6);
    const float* ob = pk.get("u2netp.outconv.bias", 1);
    if (!ow || !ob) return net;
    std::vector<float> head(7);
    for (int l = 0; l < 6; ++l) head[l] = round_f16(ow[l]);
    head[6] = round_f16(ob[0]);
    r->side = pk.add_f32(side);
    r->head = pk.add_f32(head);
    return net;
}

}  // namespace nb200

using namespace nb200;

// SODV1.infer (iw3/models/sod_v1.py:47-54) under autocast: sigmoid(U2NETP(cat(rgb, d, d ** 0.5, d ** 2))) at 192 x 192
extern "C" int nb200_sod_forward(nb200_model* m, const float* rgb, int B, int H, int W, const float* depth, int h, int w,
                                 float* saliency, float* depth192, void* stream) {
    NB_CHECK(m && rgb && depth && saliency && depth192, "null pointer");
    const SodNet* net = net_as<SodNet>(m);
    NB_CHECK(net, "model is not iw3.sod_v1");
    NB_CHECK(B > 0 && H > 0 && W > 0 && h > 0 && w > 0, "bad shape");
    return sod_forward((cudaStream_t)stream, m->blob, net->w, rgb, B, H, W, depth, h, w, saliency, depth192);
}
