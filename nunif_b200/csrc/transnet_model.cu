// TransNetV2 container, forward and entry point (nunif/utils/transnetv2.py, defaults F=16 L=3 S=2 D=1024).
//
// Activations are NHWC fp16 with the frames of all windows as images, [B*T][h][w][C].  Per DilatedDCNNV2 block:
//   * one CG_CONV3 GEMM runs the four (1,3,3) convs (they read the same input), N = 8F: branch k in channels [2Fk, 2Fk+2F);
//   * one CG_TCONV3 GEMM per branch runs the (3,1,1) conv with dilation d over [B][T][h*w][2F] (its slice of the 8F
//     buffer), with the block's BatchNorm folded into weight and bias; its epilogue writes channels [Fk, Fk+F) of the 4F
//     block output (so torch.cat is free) and applies the ReLU of the first block.  The time padding of each window is the
//     tensor map's out-of-bounds zero fill, so windows never see each other.
// The stack tail writes the pooled output and its channel means; the third stack's output lands directly in columns
// [256, 4864) of the fc1 input row, in the (h, w, c) order of the reference's flatten.
#include "model.h"
#include "gemm.h"
#include "transnet_kernels.h"
#include <cmath>

namespace nb200 {

struct NB_HIDDEN TnNet : NetW {
    TnW w;
};

static const int TN_DIL[4] = {1, 2, 4, 8};

std::unique_ptr<NetW> pack_transnet(Packer& pk) {
    auto net = std::make_unique<TnNet>();
    TnW* r = &net->w;
    const float eps = 1e-3f;   // BatchNorm3d(eps=1e-3)
    for (int s = 0; s < 3; ++s)
        for (int j = 0; j < 2; ++j) {
            TnBlock& b = r->blk[s][j];
            const int F = 16 << s;
            const int cin = j == 1 ? 4 * F : (s == 0 ? 3 : 2 * F);
            const int cin_pad = s == 0 && j == 0 ? TN_CIN : cin;
            b.F = F;
            b.cin = cin_pad;
            const std::string p = "SDDCNN." + std::to_string(s) + ".DDCNN." + std::to_string(j);
            const float* g = pk.get(p + ".bn.weight", 4 * F);
            const float* be = pk.get(p + ".bn.bias", 4 * F);
            const float* rm = pk.get(p + ".bn.running_mean", 4 * F);
            const float* rv = pk.get(p + ".bn.running_var", 4 * F);
            pk.mark(p + ".bn.num_batches_tracked");
            std::vector<float> sw((size_t)8 * F * 9 * cin_pad, 0.f);
            for (int k = 0; k < 4; ++k) {
                const std::string c = p + ".Conv3D_" + std::to_string(TN_DIL[k]) + ".layers.";
                const float* w0 = pk.get(c + "0.weight", (int64_t)2 * F * cin * 9);
                const float* w1 = pk.get(c + "1.weight", (int64_t)F * 2 * F * 3);
                if (!w0 || !w1 || !g || !be || !rm || !rv) return net;
                for (int co = 0; co < 2 * F; ++co)
                    for (int ci = 0; ci < cin; ++ci)
                        for (int tap = 0; tap < 9; ++tap)
                            sw[((size_t)(k * 2 * F + co) * 9 + tap) * cin_pad + ci] = w0[((size_t)co * cin + ci) * 9 + tap];
                std::vector<float> tw((size_t)F * 3 * 2 * F), tb(F);
                for (int co = 0; co < F; ++co) {
                    const int ch = k * F + co;
                    const float sc = g[ch] / std::sqrt(rv[ch] + eps);
                    for (int ci = 0; ci < 2 * F; ++ci)
                        for (int tap = 0; tap < 3; ++tap) tw[((size_t)co * 3 + tap) * 2 * F + ci] = w1[((size_t)co * 2 * F + ci) * 3 + tap] * sc;
                    tb[co] = be[ch] - rm[ch] * sc;
                }
                b.tw[k] = pk.add_f16(tw);
                b.tb[k] = pk.add_f32(tb);
            }
            b.sw = pk.add_f16(sw);
        }
    auto f32 = [&](const std::string& name, int64_t numel, size_t& off) {
        const float* v = pk.get(name, numel);
        if (v) off = pk.add_f32(std::vector<float>(v, v + numel));
    };
    f32("frame_sim_layer.projection.weight", (int64_t)TN_SIM * TN_FEAT, r->proj_w);
    f32("frame_sim_layer.projection.bias", TN_SIM, r->proj_b);
    f32("frame_sim_layer.fc.weight", (int64_t)TN_SIM * TN_BAND, r->sim_w);
    f32("frame_sim_layer.fc.bias", TN_SIM, r->sim_b);
    f32("color_hist_layer.fc.weight", (int64_t)TN_SIM * TN_BAND, r->hist_w);
    f32("color_hist_layer.fc.bias", TN_SIM, r->hist_b);
    const Lin fc1 = pack_linear(pk, "fc1", TN_HIDDEN, TN_ROW);
    r->fc1_w = fc1.w;
    r->fc1_b = fc1.b;
    const float* c1w = pk.get("cls_layer1.weight", TN_HIDDEN);
    const float* c1b = pk.get("cls_layer1.bias", 1);
    const float* c2w = pk.get("cls_layer2.weight", TN_HIDDEN);
    const float* c2b = pk.get("cls_layer2.bias", 1);
    if (!c1w || !c1b || !c2w || !c2b) return net;
    std::vector<float> cls(2 * TN_HIDDEN + 2);
    memcpy(cls.data(), c1w, TN_HIDDEN * 4);
    memcpy(cls.data() + TN_HIDDEN, c2w, TN_HIDDEN * 4);
    cls[2 * TN_HIDDEN] = c1b[0];
    cls[2 * TN_HIDDEN + 1] = c2b[0];
    r->cls = pk.add_f32(cls);
    return net;
}

// debug taps (nb200_debug_tap): 200 histogram counts int32 [n][512], 201 / 202 histogram / frame-similarity band fp32 [n][101],
// 203 / 204 stack-1 / stack-2 output fp16 [n][13][24][64] / [n][6][12][128], 205 fc1 input fp16 [n][4864]
static int transnet_forward(nb200_model* m, const TnW& w, cudaStream_t st, const float* x, int B, int T, float* one_hot, float* many_hot) {
    const int n = B * T;
    const size_t P0 = (size_t)TN_H * TN_W;
    __half *x16, *S, *Y1, *Y2, *P[2], *row, *hidden;
    float *feat, *emb, *bands;
    int* counts;
    if (m->carve([&](Arena& a) {
            x16 = a.take<__half>((size_t)n * P0 * TN_CIN);
            S = a.take<__half>((size_t)n * P0 * 128);   // 8F channels: largest at the first stack
            Y1 = a.take<__half>((size_t)n * P0 * 64);
            Y2 = a.take<__half>((size_t)n * P0 * 64);
            P[0] = a.take<__half>((size_t)n * 13 * 24 * 64);
            P[1] = a.take<__half>((size_t)n * 6 * 12 * 128);
            row = a.take<__half>((size_t)n * TN_ROW);
            hidden = a.take<__half>((size_t)n * TN_HIDDEN);
            feat = a.take<float>((size_t)n * TN_FEAT);
            emb = a.take<float>((size_t)n * TN_SIM);
            bands = a.take<float>((size_t)2 * n * TN_BAND);
            counts = a.take<int>((size_t)n * 512);
        })) return 1;

    if (tn_prep(st, x, n, x16)) return 1;
    if (tn_hist(st, x, n, counts)) return 1;
    if (tap_copy(st, 200, counts, (size_t)n * 512 * 4)) return 1;
    int H = TN_H, W = TN_W, mean_off = 0;
    const __half* in = x16;
    for (int s = 0; s < 3; ++s) {
        const int F = 16 << s;
        for (int j = 0; j < 2; ++j) {
            const TnBlock& b = w.blk[s][j];
            ConvGemm g;
            g.A = j == 0 ? in : Y1; g.B = n; g.Hi = H; g.Wi = W; g.Ci = b.cin; g.Cin = b.cin; g.kind = CG_CONV3; g.pad = 1;
            g.Wt = m->at<__half>(b.sw); g.N = 8 * F; g.bias = nullptr; g.act = ACT_NONE; g.out = S; g.ldo = 8 * F;
            if (conv_gemm(st, g)) return 1;
            __half* Y = j == 0 ? Y1 : Y2;
            for (int k = 0; k < 4; ++k) {
                ConvGemm t;
                t.A = S + 2 * F * k; t.B = B; t.Hi = T; t.Wi = H * W; t.Ci = 8 * F; t.Cin = 2 * F; t.kind = CG_TCONV3; t.dil = TN_DIL[k];
                t.Wt = m->at<__half>(b.tw[k]); t.N = F; t.bias = m->at<float>(b.tb[k]); t.act = j == 0 ? ACT_RELU : ACT_NONE;
                t.out = Y + F * k; t.ldo = 4 * F;
                if (conv_gemm(st, t)) return 1;
            }
        }
        const int Ho = H / 2, Wo = W / 2;
        __half* out = s < 2 ? P[s] : row + 2 * TN_SIM;
        const long long stride = s < 2 ? (long long)Ho * Wo * 4 * F : TN_ROW;
        if (tn_stack_tail(st, Y1, Y2, n, H, W, 4 * F, out, stride, feat, mean_off)) return 1;
        if (s < 2 && tap_copy(st, 203 + s, out, (size_t)n * Ho * Wo * 4 * F * 2)) return 1;
        mean_off += 4 * F;
        in = out;
        H = Ho;
        W = Wo;
    }
    if (tn_project(st, feat, n, m->at<float>(w.proj_w), m->at<float>(w.proj_b), emb)) return 1;
    if (tn_bands(st, counts, emb, B, T, m->at<float>(w.hist_w), m->at<float>(w.hist_b), m->at<float>(w.sim_w), m->at<float>(w.sim_b),
                 bands, row)) return 1;
    if (tap_copy(st, 201, bands, (size_t)n * TN_BAND * 4)) return 1;
    if (tap_copy(st, 202, bands + (size_t)n * TN_BAND, (size_t)n * TN_BAND * 4)) return 1;
    if (tap_copy(st, 205, row, (size_t)n * TN_ROW * 2)) return 1;
    Lin fc1;
    fc1.w = w.fc1_w; fc1.b = w.fc1_b; fc1.N = TN_HIDDEN; fc1.K = TN_ROW;
    if (linear_flat(st, m, fc1, row, n, TN_ROW, hidden, TN_HIDDEN, ACT_RELU)) return 1;
    return tn_heads(st, hidden, n, m->at<float>(w.cls), one_hot, many_hot);
}

}  // namespace nb200

using namespace nb200;

// TransNetV2.forward (nunif/utils/transnetv2.py:49-87) on B windows of T frames: the one_hot and many_hot logits
extern "C" int nb200_transnetv2_forward(nb200_model* m, const float* x, int B, int T, float* one_hot, float* many_hot, void* stream) {
    NB_CHECK(m && x && one_hot && many_hot, "null pointer");
    const TnNet* net = net_as<TnNet>(m);
    NB_CHECK(net, "model is not TransNetV2");
    NB_CHECK(B > 0 && T > 0 && (long long)B * T <= (1 << 20), "bad shape");
    return transnet_forward(m, net->w, (cudaStream_t)stream, x, B, T, one_hot, many_hot);
}
