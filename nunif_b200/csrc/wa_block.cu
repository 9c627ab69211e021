// The window-attention block WABlock that sbs.row_flow_v3, sbs.mlbw and iw3.depth_aa are built from (iw3/models/row_flow_v3.py
// :13-29, mlbw.py:18-34, depth_aa.py:11-26; state_dict keys `<block>.mha.mha.*`, `<block>.bias.*`, `<block>.conv_mlp.*`):
//     x = x + WindowMHA2d(x, attn_mask = WindowScoreBias())
//     x = x + act(conv3x3(ReplicationPad2d(1)(gelu(conv1x1(x)))))
// The models differ only in channels, window, heads, shift and the activation after the 3x3 (LeakyReLU(0.1) or none).
// The WindowScoreBias MLP (nunif/modules/attention.py:375-420) only depends on weights, so its (N x N) table is evaluated
// once at pack time.
#include "wa_block.h"
#include "window_mha.h"
#include <cmath>

namespace nb200 {

static size_t pack_window_bias(Packer& pk, const std::string& p, int ws) {
    const int N = ws * ws, U = (2 * ws - 1) * (2 * ws - 1), hid = (int)std::sqrt((double)N) * 2;
    const float* idx = pk.get(p + "index", (int64_t)N * N);          // int64 buffer, delivered as float32 by the loader
    const float* dl = pk.get(p + "delta", (int64_t)U * 2);
    const float* w0 = pk.get(p + "to_bias.0.weight", (int64_t)hid * 2);
    const float* b0 = pk.get(p + "to_bias.0.bias", hid);
    const float* w1 = pk.get(p + "to_bias.2.weight", hid);
    const float* b1 = pk.get(p + "to_bias.2.bias", 1);
    if (!idx || !dl || !w0 || !b0 || !w1 || !b1) return 0;
    std::vector<float> tab(U), out((size_t)N * N);
    for (int u = 0; u < U; ++u) {
        double acc = b1[0];
        for (int j = 0; j < hid; ++j) {
            const double z = (double)w0[j * 2] * dl[u * 2] + (double)w0[j * 2 + 1] * dl[u * 2 + 1] + b0[j];
            acc += (double)w1[j] * (0.5 * z * (1.0 + std::erf(z * 0.7071067811865476)));        // nn.GELU (erf)
        }
        tab[u] = (float)acc;
    }
    for (int i = 0; i < N * N; ++i) {
        const int u = (int)std::lround(idx[i]);
        if (u < 0 || u >= U) { if (pk.err.empty()) pk.err = "bad window bias index in " + p; return 0; }
        out[i] = tab[u];
    }
    return pk.add_f32(out);
}

WaBlockW pack_wa_block(Packer& pk, const std::string& p, int C, int ws, int heads, int pad_y, int pad_x, int act) {
    WaBlockW b;
    b.ws = ws; b.heads = heads; b.pad_y = pad_y; b.pad_x = pad_x; b.act = act;
    b.qkv = pack_linear(pk, p + "mha.mha.qkv_proj", 3 * C, C);
    b.proj = pack_linear(pk, p + "mha.mha.head_proj", C, C);
    b.mlp0 = pack_conv(pk, p + "conv_mlp.0", C, C, 1, 1);
    b.mlp3 = pack_conv(pk, p + "conv_mlp.3", C, C, 3, 3);
    b.bias = pack_window_bias(pk, p + "bias.", ws);
    return b;
}

void wa_plan(Arena& a, WaBufs& w, int B, int H, int W, int C) {
    const size_t M = (size_t)B * H * W;
    w.X = a.take<__half>(M * C);
    w.QKV = a.take<__half>(M * 3 * C);
    w.ATT = a.take<__half>(M * C);
    w.T = a.take<__half>(M * C);
    w.TP = a.take<__half>((size_t)B * (H + 2) * (W + 2) * C);
}

int wa_block(cudaStream_t st, const nb200_model* m, const WaBlockW& b, const WaBufs& w, int B, int H, int W) {
    const int C = b.proj.N;
    const long long M = (long long)B * H * W;
    // x = x + mha(x, attn_mask=bias)
    if (linear_flat(st, m, b.qkv, w.X, M, C, w.QKV, 3 * C, ACT_NONE)) return 1;
    if (window_mha(st, w.QKV, m->at<float>(b.qkv.b), m->at<float>(b.bias), w.ATT, B, H, W, C, b.ws, b.heads, b.pad_y, b.pad_x)) return 1;
    if (linear_flat(st, m, b.proj, w.ATT, M, C, w.X, C, ACT_NONE, w.X, C)) return 1;
    // x = x + act(conv3x3(reppad(gelu(conv1x1(x)))))
    if (linear_flat(st, m, b.mlp0, w.X, M, C, w.T, C, ACT_GELU)) return 1;
    if (reppad1(st, w.T, B, H, W, C, w.TP)) return 1;
    ConvGemm g;
    g.A = w.TP; g.B = B; g.Hi = H + 2; g.Wi = W + 2; g.Ci = C; g.Cin = C; g.kind = CG_CONV3;
    g.Wt = m->at<__half>(b.mlp3.w); g.N = C; g.bias = m->at<float>(b.mlp3.b); g.act = b.act; g.out = w.X; g.ldo = C;
    g.res = w.X; g.ldr = C; g.res_H = H; g.res_W = W;
    return conv_gemm(st, g);
}

int stereo_geometry(int B, int H, int W, int ph1, int pw1, int Hp, int Wp) {
    NB_CHECK(B > 0 && H > 0 && W > 0, "empty input");
    NB_CHECK(ph1 >= 0 && pw1 >= 0, "negative leading pad");
    NB_CHECK(ph1 + H <= Hp, "padded height < ph1 + H");
    NB_CHECK(pw1 + W <= Wp, "padded width < pw1 + W");
    return 0;
}

}  // namespace nb200
