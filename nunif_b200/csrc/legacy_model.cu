// UpConv7 / VGG7: weight packing and forward, and the test entry point of the output layer.
// Reference: waifu2x/models/upconv_7.py:6-38, waifu2x/models/vgg_7.py:6-36.  Both are nn.Sequential stacks `net.{0..12}` of
// 3x3 valid convs + LeakyReLU(0.1) and one 3-channel output layer, clamped to [0, 1] in eval mode.
#include "model.h"
#include "gemm.h"
#include "swin_kernels.h"
#include "legacy_kernels.h"

namespace nb200 {

struct NB_HIDDEN LegacyW : NetW {
    bool up = false;      // upconv_7 (ConvTranspose head) vs vgg_7
    Lin stem;             // net.0, fp32 stem weights (cout padded to 32)
    Lin conv[5];          // net.2 .. net.10 as implicit-GEMM operands
    int cin[5] = {}, cout[5] = {};
    size_t head_w = 0, head_b = 0;
    int head_cin = 0;
};

// output layer: fp32 [tap][ci][co] (values at fp16 precision, SIMT kernel) followed by fp16 mma.sync B fragments
// [chunk (cin / 64)][tap][kc (4 x 16 channels)][n (8, rows >= 3 zero)][16] (head_conv_mma_kernel streams one chunk at a time)
// from the Conv2d [3][cin][3][3] / ConvTranspose2d [cin][3][4][4] weight
static std::vector<float> pack_head_w(const float* w, bool deconv, int cin) {
    const int taps = deconv ? 16 : 9;
    std::vector<float> wv((size_t)taps * cin * 3);
    for (int t = 0; t < taps; ++t)
        for (int ci = 0; ci < cin; ++ci)
            for (int co = 0; co < 3; ++co) {
                // Conv2d: [co][ci][ky][kx] ; ConvTranspose2d: [ci][co][ky][kx]
                const float v = deconv ? w[((size_t)ci * 3 + co) * 16 + t] : w[((size_t)co * cin + ci) * 9 + t];
                wv[((size_t)t * cin + ci) * 3 + co] = round_f16(v);
            }
    const size_t nf = wv.size();
    wv.resize(nf + (size_t)taps * cin * 4, 0.f);   // taps * (cin / 16) * 128 halves
    __half* frag = reinterpret_cast<__half*>(wv.data() + nf);
    for (int c = 0; c < cin / 64; ++c)
        for (int t = 0; t < taps; ++t)
            for (int kc = 0; kc < 4; ++kc)
                for (int nn = 0; nn < 8; ++nn)
                    for (int k = 0; k < 16; ++k)
                        frag[((((size_t)c * taps + t) * 4 + kc) * 8 + nn) * 16 + k] =
                            __float2half_rn(nn < 3 ? wv[((size_t)t * cin + c * 64 + kc * 16 + k) * 3 + nn] : 0.f);
    return wv;
}
static void pack_head(Packer& pk, const std::string& name, bool deconv, int cin, size_t* w_off, size_t* b_off) {
    const float* w = pk.get(name + ".weight", (int64_t)cin * 3 * (deconv ? 16 : 9));
    const float* b = pk.get(name + ".bias", 3);
    if (!w || !b) return;
    *w_off = pk.add_f32(pack_head_w(w, deconv, cin));
    *b_off = pk.add_f32(std::vector<float>(b, b + 3));
}

std::unique_ptr<NetW> pack_legacy(Packer& pk, bool up) {
    auto w = std::make_unique<LegacyW>();
    w->up = up;
    // upconv_7.py:12-25 / vgg_7.py:12-25
    static const int up_ch[7] = {3, 16, 32, 64, 128, 128, 256};
    static const int vgg_ch[7] = {3, 32, 32, 64, 64, 128, 128};
    const int* ch = up ? up_ch : vgg_ch;
    // net.0: upconv_7's 16 output channels are padded to 32 with zero weights and biases, so the padded channels are
    // exactly 0 after the LeakyReLU and net.2 can run with K per tap = 32 (the implicit GEMM's minimum)
    w->stem = pack_stem(pk, "net.0", ch[1], 32);
    for (int i = 0; i < 5; ++i) {
        w->cin[i] = ch[i + 1] < 32 ? 32 : ch[i + 1];
        w->cout[i] = ch[i + 2];
        w->conv[i] = pack_conv(pk, "net." + std::to_string(2 * i + 2), ch[i + 2], ch[i + 1], 3, 3, /*cin_pad=*/w->cin[i]);
    }
    w->head_cin = ch[6];
    pack_head(pk, "net.12", up, ch[6], &w->head_w, &w->head_b);
    return w;
}

// x [n][T][T][8] fp16 -> z [n][3][S][S] fp16; S = 2T - 28 (upconv_7) or T - 14 (vgg_7)
int legacy_forward(nb200_model* m, cudaStream_t st, const __half* x, int n, int T, int /*down*/, void* z) {
    const LegacyW& w = *net_as<LegacyW>(m);
    NB_CHECK(T >= 15, "tile_size too small for " + std::string(w.up ? "upconv_7" : "vgg_7") + ": input_tile_step = tile_size - 14 must be positive");
    // ping-pong workspaces sized for the largest activation (net.0 .. net.10 outputs: T-2 .. T-12)
    size_t e_max = (size_t)n * (T - 2) * (T - 2) * 32;
    for (int i = 0; i < 5; ++i) {
        const size_t H = T - 4 - 2 * i;
        const size_t e = (size_t)n * H * H * w.cout[i];
        if (e > e_max) e_max = e;
    }
    __half* buf[2];
    if (m->carve([&](Arena& a) { buf[0] = a.take<__half>(e_max); buf[1] = a.take<__half>(e_max); })) return 1;
    if (stem_conv3x3(st, x, m->at<float>(w.stem.w), m->at<float>(w.stem.b), buf[0], n, T, T, 32, 32)) return 1;
    int H = T - 2;
    for (int i = 0; i < 5; ++i, H -= 2) {
        ConvGemm g;
        g.A = buf[i & 1]; g.B = n; g.Hi = H; g.Wi = H; g.Ci = w.cin[i]; g.Cin = w.cin[i]; g.kind = CG_CONV3;
        g.Wt = m->at<__half>(w.conv[i].w); g.N = w.cout[i]; g.bias = m->at<float>(w.conv[i].b); g.act = ACT_LRELU01;
        g.out = buf[(i + 1) & 1]; g.ldo = w.cout[i];
        if (conv_gemm(st, g)) return 1;
    }
    // H = T - 12: the last hidden activation (in buf[1]); net.12 + clamp (upconv_7.py:33-38, vgg_7.py:31-36)
    return head_conv(st, w.up ? 1 : 0, w.head_cin, buf[1], m->at<float>(w.head_w), m->at<float>(w.head_b), (__half*)z, n, H, H);
}

}  // namespace nb200

using namespace nb200;

// ---- test entry point of the output layer: the weights are host fp32 tensors in the PyTorch layout, packed by pack_head_w
extern "C" int nb200_head_conv_f16(const void* x, const float* w, const float* b, int mode, int cin, int n, int Hi, int Wi, void* out,
                                   void* stream) {
    NB_CHECK(x && w && b && out, "null pointer");
    NB_CHECK((mode == 0 && cin == 128) || (mode == 1 && cin == 256), "unsupported (mode, input channels)");
    NB_CHECK(n > 0, "empty batch");
    const std::vector<float> wv = pack_head_w(w, mode == 1, cin), bv(b, b + 3);
    cudaStream_t st = (cudaStream_t)stream;
    return with_uploaded(st, {&wv, &bv}, [&](const std::vector<const float*>& p) {
        return head_conv(st, mode, cin, (const __half*)x, p[0], p[1], (__half*)out, n, Hi, Wi);
    });
}
