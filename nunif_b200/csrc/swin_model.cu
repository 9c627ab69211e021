// SwinUNet 1x / 2x / 4x (waifu2x/models/swin_unet.py:119-199): weight packing, the Swin bias-fragment build after upload and
// the forward as a sequence of the sm_90a kernels.  Also the stem convolution's test entry point.
#include "model.h"
#include "gemm.h"
#include "swin_kernels.h"

namespace nb200 {

struct SwinBlockW {
    Lin qkv, proj, fc1, fc2;
    size_t rpb = 0;       // relative_position_bias_table [121][6] fp32, as in the state_dict
    // rpb in the attention core's accumulator-fragment order, built on the device at load by build_bias_frag_kernel
    // (swin_attention_mma.cu), the only definition of that layout
    size_t table = 0;
    int C = 0, shift = 0;
};

struct NB_HIDDEN SwinW : NetW {
    int C = 96, r = 4, cs = 48;
    Lin stem, conv2, down1, down2, up2, up1, toimg;   // 4x: up1 carries proj2 (pack_linear_pixshuf2 with a skip)
    std::vector<SwinBlockW> s1, s2, s3, s4, s5;
};

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
            b.table = pk.add_f32(std::vector<float>(BIAS_FRAG_FLOATS));   // filled by swin_build_bias_frags
        }
        pk.mark(p + ".attn.relative_position_index");  // buffer; the kernel recomputes the index (swin_transformer.py:267-279)
        out.push_back(b);
    }
}

std::unique_ptr<NetW> pack_swin(Packer& pk, int r) {
    auto sw = std::make_unique<SwinW>();
    SwinW& w = *sw;
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
    return sw;
}

// once the blob is on the device: each block's bias-fragment slot is built from its raw table (on the null stream)
int swin_build_bias_frags(nb200_model* m) {
    const SwinW& w = *net_as<SwinW>(m);
    for (const auto* blocks : {&w.s1, &w.s2, &w.s3, &w.s4, &w.s5})
        for (const SwinBlockW& b : *blocks)
            if (build_bias_frag(0, m->at<float>(b.rpb), m->at<float>(b.table))) return 1;
    return 0;
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

int swin_forward(nb200_model* m, cudaStream_t st, const __half* x, int n, int T, int down, void* z) {
    const SwinW& w = *net_as<SwinW>(m);
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

using namespace nb200;

// ---- test entry point of the stem convolution (also CUNet's and UpConv7 / VGG7's first layer): the weights are host fp32
// tensors in the PyTorch layout, packed by the stem packer
extern "C" int nb200_stem_conv_f16(const void* x, const float* w, const float* b, int cout, int cout_pad, int n, int Hi, int Wi,
                                   void* out, int ldo, void* stream) {
    NB_CHECK(x && w && b && out, "null pointer");
    NB_CHECK(cout > 0 && cout <= cout_pad && (cout_pad == 32 || cout_pad == 64), "cout_pad must be 32 or 64, cout at most cout_pad");
    NB_CHECK(n > 0 && Hi > 2 && Wi > 2, "input too small");
    std::vector<float> wv, bv;
    pack_stem_w(w, b, cout, cout_pad, wv, bv);
    cudaStream_t st = (cudaStream_t)stream;
    return with_uploaded(st, {&wv, &bv}, [&](const std::vector<const float*>& p) {
        return stem_conv3x3(st, (const __half*)x, p[0], p[1], (__half*)out, n, Hi, Wi, cout_pad, ldo);
    });
}
