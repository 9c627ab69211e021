// CUNet / UpCUNet: weight packing and forward, and the test entry points of the tail convolution and the SE block.
// Reference: waifu2x/models/cunet.py:10-203, nunif/modules/attention.py:29-44.
#include "model.h"
#include "gemm.h"
#include "swin_kernels.h"
#include "cunet_kernels.h"
#include <algorithm>

namespace nb200 {

struct SEW {
    size_t w1 = 0, b1 = 0, w2 = 0, b2 = 0;
    int C = 0;
};
struct UNetConvW {
    Lin c0, c1;  // c0 is a stem (fp32) when cin == 3
    SEW se;
    bool has_se = false, stem = false;
    int cin = 0, cmid = 0, cout = 0;
};
struct NB_HIDDEN CUNetW : NetW {
    bool up = false;
    // unet1
    UNetConvW u1c1, u1c2;
    Lin u1down, u1up, u1c3;
    size_t u1bot_w = 0, u1bot_b = 0;
    // unet2
    UNetConvW u2c1, u2c2, u2c3, u2c4;
    Lin u2down1, u2down2, u2up3, u2up4, u2c5;
    size_t u2bot_w = 0, u2bot_b = 0;
};

// SE 1x1 convs conv1 [C/8][C], conv2 [C][C/8] and their biases -> fp32 at fp16 precision (they run in fp16 under autocast)
static std::vector<float> pack_se_w(const float* a, size_t n) {
    std::vector<float> v(n);
    for (size_t i = 0; i < n; ++i) v[i] = round_f16(a[i]);
    return v;
}
static SEW pack_se(Packer& pk, const std::string& p, int C) {
    SEW s;
    s.C = C;
    const int R = C / 8;
    const float* w1 = pk.get(p + ".conv1.weight", (int64_t)R * C);
    const float* b1 = pk.get(p + ".conv1.bias", R);
    const float* w2 = pk.get(p + ".conv2.weight", (int64_t)C * R);
    const float* b2 = pk.get(p + ".conv2.bias", C);
    if (!w1 || !b1 || !w2 || !b2) return s;
    s.w1 = pk.add_f32(pack_se_w(w1, (size_t)R * C));
    s.b1 = pk.add_f32(pack_se_w(b1, R));
    s.w2 = pk.add_f32(pack_se_w(w2, (size_t)C * R));
    s.b2 = pk.add_f32(pack_se_w(b2, C));
    return s;
}

static UNetConvW pack_unet_conv(Packer& pk, const std::string& p, int cin, int cmid, int cout, bool se) {
    UNetConvW u;
    u.cin = cin; u.cmid = cmid; u.cout = cout; u.has_se = se; u.stem = (cin == 3);
    u.c0 = u.stem ? pack_stem(pk, p + ".conv.0", cmid, cmid) : pack_conv(pk, p + ".conv.0", cmid, cin, 3, 3);
    u.c1 = pack_conv(pk, p + ".conv.2", cout, cmid, 3, 3);
    if (se) u.se = pack_se(pk, p + ".seblock", cout);
    return u;
}

// tail weights (Conv2d [3][64][3][3] or ConvTranspose2d [64][3][4][4]) as fp32 [tap][ci][co] (values at fp16 precision)
static std::vector<float> pack_tail_w(const float* w, bool deconv) {
    const int taps = deconv ? 16 : 9;
    std::vector<float> wv((size_t)taps * 64 * 3);
    for (int t = 0; t < taps; ++t)
        for (int ci = 0; ci < 64; ++ci)
            for (int co = 0; co < 3; ++co) {
                // Conv2d: [co][ci][ky][kx] ; ConvTranspose2d: [ci][co][ky][kx]
                const float v = deconv ? w[((size_t)ci * 3 + co) * 16 + t] : w[((size_t)co * 64 + ci) * 9 + t];
                wv[((size_t)t * 64 + ci) * 3 + co] = round_f16(v);
            }
    // ... followed by the same weights as fp16 mma.sync B fragments [tap][kc (4 x 16 channels)][n (8, rows >= 3 zero)][16]
    // (tail_conv_mma_kernel copies this block to shared memory with 16-byte loads)
    const size_t nf = wv.size();
    wv.resize(nf + (size_t)taps * 256, 0.f);
    __half* frag = reinterpret_cast<__half*>(wv.data() + nf);
    for (int t = 0; t < taps; ++t)
        for (int kc = 0; kc < 4; ++kc)
            for (int nn = 0; nn < 8; ++nn)
                for (int k = 0; k < 16; ++k)
                    frag[(((size_t)t * 4 + kc) * 8 + nn) * 16 + k] = __float2half_rn(nn < 3 ? wv[((size_t)t * 64 + kc * 16 + k) * 3 + nn] : 0.f);
    return wv;
}
static void pack_tail(Packer& pk, const std::string& name, bool deconv, size_t* w_off, size_t* b_off) {
    const float* w = pk.get(name + ".weight", (int64_t)64 * 3 * (deconv ? 16 : 9));
    const float* b = pk.get(name + ".bias", 3);
    if (!w || !b) return;
    *w_off = pk.add_f32(pack_tail_w(w, deconv));
    *b_off = pk.add_f32(std::vector<float>(b, b + 3));
}

// ConvTranspose2d(k=2, s=2) weight [Cin][Cout][2][2] -> rows n = (dy*2+dx)*cout + co, K = cin
static Lin pack_convT2(Packer& pk, const std::string& name, int cin, int cout) {
    Lin l;
    l.N = 4 * cout;
    l.K = cin;
    const float* w = pk.get(name + ".weight", (int64_t)cin * cout * 4);
    const float* b = pk.get(name + ".bias", cout);
    if (!w || !b) return l;
    std::vector<float> wv((size_t)l.N * cin), bv(l.N);
    for (int g = 0; g < 4; ++g)
        for (int co = 0; co < cout; ++co) {
            for (int ci = 0; ci < cin; ++ci) wv[((size_t)g * cout + co) * cin + ci] = w[((size_t)ci * cout + co) * 4 + g];
            bv[g * cout + co] = b[co];
        }
    l.w = pk.add_f16(wv);
    l.b = pk.add_f32(bv);
    return l;
}
std::unique_ptr<NetW> pack_cunet(Packer& pk, bool up) {
    auto w = std::make_unique<CUNetW>();
    w->up = up;
    w->u1c1 = pack_unet_conv(pk, "unet1.conv1", 3, 32, 64, false);
    w->u1down = pack_conv(pk, "unet1.conv1_down", 64, 64, 2, 2);
    w->u1c2 = pack_unet_conv(pk, "unet1.conv2", 64, 128, 64, true);
    w->u1up = pack_convT2(pk, "unet1.conv2_up", 64, 64);
    w->u1c3 = pack_conv(pk, "unet1.conv3", 64, 64, 3, 3);
    pack_tail(pk, "unet1.conv_bottom", up, &w->u1bot_w, &w->u1bot_b);
    w->u2c1 = pack_unet_conv(pk, "unet2.conv1", 3, 32, 64, false);
    w->u2down1 = pack_conv(pk, "unet2.conv1_down", 64, 64, 2, 2);
    w->u2c2 = pack_unet_conv(pk, "unet2.conv2", 64, 64, 128, true);
    w->u2down2 = pack_conv(pk, "unet2.conv2_down", 128, 128, 2, 2);
    w->u2c3 = pack_unet_conv(pk, "unet2.conv3", 128, 256, 128, true);
    w->u2up3 = pack_convT2(pk, "unet2.conv3_up", 128, 128);
    w->u2c4 = pack_unet_conv(pk, "unet2.conv4", 128, 64, 64, true);
    w->u2up4 = pack_convT2(pk, "unet2.conv4_up", 64, 64);
    w->u2c5 = pack_conv(pk, "unet2.conv5", 64, 64, 3, 3);
    pack_tail(pk, "unet2.conv_bottom", false, &w->u2bot_w, &w->u2bot_b);
    return w;
}

struct NB_HIDDEN CuCtx {
    nb200_model* m;
    cudaStream_t st;
    int n;
    float *se_partial, *se_scale;
};

static int conv3(CuCtx& c, const Lin& l, const __half* A, int H, int W, int Cin, __half* out, int act) {
    ConvGemm g;
    g.A = A; g.B = c.n; g.Hi = H; g.Wi = W; g.Ci = Cin; g.Cin = Cin; g.kind = CG_CONV3;
    g.Wt = c.m->at<__half>(l.w); g.N = l.N; g.bias = c.m->at<float>(l.b); g.act = act; g.out = out; g.ldo = l.N;
    return conv_gemm(c.st, g);
}
static int down2(CuCtx& c, const Lin& l, const __half* A, int H, int W, int Cin, __half* out) {
    ConvGemm g;
    g.A = A; g.B = c.n; g.Hi = H; g.Wi = W; g.Ci = Cin; g.Cin = Cin; g.kind = CG_DOWN2;
    g.Wt = c.m->at<__half>(l.w); g.N = l.N; g.bias = c.m->at<float>(l.b); g.act = ACT_LRELU01; g.out = out; g.ldo = l.N;
    return conv_gemm(c.st, g);
}
// ConvTranspose 2x2 s2 + LeakyReLU, then "+ skip[crop]" (cunet.py:60-64, 109-117)
static int up2_add(CuCtx& c, const Lin& l, const __half* A, int H, int W, int Cin, __half* out, int cout, const __half* skip,
                   int skipH, int skipW, int crop) {
    ConvGemm g;
    g.A = A; g.B = c.n; g.Hi = H; g.Wi = W; g.Ci = Cin; g.Cin = Cin; g.kind = CG_LINEAR_2D;
    g.Wt = c.m->at<__half>(l.w); g.N = l.N; g.bias = c.m->at<float>(l.b); g.act = ACT_LRELU01; g.out = out; g.ldo = cout;
    g.out_mode = OUT_PIXSHUF2; g.cout = cout; g.res = skip; g.ldr = cout; g.res_H = skipH; g.res_W = skipW;
    g.res_cy = crop; g.res_cx = crop;
    return conv_gemm(c.st, g);
}
// UNetConv (cunet.py:10-28): A [n][H][W][cin_stride] -> out [n][H-4][W-4][cout]; tmp holds the mid activation
static int unet_conv(CuCtx& c, const UNetConvW& u, const __half* A, int H, int W, __half* tmp, __half* out) {
    if (u.stem) {
        if (stem_conv3x3(c.st, A, c.m->at<float>(u.c0.w), c.m->at<float>(u.c0.b), tmp, c.n, H, W, u.cmid, u.cmid)) return 1;
    } else {
        if (conv3(c, u.c0, A, H, W, u.cin, tmp, ACT_LRELU01)) return 1;
    }
    if (conv3(c, u.c1, tmp, H - 2, W - 2, u.cmid, out, ACT_LRELU01)) return 1;
    if (u.has_se)
        return se_block(c.st, out, c.n, H - 4, W - 4, u.cout, c.m->at<float>(u.se.w1), c.m->at<float>(u.se.b1),
                        c.m->at<float>(u.se.w2), c.m->at<float>(u.se.b2), c.se_partial, c.se_scale);
    return 0;
}

int cunet_forward(nb200_model* m, cudaStream_t st, const __half* x, int n, int T, int /*down*/, void* z) {
    const CUNetW& w = *net_as<CUNetW>(m);
    NB_CHECK(T % 4 == 0 && T >= 64, "invalid tile size for cunet (cunet.py:124-125)");
    // ---- geometry
    const int a1 = T - 4;                 // unet1 x1
    const int a2 = a1 / 2;                // after conv1_down
    const int a3 = a2 - 4;                // conv2 out
    const int a4 = 2 * a3;                // conv2_up out == a1 - 8
    const int a5 = a4 - 2;                // conv3 out
    const int Hz = w.up ? 2 * a5 - 4 : a5 - 2;  // z1
    const int b1 = Hz - 4, b2 = b1 / 2, b3 = b2 - 4, b4 = b3 / 2, b5 = b4 - 4, b6 = 2 * b5, b7 = b6 - 4, b8 = 2 * b7,
              b9 = b8 - 2, Ho = b9 - 2;
    NB_CHECK(b5 > 0 && b6 == b3 - 8 && b8 == b1 - 32 && Ho == Hz - 40, "tile too small for cunet");
    // ---- workspace
    const size_t nn = (size_t)n;
    // TMP holds the mid activation of every UNetConv: the largest of them
    size_t e_tmp_max = nn * (size_t)(T - 2) * (T - 2) * 32;
    for (size_t e : {nn * (a2 - 2) * (a2 - 2) * 128, nn * (Hz - 2) * (Hz - 2) * 32, nn * (b2 - 2) * (b2 - 2) * 64,
                     nn * (b4 - 2) * (b4 - 2) * 256, nn * (b6 - 2) * (b6 - 2) * 64})
        e_tmp_max = std::max(e_tmp_max, e);
    const size_t se_p = se_partial_floats(n, b3, b3, 128) + se_partial_floats(n, a3, a3, 64) + 1024;
    __half *TMP, *X1, *D1, *C2, *U2, *C3, *Z1, *Y1, *E1, *Y2, *E2, *Y3, *U3, *Y4, *U4, *Y5;
    float *se_partial, *se_scale;
    if (m->carve([&](Arena& a) {
            TMP = a.take<__half>(e_tmp_max);
            X1 = a.take<__half>(nn * a1 * a1 * 64);
            D1 = a.take<__half>(nn * a2 * a2 * 64);
            C2 = a.take<__half>(nn * a3 * a3 * 64);
            U2 = a.take<__half>(nn * a4 * a4 * 64);   // x1crop + up
            C3 = a.take<__half>(nn * a5 * a5 * 64);
            Z1 = a.take<__half>(nn * Hz * Hz * 8);
            Y1 = a.take<__half>(nn * b1 * b1 * 64);
            E1 = a.take<__half>(nn * b2 * b2 * 64);
            Y2 = a.take<__half>(nn * b3 * b3 * 128);
            E2 = a.take<__half>(nn * b4 * b4 * 128);
            Y3 = a.take<__half>(nn * b5 * b5 * 128);
            U3 = a.take<__half>(nn * b6 * b6 * 128);
            Y4 = a.take<__half>(nn * b7 * b7 * 64);
            U4 = a.take<__half>(nn * b8 * b8 * 64);
            Y5 = a.take<__half>(nn * b9 * b9 * 64);
            se_partial = a.take<float>(se_p);
            se_scale = a.take<float>(nn * 128);
        })) return 1;
    CuCtx c{m, st, n, se_partial, se_scale};

    // ---- unet1 (cunet.py:55-67)
    if (unet_conv(c, w.u1c1, x, T, T, TMP, X1)) return 1;
    if (down2(c, w.u1down, X1, a1, a1, 64, D1)) return 1;
    if (unet_conv(c, w.u1c2, D1, a2, a2, TMP, C2)) return 1;
    if (up2_add(c, w.u1up, C2, a3, a3, 64, U2, 64, X1, a1, a1, 4)) return 1;
    if (conv3(c, w.u1c3, U2, a4, a4, 64, C3, ACT_LRELU01)) return 1;
    if (tail_conv(st, w.up ? 1 : 0, 0, C3, m->at<float>(w.u1bot_w), m->at<float>(w.u1bot_b), Z1, nullptr, n, a5, a5, 0, 0,
                  m->no_clip ? 0 : 1)) return 1;
    // ---- unet2 (cunet.py:99-121)
    if (unet_conv(c, w.u2c1, Z1, Hz, Hz, TMP, Y1)) return 1;
    if (down2(c, w.u2down1, Y1, b1, b1, 64, E1)) return 1;
    if (unet_conv(c, w.u2c2, E1, b2, b2, TMP, Y2)) return 1;
    if (down2(c, w.u2down2, Y2, b3, b3, 128, E2)) return 1;
    if (unet_conv(c, w.u2c3, E2, b4, b4, TMP, Y3)) return 1;
    if (up2_add(c, w.u2up3, Y3, b5, b5, 128, U3, 128, Y2, b3, b3, 4)) return 1;
    if (unet_conv(c, w.u2c4, U3, b6, b6, TMP, Y4)) return 1;
    if (up2_add(c, w.u2up4, Y4, b7, b7, 64, U4, 64, Y1, b1, b1, 16)) return 1;
    if (conv3(c, w.u2c5, U4, b8, b8, 64, Y5, ACT_LRELU01)) return 1;
    // z = clamp(z1[20:-20] + unet2(z1))  (cunet.py:154-163)
    return tail_conv(st, 0, 1, Y5, m->at<float>(w.u2bot_w), m->at<float>(w.u2bot_b), (__half*)z, Z1, n, b9, b9, Hz, Hz, 1);
}

}  // namespace nb200

using namespace nb200;

// ---- test entry points of the tail convolution and the SE block: the weights are host fp32 tensors in the PyTorch layout,
// packed by this file's packers
extern "C" int nb200_tail_conv_f16(const void* x, const float* w, const float* b, int mode, int epi, int n, int Hi, int Wi, void* out,
                                   const void* z1, int z1H, int z1W, int clip, void* stream) {
    NB_CHECK(x && w && b && out && (epi == 0 || z1), "null pointer");
    NB_CHECK((mode == 0 && (epi == 0 || epi == 1)) || (mode == 1 && epi == 0), "unsupported (mode, epilogue)");
    const int Ho = mode == 0 ? Hi - 2 : 2 * Hi - 4, Wo = mode == 0 ? Wi - 2 : 2 * Wi - 4;
    NB_CHECK(n > 0 && Ho > 0 && Wo > 0, "input too small");
    NB_CHECK(epi == 0 || (z1H >= Ho + 40 && z1W >= Wo + 40), "z1 smaller than the output plus its 20-pixel crop");
    const std::vector<float> wv = pack_tail_w(w, mode == 1), bv(b, b + 3);
    cudaStream_t st = (cudaStream_t)stream;
    return with_uploaded(st, {&wv, &bv}, [&](const std::vector<const float*>& p) {
        return tail_conv(st, mode, epi, (const __half*)x, p[0], p[1], (__half*)out, (const __half*)z1, n, Hi, Wi, z1H, z1W, clip);
    });
}

extern "C" int nb200_se_block_f16(void* x, const float* w1, const float* b1, const float* w2, const float* b2, int n, int H, int W, int C,
                                  void* stream) {
    NB_CHECK(x && w1 && b1 && w2 && b2, "null pointer");
    NB_CHECK(C == 64 || C == 128, "channels must be 64 or 128");
    NB_CHECK(n > 0 && n <= 65535 && H > 0 && W > 0, "bad geometry");
    const int R = C / 8;
    const std::vector<float> W1 = pack_se_w(w1, (size_t)R * C), B1 = pack_se_w(b1, R), W2 = pack_se_w(w2, (size_t)C * R),
                             B2 = pack_se_w(b2, C);
    const std::vector<float> scratch(se_partial_floats(n, H, W, C) + (size_t)n * C);   // partial sums, then the scales
    cudaStream_t st = (cudaStream_t)stream;
    return with_uploaded(st, {&W1, &B1, &W2, &B2, &scratch}, [&](const std::vector<const float*>& p) {
        float* partial = const_cast<float*>(p[4]);
        return se_block(st, (__half*)x, n, H, W, C, p[0], p[1], p[2], p[3], partial, partial + se_partial_floats(n, H, W, C));
    });
}
