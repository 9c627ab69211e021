// inpaint.light_inpaint_v1 (iw3/models/light_inpaint_v1.py): weight packing and forward, and the hole-mask preparation that
// feeds it (nb200_inpaint_mask, nb200_inpaint_blur).
#include "model.h"
#include "gemm.h"
#include "inpaint_kernels.h"
#include <algorithm>
#include <cmath>

namespace nb200 {

struct GmlpW {                 // GMLPBlock (light_inpaint_v1.py:37-49, nunif/modules/attention.py:621-693)
    int C = 0, ws = 0, shift = 0, cpad = 0;
    Lin pin, pout, w1, w2;     // proj_in C -> 4C, proj_out 2C -> C, glu_conv.w1 1x1 C -> C, glu_conv.w2 3x3 C/2 (padded to cpad) -> C
    size_t g1 = 0, g2 = 0;     // norm1 [C], norm2 [2C] fp32
    size_t ws_frag = 0, ws_f32 = 0, ws_b = 0;   // proj_spatial: fp16 mma.sync A fragments, fp32 [N][N], bias [N]
};

struct NB_HIDDEN InpW : NetW {
    size_t stem_w = 0, stem_b = 0, mask_bias = 0;   // patch.0 as fp32 [48][96] (fp16 precision), bias, mask_bias [96]
    GmlpW enc1, enc2[4], dec1;
    Lin down, up, toimg;
};

static size_t pack_f32(Packer& pk, const std::string& name, int64_t n, bool f16_precision = false) {
    const float* p = pk.get(name, n);
    if (!p) return 0;
    std::vector<float> v(p, p + n);
    if (f16_precision)
        for (auto& x : v) x = round_f16(x);
    return pk.add_f32(v);
}

static GmlpW pack_gmlp(Packer& pk, const std::string& p, int C, int ws, bool shift) {
    GmlpW b;
    b.C = C; b.ws = ws; b.shift = shift; b.cpad = (C / 2 + 31) / 32 * 32;
    const std::string g = p + ".gmlp.gmlp";
    b.pin = pack_linear(pk, g + ".proj_in", 4 * C, C);
    b.pout = pack_linear(pk, g + ".proj_out", C, 2 * C);
    b.w1 = pack_conv(pk, p + ".glu_conv.w1", C, C, 1, 1);
    b.w2 = pack_conv(pk, p + ".glu_conv.w2", C, C / 2, 3, 3, /*cin_pad=*/b.cpad);
    b.g1 = pack_f32(pk, p + ".norm1.weight", C);
    b.g2 = pack_f32(pk, p + ".norm2.weight", 2 * C);
    const int N = ws * ws;
    const float* w = pk.get(g + ".proj_spatial.weight", (int64_t)N * N);   // Conv1d(N, N, 1): [n][m][1]
    b.ws_b = pack_f32(pk, g + ".proj_spatial.bias", N);
    if (!w) return b;
    // A fragments of mma.sync m16n8k16 (row = n, k = m): [row tile][k tile][lane][8 halves] with the register order
    // a0 = (g, 2t..2t+1), a1 = (g+8, 2t..), a2 = (g, 2t+8..), a3 = (g+8, 2t+8..), g = lane/4, t = lane%4
    std::vector<float> frag((size_t)N * N);
    for (int mt = 0; mt < N / 16; ++mt)
        for (int kt = 0; kt < N / 16; ++kt)
            for (int lane = 0; lane < 32; ++lane)
                for (int e = 0; e < 8; ++e) {
                    const int r = mt * 16 + lane / 4 + ((e >> 1) & 1) * 8, k = kt * 16 + 2 * (lane % 4) + (e & 1) + (e >> 2) * 8;
                    frag[(((size_t)mt * (N / 16) + kt) * 32 + lane) * 8 + e] = w[(size_t)r * N + k];
                }
    b.ws_frag = pk.add_f16(frag);
    std::vector<float> wf(w, w + (size_t)N * N);
    for (auto& x : wf) x = round_f16(x);
    b.ws_f32 = pk.add_f32(wf);
    return b;
}

std::unique_ptr<NetW> pack_light_inpaint(Packer& pk) {
    auto w = std::make_unique<InpW>();
    const int C = 96;
    const float* pw = pk.get("patch.0.weight", 96 * 48);
    if (pw) {
        std::vector<float> t(48 * 96);
        for (int co = 0; co < 96; ++co)
            for (int k = 0; k < 48; ++k) t[(size_t)k * 96 + co] = round_f16(pw[(size_t)co * 48 + k]);
        w->stem_w = pk.add_f32(t);
    }
    w->stem_b = pack_f32(pk, "patch.0.bias", 96);
    w->mask_bias = pack_f32(pk, "mask_bias", 96);
    w->enc1 = pack_gmlp(pk, "enc1", C, 16, true);
    w->down = pack_conv(pk, "down", 2 * C, C, 2, 2);
    for (int i = 0; i < 4; ++i) w->enc2[i] = pack_gmlp(pk, "enc2." + std::to_string(i), 2 * C, 8, i % 2 == 1);
    w->up = pack_linear_pixshuf2(pk, "up", C, 2 * C);
    w->dec1 = pack_gmlp(pk, "dec1", C, 16, false);
    w->toimg = pack_conv(pk, "to_image.1", 48, C, 3, 3);
    return w;
}

struct InpBufs { __half *T, *U, *H1, *P; };

// x [B][H][W][C] in place.  The shifted block zero-pads by ws/2 (attention.py:673-691: F.pad, not a roll); the ring tokens go
// through LN1 (= 0), proj_in and the token mixing like every other token and are cropped before proj_out.
// tap: debug tap ids tap + 0..7 (block input, T, U, U after the token mixing, X after proj_out, H1, P, block output).
static int gmlp_block(cudaStream_t st, const nb200_model* m, const GmlpW& w, __half* X, int B, int H, int W, const InpBufs& bf,
                      int tap) {
    const int C = w.C, p = w.shift ? w.ws / 2 : 0, Hq = H + 2 * p, Wq = W + 2 * p;
    const size_t tok = (size_t)B * H * W, tokq = (size_t)B * Hq * Wq;
    if (tap_copy(st, tap + 0, X, tok * C * 2)) return 1;
    if (inpaint_ln_pad(st, X, m->at<float>(w.g1), bf.T, B, H, W, C, p)) return 1;   // also X <- 2X (GMLP's own shortcut + the block's)
    if (tap_copy(st, tap + 1, bf.T, tokq * C * 2)) return 1;
    if (linear_flat(st, m, w.pin, bf.T, (long long)B * Hq * Wq, C, bf.U, 4 * C, ACT_GELU)) return 1;
    if (tap_copy(st, tap + 2, bf.U, tokq * 4 * C * 2)) return 1;
    if (inpaint_token_mix(st, bf.U, B, Hq, Wq, C, w.ws, m->at<__half>(w.ws_frag), m->at<float>(w.ws_f32), m->at<float>(w.ws_b),
                          m->at<float>(w.g2))) return 1;
    if (tap_copy(st, tap + 3, bf.U, tokq * 4 * C * 2)) return 1;
    {   // proj_out on the cropped u * v' view + 2x
        ConvGemm g;
        g.A = bf.U + ((size_t)p * Wq + p) * 4 * C; g.B = B; g.Hi = H; g.Wi = W; g.Ci = 4 * C; g.Cin = 2 * C;
        g.a_row_stride = (long long)Wq * 4 * C; g.a_img_stride = (long long)Hq * Wq * 4 * C; g.kind = CG_LINEAR_2D;
        g.Wt = m->at<__half>(w.pout.w); g.N = C; g.bias = m->at<float>(w.pout.b); g.out = X; g.ldo = C;
        g.res = X; g.ldr = C; g.res_H = H; g.res_W = W;
        if (conv_gemm(st, g)) return 1;
    }
    if (tap_copy(st, tap + 4, X, tok * C * 2)) return 1;
    // GLUConvMLP (light_inpaint_v1.py:15-34): 1x1, GLU into a replicate-padded buffer, valid 3x3 + residual
    if (linear_flat(st, m, w.w1, X, (long long)B * H * W, C, bf.H1, C, ACT_NONE)) return 1;
    if (tap_copy(st, tap + 5, bf.H1, tok * C * 2)) return 1;
    if (inpaint_pad(st, bf.H1, B, H, W, C, w.cpad, 1, bf.P)) return 1;
    if (tap_copy(st, tap + 6, bf.P, (size_t)B * (H + 2) * (W + 2) * w.cpad * 2)) return 1;
    ConvGemm g;
    g.A = bf.P; g.B = B; g.Hi = H + 2; g.Wi = W + 2; g.Ci = w.cpad; g.Cin = w.cpad; g.kind = CG_CONV3; g.pad = 0;
    g.Wt = m->at<__half>(w.w2.w); g.N = C; g.bias = m->at<float>(w.w2.b); g.out = X; g.ldo = C;
    g.res = X; g.ldr = C; g.res_H = H; g.res_W = W;
    if (conv_gemm(st, g)) return 1;
    return tap_copy(st, tap + 7, X, tok * C * 2);
}

// LightInpaintV1.infer(x, mask) (light_inpaint_v1.py:88-154): x [B][3][H][W] (the warped eye), hole [B][1][H][W] (the prepared
// binary mask), both in image coordinates; mirror = forward_left's flip of both and of the result.
// Debug taps (nb200_debug_tap; the id table is in DESIGN.md §5): 100 blur, 101 stem output, 110 + 10k + s stage s of GMLP block k
// (0 enc1, 1..4 enc2, 5 dec1), 170 down, 171 up + skip, 172 to_image's padded input, 173 to_image output.
static int light_inpaint_forward(nb200_model* m, const InpW& w, cudaStream_t st, const float* x, const float* hole, int B, int H, int W,
                                 int mirror, float* out) {
    const int Hp = H + 64 - H % 64, Wp = W + 64 - W % 64;   // light_inpaint_v1.py:134-139: 64 (not 0) when already a multiple
    const int H4 = Hp / 4, W4 = Wp / 4, H8 = H4 / 2, W8 = W4 / 2;
    const size_t t4 = (size_t)B * H4 * W4, t8 = (size_t)B * H8 * W8;
    const size_t q4 = (size_t)B * (H4 + 16) * (W4 + 16), q8 = (size_t)B * (H8 + 8) * (W8 + 8);
    const size_t px = (size_t)B * H * W;
    const size_t eT = std::max(q4 * 96, q8 * 192), eU = 4 * eT, eH = std::max(t4 * 96, t8 * 192);
    const size_t eP = std::max((size_t)B * (H4 + 2) * (W4 + 2) * 96, (size_t)B * (H8 + 2) * (W8 + 2) * 96);
    float *blur, *tmp;
    __half *X1, *X2, *X5, *Y;
    InpBufs bf;
    if (m->carve([&](Arena& a) {
            blur = a.take<float>(px);
            tmp = a.take<float>(px);
            X1 = a.take<__half>(t4 * 96);
            X2 = a.take<__half>(t8 * 192);
            X5 = a.take<__half>(t4 * 96);
            bf = {a.take<__half>(eT), a.take<__half>(eU), a.take<__half>(eH), a.take<__half>(eP)};
            Y = a.take<__half>(t4 * 48);
        })) return 1;

    if (inpaint_blur(st, hole, B, H, W, mirror, tmp, blur)) return 1;
    if (tap_copy(st, 100, blur, px * 4)) return 1;
    if (inpaint_stem(st, x, hole, blur, B, H, W, Hp, Wp, mirror, m->at<float>(w.stem_w), m->at<float>(w.stem_b),
                     m->at<float>(w.mask_bias), X1)) return 1;
    if (tap_copy(st, 101, X1, t4 * 96 * 2)) return 1;
    if (gmlp_block(st, m, w.enc1, X1, B, H4, W4, bf, 110)) return 1;
    {   // down: conv 2x2 s2
        ConvGemm g;
        g.A = X1; g.B = B; g.Hi = H4; g.Wi = W4; g.Ci = 96; g.Cin = 96; g.kind = CG_DOWN2;
        g.Wt = m->at<__half>(w.down.w); g.N = 192; g.bias = m->at<float>(w.down.b); g.out = X2; g.ldo = 192;
        if (conv_gemm(st, g)) return 1;
    }
    if (tap_copy(st, 170, X2, t8 * 192 * 2)) return 1;
    for (int i = 0; i < 4; ++i) if (gmlp_block(st, m, w.enc2[i], X2, B, H8, W8, bf, 120 + 10 * i)) return 1;
    {   // up (1x1 192 -> 384) + pixel_shuffle(2) + x1
        ConvGemm g;
        g.A = X2; g.B = B; g.Hi = H8; g.Wi = W8; g.Ci = 192; g.Cin = 192; g.kind = CG_LINEAR_2D;
        g.Wt = m->at<__half>(w.up.w); g.N = w.up.N; g.bias = m->at<float>(w.up.b); g.out = X5; g.ldo = 96;
        g.out_mode = OUT_PIXSHUF2; g.cout = 96; g.res = X1; g.ldr = 96; g.res_H = H4; g.res_W = W4;
        if (conv_gemm(st, g)) return 1;
    }
    if (tap_copy(st, 171, X5, t4 * 96 * 2)) return 1;
    if (gmlp_block(st, m, w.dec1, X5, B, H4, W4, bf, 160)) return 1;
    // to_image: replicate pad 1 + valid 3x3 96 -> 48, then pixel_shuffle(4), crop and composite in the tail
    if (inpaint_pad(st, X5, B, H4, W4, 96, 96, 0, bf.P)) return 1;
    if (tap_copy(st, 172, bf.P, (size_t)B * (H4 + 2) * (W4 + 2) * 96 * 2)) return 1;
    {
        ConvGemm g;
        g.A = bf.P; g.B = B; g.Hi = H4 + 2; g.Wi = W4 + 2; g.Ci = 96; g.Cin = 96; g.kind = CG_CONV3; g.pad = 0;
        g.Wt = m->at<__half>(w.toimg.w); g.N = 48; g.bias = m->at<float>(w.toimg.b); g.out = Y; g.ldo = 48;
        if (conv_gemm(st, g)) return 1;
    }
    if (tap_copy(st, 173, Y, t4 * 48 * 2)) return 1;
    return inpaint_tail(st, Y, x, hole, blur, B, H, W, Hp, Wp, mirror, out);
}

}  // namespace nb200

using namespace nb200;

// iw3/dilation.py:67-98: n = max(round(W / base_width * n_iter), 1) (Python's round: half to even), 0 when n_iter <= 0
static int dilation_run(int n_iter, int base_width, int W) {
    if (n_iter <= 0) return 0;
    if (base_width <= 0) return n_iter;
    const double n = std::nearbyint((double)W / base_width * n_iter);
    return n < 1 ? 1 : (int)n;
}

extern "C" int nb200_inpaint_mask(const float* mask, int B, int H, int W, int binarize, int closing, int outer_iter, int inner_iter,
                                  int base_width, int mirror, float* out, void* stream) {
    NB_CHECK(mask && out, "null pointer");
    NB_CHECK(B > 0 && H > 0 && W > 0, "empty mask");
    const int no = dilation_run(outer_iter, base_width, W), ni = dilation_run(inner_iter, base_width, W);
    cudaStream_t st = (cudaStream_t)stream;
    float* tmp = nullptr;
    if (closing) NB_CUDA(cudaMallocAsync((void**)&tmp, (size_t)B * H * W * 4, st));
    // in image coordinates the mirrored mask's right-hand runs (dilate_outer) grow to the left
    const int rc = inpaint_mask(st, mask, B, H, W, binarize, closing, mirror ? ni : no, mirror ? no : ni, tmp, out);
    if (tmp) cudaFreeAsync(tmp, st);
    return rc;
}

extern "C" int nb200_inpaint_blur(const float* mask, int B, int H, int W, float* out, void* stream) {
    NB_CHECK(mask && out, "null pointer");
    NB_CHECK(B > 0 && H > 0 && W > 0, "empty mask");
    cudaStream_t st = (cudaStream_t)stream;
    float* tmp = nullptr;
    NB_CUDA(cudaMallocAsync((void**)&tmp, (size_t)B * H * W * 4, st));
    const int rc = inpaint_blur(st, mask, B, H, W, 0, tmp, out);
    cudaFreeAsync(tmp, st);
    return rc;
}

extern "C" int nb200_light_inpaint(nb200_model* m, const float* x, const float* mask, int B, int H, int W, int mirror, float* out,
                                   void* stream) {
    NB_CHECK(m && x && mask && out, "null pointer");
    const InpW* w = net_as<InpW>(m);
    NB_CHECK(w, "model is not inpaint.light_inpaint_v1");
    NB_CHECK(B > 0 && H > 0 && W > 0, "empty input");
    return light_inpaint_forward(m, *w, (cudaStream_t)stream, x, mask, B, H, W, mirror, out);
}
