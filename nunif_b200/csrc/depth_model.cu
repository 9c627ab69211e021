// The ViT encoder + DPT head that Depth-Anything and ZoeD_N / ZoeD_Any (zoe_model.cu) share, and the Depth-Anything V2 / V1
// (DINOv2 ViT encoder + DPT head) container: weight packing from the upstream state_dict keys (`pretrained.*`, `depth_head.*`;
// what torch.hub "nagadomi/Depth-Anything_iw3" DepthAnything(encoder="v2_vits") loads, iw3/depth_anything_model.py:223-230) and the
// forward pass as a sequence of wgmma GEMMs and the kernels in depth_kernels.cu.  Restated architecture + parity anchor:
// oracle/depth_anything.py.
//
// Shared through vit_dpt.h: the pre-norm ViT block and the encoder loop over the fp32 residual stream (with an optional per-layer
// attention bias, and the hooked hidden states either through the final LayerNorm or cast to fp16), the DPT neck (readout
// "ignore" or "project", reassemble, layerN_rn, the four fusion blocks, output_conv) and its workspace.  Model-specific:
// the patch embedding, the token assembly and the position encoding.
//
// Pack-time algebra (exact in real arithmetic, fewer roundings than the reference's fp16 intermediates):
//   * LayerScale folded into the producing Linear:  gamma * (W x + b) = (gamma . W) x + gamma . b
//   * DPT "projects[i]" (1x1 conv) folded into the following ConvTranspose2d (k = s = 4 or 2): both are linear per pixel
// The residual stream is fp32 (as in the reference under autocast, where cat([cls fp32, tokens fp16]) promotes it);
// every Linear emits an fp16 delta that the fused add+LayerNorm kernel accumulates.
#include "vit_dpt.h"
#include "gemm.h"
#include "depth_kernels.h"
#include "zoe_kernels.h"
#include <algorithm>
#include <cmath>

namespace nb200 {

// Linear [N][K] with a per-output scale folded in (LayerScale)
static Lin pack_linear_scaled(Packer& pk, const std::string& name, int N, int K, const std::string& gamma_name) {
    Lin l;
    l.N = N; l.K = K;
    const float* w = pk.get(name + ".weight", (int64_t)N * K);
    const float* b = pk.get(name + ".bias", N);
    const float* g = pk.get(gamma_name, N);
    if (!w || !b || !g) return l;
    std::vector<float> wv((size_t)N * K), bv(N);
    for (int n = 0; n < N; ++n) {
        for (int k = 0; k < K; ++k) wv[(size_t)n * K + k] = g[n] * w[(size_t)n * K + k];
        bv[n] = g[n] * b[n];
    }
    l.w = pk.add_f16(wv);
    l.b = pk.add_f32(bv);
    return l;
}

// projects[i] (Conv2d dim->c, k1) followed by ConvTranspose2d(c, c, k=r, s=r): one Linear dim -> r*r*c,
// rows n = (dy*r + dx)*c + co
static Lin pack_project_convT(Packer& pk, const std::string& proj, const std::string& convt, int dim, int c, int r) {
    Lin l;
    l.N = r * r * c; l.K = dim;
    const float* wp = pk.get(proj + ".weight", (int64_t)c * dim);
    const float* bp = pk.get(proj + ".bias", c);
    const float* wt = pk.get(convt + ".weight", (int64_t)c * c * r * r);   // [cin][cout][r][r]
    const float* bt = pk.get(convt + ".bias", c);
    if (!wp || !bp || !wt || !bt) return l;
    std::vector<float> wv((size_t)l.N * dim, 0.f), bv(l.N, 0.f);
    for (int g = 0; g < r * r; ++g)
        for (int co = 0; co < c; ++co) {
            float* row = &wv[((size_t)g * c + co) * dim];
            double bacc = bt[co];
            for (int m = 0; m < c; ++m) {
                const float t = wt[((size_t)m * c + co) * r * r + g];
                bacc += (double)t * bp[m];
                const float* src = wp + (size_t)m * dim;
                for (int k = 0; k < dim; ++k) row[k] += t * src[k];
            }
            bv[g * c + co] = (float)bacc;
        }
    l.w = pk.add_f16(wv);
    l.b = pk.add_f32(bv);
    return l;
}

// Conv2d without bias (scratch.layerN_rn)
static Lin pack_conv_nobias(Packer& pk, const std::string& name, int cout, int cin, int cin_pad) {
    Lin l;
    l.N = cout; l.K = 9 * cin_pad;
    const float* w = pk.get(name + ".weight", (int64_t)cout * cin * 9);
    if (!w) return l;
    std::vector<float> wv((size_t)cout * l.K, 0.f), bv(cout, 0.f);
    for (int co = 0; co < cout; ++co)
        for (int ci = 0; ci < cin; ++ci)
            for (int k = 0; k < 9; ++k) wv[(size_t)co * l.K + (size_t)k * cin_pad + ci] = w[((size_t)co * cin + ci) * 9 + k];
    l.w = pk.add_f16(wv);
    l.b = pk.add_f32(bv);
    return l;
}

VitBlockW pack_vit_block(Packer& pk, const std::string& p, int dim, const Lin& qkv, const char* gamma1, const char* gamma2) {
    VitBlockW b;
    b.qkv = qkv;
    b.n1w = pack_vec_f32(pk, p + "norm1.weight", dim);
    b.n1b = pack_vec_f32(pk, p + "norm1.bias", dim);
    b.proj = pack_linear_scaled(pk, p + "attn.proj", dim, dim, p + gamma1);
    b.n2w = pack_vec_f32(pk, p + "norm2.weight", dim);
    b.n2b = pack_vec_f32(pk, p + "norm2.bias", dim);
    b.fc1 = pack_linear(pk, p + "mlp.fc1", 4 * dim, dim);
    b.fc2 = pack_linear_scaled(pk, p + "mlp.fc2", dim, 4 * dim, p + gamma2);
    return b;
}

void pack_dpt(Packer& pk, DptW& d, int dim, const DptKeys& k) {
    d.c0pad = (d.oc[0] + 31) / 32 * 32;
    for (int i = 0; i < 4; ++i)
        if (!k.readout[i].empty()) d.readout[i] = pack_linear(pk, k.readout[i], dim, 2 * dim);
    d.reasm[0] = pack_project_convT(pk, k.project[0], k.resize[0], dim, d.oc[0], 4);
    d.reasm[1] = pack_project_convT(pk, k.project[1], k.resize[1], dim, d.oc[1], 2);
    d.reasm[2] = pack_conv(pk, k.project[2], d.oc[2], dim, 1, 1);
    d.reasm[3] = pack_conv(pk, k.project[3], d.oc[3], dim, 1, 1);
    d.resize3 = pack_conv(pk, k.resize[3], d.oc[3], d.oc[3], 3, 3);
    for (int i = 0; i < 4; ++i)
        d.rn[i] = pack_conv_nobias(pk, k.scratch + "layer" + std::to_string(i + 1) + "_rn", d.feat, d.oc[i], i == 0 ? d.c0pad : d.oc[i]);
    for (int r = 0; r < 4; ++r) {
        const std::string p = k.scratch + "refinenet" + std::to_string(r + 1) + ".";
        d.ref[r].out_conv = pack_conv(pk, p + "out_conv", d.feat, d.feat, 1, 1);
        for (int u = 0; u < 2; ++u)
            for (int c = 0; c < 2; ++c) {
                const std::string cn = p + "resConfUnit" + std::to_string(u + 1) + ".conv" + std::to_string(c + 1);
                if (r == 3 && u == 0) {   // refinenet4 has no second input: its resConfUnit1 is never evaluated
                    pk.mark(cn + ".weight");
                    pk.mark(cn + ".bias");
                    continue;
                }
                d.ref[r].c[u][c] = pack_conv(pk, cn, d.feat, d.feat, 3, 3);
            }
    }
    d.oc1 = pack_conv(pk, k.out_conv[0], d.feat / 2, d.feat, 3, 3);
    d.oc2 = pack_conv(pk, k.out_conv[1], 32, d.feat / 2, 3, 3);
    d.oc3w = pack_vec_f32(pk, k.out_conv[2] + ".weight", 32);
    if (const float* b3 = pk.get(k.out_conv[2] + ".bias", 1)) d.oc3b = b3[0];
}

int64_t key_numel(Packer& pk, const std::string& name) {
    auto it = pk.src.find(name);
    if (it == pk.src.end()) {
        if (pk.err.empty()) pk.err = "missing key in state_dict: " + name;
        return 0;
    }
    return it->second.numel;
}

std::unique_ptr<DaW> pack_dinov2_dpt(Packer& pk, int encoder, const std::string& pre, bool last4) {
    struct Cfg { int dim, depth, heads, feat, oc[4], hooks[4]; };
    static const Cfg cfg[3] = {
        {384, 12, 6, 64, {48, 96, 192, 384}, {2, 5, 8, 11}},
        {768, 12, 12, 128, {96, 192, 384, 768}, {2, 5, 8, 11}},
        {1024, 24, 16, 256, {256, 512, 1024, 1024}, {4, 11, 17, 23}},
    };
    auto d = std::make_unique<DaW>();
    DaW& w = *d;
    const std::string enc = pre + "pretrained.", h = pre + "depth_head.";
    Cfg c{};
    if (encoder >= 0) {
        c = cfg[encoder];
    } else {
        c.dim = (int)key_numel(pk, enc + "cls_token");
        c.heads = c.dim / 64;                                              // DINOv2: head dim 64 in every size
        while (pk.src.count(enc + "blocks." + std::to_string(c.depth) + ".norm1.weight")) ++c.depth;
        for (int i = 0; i < 4; ++i) c.oc[i] = (int)key_numel(pk, h + "projects." + std::to_string(i) + ".bias");
        if (!pk.err.empty()) return d;
        c.feat = (int)(key_numel(pk, h + "scratch.layer1_rn.weight") / ((int64_t)c.oc[0] * 9));
        if (c.dim < 64 || c.dim % 64) { pk.err = "Depth-Anything: embedding dim must be a multiple of 64 (head dim 64)"; return d; }
        if (c.depth < 4) { pk.err = "Depth-Anything: the encoder needs at least 4 blocks"; return d; }
        if (c.feat < 64 || c.feat % 64) { pk.err = "Depth-Anything: fusion width must be a multiple of 64"; return d; }
        for (int i = 1; i < 4; ++i)
            if (c.oc[i] % 32) { pk.err = "Depth-Anything: reassemble widths 1..3 must be multiples of 32"; return d; }
    }
    if (last4)
        for (int i = 0; i < 4; ++i) c.hooks[i] = c.depth - 4 + i;
    const int dim = c.dim;
    w.vit.dim = dim; w.vit.depth = c.depth; w.vit.heads = c.heads;
    w.dpt.feat = c.feat;
    for (int i = 0; i < 4; ++i) { w.dpt.oc[i] = c.oc[i]; w.vit.hooks[i] = c.hooks[i]; }
    {   // patch embedding: Conv2d(3, dim, 14, 14) as a Linear over im2col rows, K = 588 zero-padded to 640
        Lin l;
        l.N = dim; l.K = w.kpad;
        const float* pw = pk.get(enc + "patch_embed.proj.weight", (int64_t)dim * 588);
        const float* pb = pk.get(enc + "patch_embed.proj.bias", dim);
        if (pw && pb) {
            std::vector<float> wv((size_t)dim * w.kpad, 0.f);
            for (int n = 0; n < dim; ++n) memcpy(&wv[(size_t)n * w.kpad], pw + (size_t)n * 588, 588 * 4);
            l.w = pk.add_f16(wv);
            l.b = pk.add_f32(std::vector<float>(pb, pb + dim));
        }
        w.patch = l;
    }
    w.cls = pack_vec_f32(pk, enc + "cls_token", dim);
    pk.mark(enc + "mask_token");
    {
        auto it = pk.src.find(enc + "pos_embed");
        if (it == pk.src.end()) { if (pk.err.empty()) pk.err = "missing key in state_dict: " + enc + "pos_embed"; }
        else {
            const int64_t rows = it->second.numel / dim;
            const int g = (int)std::lround(std::sqrt((double)(rows - 1)));
            if (rows < 2 || (int64_t)g * g + 1 != rows || it->second.numel % dim) { if (pk.err.empty()) pk.err = enc + "pos_embed must be [1, 1+g*g, dim]"; }
            else {
                w.pos_grid = g;
                w.pos_host.assign(it->second.data, it->second.data + it->second.numel);
                it->second.used = true;
            }
        }
    }
    for (int i = 0; i < c.depth; ++i) {
        const std::string p = enc + "blocks." + std::to_string(i) + ".";
        w.vit.blocks.push_back(pack_vit_block(pk, p, dim, pack_linear(pk, p + "attn.qkv", 3 * dim, dim), "ls1.gamma", "ls2.gamma"));
    }
    // get_intermediate_layers(..., norm=True): the final LayerNorm applied to every hooked block output
    w.vit.hook_norm = true;
    w.vit.normw = pack_vec_f32(pk, enc + "norm.weight", dim);
    w.vit.normb = pack_vec_f32(pk, enc + "norm.bias", dim);
    DptKeys k;
    for (int i = 0; i < 4; ++i) {
        k.project[i] = h + "projects." + std::to_string(i);
        k.resize[i] = h + "resize_layers." + std::to_string(i);
    }
    k.scratch = h + "scratch.";
    k.out_conv[0] = h + "scratch.output_conv1";
    k.out_conv[1] = h + "scratch.output_conv2.0";
    k.out_conv[2] = h + "scratch.output_conv2.2";
    pack_dpt(pk, w.dpt, dim, k);
    return d;
}

// dinov2 interpolate_pos_encoding (interpolate_offset 0.1): bicubic (A = -0.75, align_corners=False) resample of the
// grid x grid table with scale factors (ph+0.1)/grid, (pw+0.1)/grid; ATen upsample_bicubic2d arithmetic in fp32.
// table: the learned [1 + g*g][dim] (class row first) -> out [1 + ph*pw][dim]
static void interp_pos_table(const float* table, int g, int dim, int ph, int pw, float* out) {
    memcpy(out, table, (size_t)dim * 4);
    if (ph == g && pw == g) {
        memcpy(out + dim, table + dim, (size_t)g * g * dim * 4);
        return;
    }
    const float sy = (float)(1.0 / ((double)(ph + 0.1) / g)), sx = (float)(1.0 / ((double)(pw + 0.1) / g));
    auto cc1 = [](float x) { const float A = -0.75f; return ((A + 2.f) * x - (A + 3.f)) * x * x + 1.f; };
    auto cc2 = [](float x) { const float A = -0.75f; return ((A * x - 5.f * A) * x + 8.f * A) * x - 4.f * A; };
    auto clampi = [](int v, int hi) { return v < 0 ? 0 : (v > hi ? hi : v); };
    const float* tab = table + dim;
    for (int oy = 0; oy < ph; ++oy) {
        const float ry = sy * ((float)oy + 0.5f) - 0.5f;
        const int iy = (int)std::floor(ry);
        const float ty = ry - (float)iy;
        const float cy[4] = {cc2(ty + 1.f), cc1(ty), cc1(1.f - ty), cc2((1.f - ty) + 1.f)};
        for (int ox = 0; ox < pw; ++ox) {
            const float rx = sx * ((float)ox + 0.5f) - 0.5f;
            const int ix = (int)std::floor(rx);
            const float tx = rx - (float)ix;
            const float cx[4] = {cc2(tx + 1.f), cc1(tx), cc1(1.f - tx), cc2((1.f - tx) + 1.f)};
            float* dst = out + (size_t)(1 + oy * pw + ox) * dim;
            for (int c = 0; c < dim; ++c) {
                float acc = 0.f;
                for (int a = 0; a < 4; ++a) {
                    const float* row = tab + (size_t)clampi(iy - 1 + a, g - 1) * g * dim;
                    float h = 0.f;
                    for (int b = 0; b < 4; ++b) h += row[(size_t)clampi(ix - 1 + b, g - 1) * dim + c] * cx[b];
                    acc += h * cy[a];
                }
                dst[c] = acc;
            }
        }
    }
}

int da_linear(cudaStream_t st, const nb200_model* m, const Lin& l, const __half* A, long long M, int lda, __half* out, int act) {
    return linear_flat(st, m, l, A, M, lda, out, l.N, act);
}

int da_conv(cudaStream_t st, const nb200_model* m, const Lin& l, const __half* A, int B, int H, int W, int Ci, int Cin, __half* out,
                   int act, const __half* res, bool k3) {
    ConvGemm g;
    g.A = A; g.B = B; g.Hi = H; g.Wi = W; g.Ci = Ci; g.Cin = Cin; g.kind = k3 ? CG_CONV3 : CG_LINEAR_2D; g.pad = k3 ? 1 : 0;
    g.Wt = m->at<__half>(l.w); g.N = l.N; g.bias = m->at<float>(l.b); g.act = act; g.out = out; g.ldo = l.N;
    if (res) { g.res = res; g.ldr = l.N; g.res_H = H; g.res_W = W; }
    return conv_gemm(st, g);
}

// FeatureFusionBlock (dpt blocks.py): x0 (+ resConfUnit1(x1)) -> resConfUnit2 -> bilinear resize -> out_conv
static int da_fusion(cudaStream_t st, const nb200_model* m, const DaRefineW& r, int F, const __half* x0, const __half* x1, int B, int h, int w,
                     int oh, int ow, __half* t_relu, __half* t_c1, __half* t_sum, __half* t_u, __half* t_up, __half* out) {
    const long long n = (long long)B * h * w * F;
    const __half* cur = x0;
    if (x1) {
        // res = conv2(relu(conv1(relu(x1)))) + x1 ; output = x0 + res  ==  conv2(...) + (x0 + x1)
        if (da_relu_add(st, x1, x0, t_relu, t_sum, n)) return 1;
        if (da_conv(st, m, r.c[0][0], t_relu, B, h, w, F, F, t_c1, ACT_RELU, nullptr, true)) return 1;
        if (da_conv(st, m, r.c[0][1], t_c1, B, h, w, F, F, t_u, ACT_NONE, t_sum, true)) return 1;
        cur = t_u;
    }
    if (da_relu_add(st, cur, nullptr, t_relu, nullptr, n)) return 1;
    if (da_conv(st, m, r.c[1][0], t_relu, B, h, w, F, F, t_c1, ACT_RELU, nullptr, true)) return 1;
    __half* u2 = cur == t_u ? t_sum : t_u;   // t_sum is free again once the first unit has consumed it
    if (da_conv(st, m, r.c[1][1], t_c1, B, h, w, F, F, u2, ACT_NONE, cur, true)) return 1;
    if (da_upsample_bilinear(st, u2, B, h, w, F, t_up, oh, ow)) return 1;
    return da_conv(st, m, r.out_conv, t_up, B, oh, ow, F, F, out, ACT_NONE, nullptr, false);
}

DptGeom dpt_geom(int B, int H, int W, int patch) {
    DptGeom g;
    g.B = B; g.H = H; g.W = W; g.ph = H / patch; g.pw = W / patch; g.P = g.ph * g.pw; g.N = g.P + 1;
    const int lh[4] = {4 * g.ph, 2 * g.ph, g.ph, (g.ph + 1) / 2}, lw[4] = {4 * g.pw, 2 * g.pw, g.pw, (g.pw + 1) / 2};
    for (int i = 0; i < 4; ++i) { g.lh[i] = lh[i]; g.lw[i] = lw[i]; }
    g.hp = 2 * g.lh[0]; g.wp = 2 * g.lw[0];
    return g;
}

void dpt_plan(Arena& a, const VitW& v, const DptW& d, const DptGeom& g, DptBufs& b) {
    const size_t B = g.B, M = B * g.N, dim = v.dim, F = d.feat, npix = B * g.H * g.W;
    const bool readout = d.readout[0].N != 0;
    const size_t c0 = d.oc[0], c3 = d.oc[3], lv0 = B * g.lh[0] * g.lw[0], lv3 = B * g.lh[3] * g.lw[3], lvp = B * g.hp * g.wp;
    b.T = a.take<__half>(B * g.P * std::max(16 * c0, readout ? 2 * dim : dim));
    b.X32 = a.take<float>(M * dim);
    b.Hn = a.take<__half>(M * dim);
    b.QKV = a.take<__half>(M * 3 * dim);
    b.ATT = a.take<__half>(M * dim);
    b.HID = a.take<__half>(M * 4 * dim);
    b.D = a.take<__half>(M * dim);
    for (int i = 0; i < 4; ++i) b.FE[i] = a.take<__half>(M * dim);
    b.Y = readout ? a.take<__half>(B * g.P * dim) : nullptr;
    b.L[0] = a.take<__half>(lv0 * d.c0pad);
    for (int i = 1; i < 3; ++i) b.L[i] = a.take<__half>(B * g.lh[i] * g.lw[i] * d.oc[i]);
    b.L4lin = a.take<__half>(B * g.lh[2] * g.lw[2] * c3);
    b.L4col = a.take<__half>(lv3 * 9 * c3);
    b.L[3] = a.take<__half>(lv3 * c3);
    for (int i = 0; i < 4; ++i) b.R[i] = a.take<__half>(B * g.lh[i] * g.lw[i] * F);
    // fusion temporaries at the largest fusion resolution
    b.t_relu = a.take<__half>(lv0 * F);
    b.t_c1 = a.take<__half>(lv0 * F);
    b.t_sum = a.take<__half>(lv0 * F);
    b.t_u = a.take<__half>(lv0 * F);
    b.t_up = a.take<__half>(lvp * F);
    for (int i = 0; i < 3; ++i) b.PATH[i] = a.take<__half>(B * g.lh[2 - i] * g.lw[2 - i] * F);
    b.PATH[3] = a.take<__half>(lvp * F);
    b.O1 = a.take<__half>(lvp * (F / 2));
    b.O1u = a.take<__half>(npix * (F / 2));
    b.O2 = a.take<__half>(npix * 32);
}

int vit_encoder(cudaStream_t st, const nb200_model* m, const VitW& v, const DptBufs& b, const DptGeom& g, const float* bias,
                       size_t bias_layer, int ldb) {
    const int dim = v.dim;
    const long long M = (long long)g.B * g.N;
    const __half* pending = nullptr;
    int nf = 0;
    for (int i = 0; i < v.depth; ++i) {
        const VitBlockW& k = v.blocks[i];
        if (da_add_layernorm(st, b.X32, pending, m->at<float>(k.n1w), m->at<float>(k.n1b), b.Hn, M, dim)) return 1;
        if (da_linear(st, m, k.qkv, b.Hn, M, dim, b.QKV, ACT_NONE)) return 1;
        if (da_attention(st, b.QKV, b.ATT, g.B, g.N, v.heads, bias ? bias + (size_t)i * bias_layer : nullptr, bias ? ldb : 0)) return 1;
        if (da_linear(st, m, k.proj, b.ATT, M, dim, b.D, ACT_NONE)) return 1;                 // LayerScale 1 folded
        if (da_add_layernorm(st, b.X32, b.D, m->at<float>(k.n2w), m->at<float>(k.n2b), b.Hn, M, dim)) return 1;
        if (da_linear(st, m, k.fc1, b.Hn, M, dim, b.HID, ACT_GELU)) return 1;
        if (da_linear(st, m, k.fc2, b.HID, M, 4 * dim, b.D, ACT_NONE)) return 1;              // LayerScale 2 folded
        pending = b.D;
        if (nf < 4 && i == v.hooks[nf]) {
            if (v.hook_norm) {
                if (da_add_layernorm(st, b.X32, b.D, m->at<float>(v.normw), m->at<float>(v.normb), b.FE[nf], M, dim)) return 1;
            } else {
                if (zoe_add_cast(st, b.X32, b.D, b.FE[nf], M * dim)) return 1;
            }
            pending = nullptr;
            ++nf;
        }
    }
    return 0;
}

int dpt_fuse(cudaStream_t st, const nb200_model* m, const DptW& d, int dim, const DptBufs& b, const DptGeom& g) {
    const int B = g.B, F = d.feat, c3 = d.oc[3];
    auto reassemble = [&](int i, __half* out, int out_mode, int cout) {
        ConvGemm c;
        if (d.readout[i].N) {   // ProjectReadout: cat(token, cls) -> Linear -> GELU
            if (zoe_readout_concat(st, b.FE[i], B, g.P, dim, b.T)) return 1;
            if (da_linear(st, m, d.readout[i], b.T, (long long)B * g.P, 2 * dim, b.Y, ACT_GELU)) return 1;
            c.A = b.Y;
        } else {                // readout "ignore": the class token row of every image is skipped by the A view
            c.A = b.FE[i] + dim; c.a_row_stride = (long long)g.pw * dim; c.a_img_stride = (long long)g.N * dim;
        }
        c.B = B; c.Hi = g.ph; c.Wi = g.pw; c.Ci = dim; c.Cin = dim; c.kind = CG_LINEAR_2D;
        c.Wt = m->at<__half>(d.reasm[i].w); c.N = d.reasm[i].N; c.bias = m->at<float>(d.reasm[i].b); c.act = ACT_NONE;
        c.out = out; c.ldo = out_mode == OUT_PIXSHUF2 ? cout : d.reasm[i].N; c.out_mode = out_mode; c.cout = cout;
        return conv_gemm(st, c);
    };
    if (reassemble(0, b.T, 0, 0)) return 1;                                          // [B*P][16*c0]
    if (da_depth_to_space4(st, b.T, B, g.ph, g.pw, d.oc[0], b.L[0], d.c0pad)) return 1;   // [B][4ph][4pw][c0 -> c0pad]
    if (reassemble(1, b.L[1], OUT_PIXSHUF2, d.oc[1])) return 1;                      // [B][2ph][2pw][c1]
    if (reassemble(2, b.L[2], 0, 0)) return 1;
    if (reassemble(3, b.L4lin, 0, 0)) return 1;
    if (da_im2col_s2(st, b.L4lin, B, g.ph, g.pw, c3, b.L4col)) return 1;
    if (da_linear(st, m, d.resize3, b.L4col, (long long)B * g.lh[3] * g.lw[3], 9 * c3, b.L[3], ACT_NONE)) return 1;
    for (int i = 0; i < 4; ++i) {
        const int ci = i == 0 ? d.c0pad : d.oc[i];
        if (da_conv(st, m, d.rn[i], b.L[i], B, g.lh[i], g.lw[i], ci, ci, b.R[i], ACT_NONE, nullptr, true)) return 1;
    }
    // refinenet4 (R[3] alone) .. refinenet1 (+ R[0]); each fusion upsamples to the next level, the last one to hp x wp
    for (int j = 0; j < 4; ++j) {
        const int l = 3 - j, oh = l ? g.lh[l - 1] : g.hp, ow = l ? g.lw[l - 1] : g.wp;
        if (da_fusion(st, m, d.ref[l], F, j ? b.PATH[j - 1] : b.R[3], j ? b.R[l] : nullptr, B, g.lh[l], g.lw[l], oh, ow, b.t_relu,
                      b.t_c1, b.t_sum, b.t_u, b.t_up, b.PATH[j])) return 1;
    }
    return 0;
}

int dpt_output(cudaStream_t st, const nb200_model* m, const DptW& d, const DptBufs& b, const DptGeom& g, float* rel) {
    const int B = g.B, F = d.feat, F2 = d.feat / 2;
    if (da_conv(st, m, d.oc1, b.PATH[3], B, g.hp, g.wp, F, F, b.O1, ACT_NONE, nullptr, true)) return 1;
    if (da_upsample_bilinear(st, b.O1, B, g.hp, g.wp, F2, b.O1u, g.H, g.W)) return 1;
    if (da_conv(st, m, d.oc2, b.O1u, B, g.H, g.W, F2, F2, b.O2, ACT_RELU, nullptr, true)) return 1;
    return da_head_final(st, b.O2, (long long)B * g.H * g.W, 32, m->at<float>(d.oc3w), d.oc3b, rel);
}

int da_prepare_pos(DaW& w, cudaStream_t st, int ph, int pw) {
    if (w.pos_dev && w.pos_ph == ph && w.pos_pw == pw) return 0;
    std::vector<float> tab((size_t)(1 + ph * pw) * w.vit.dim);
    interp_pos_table(w.pos_host.data(), w.pos_grid, w.vit.dim, ph, pw, tab.data());
    if (w.pos_dev) cudaFree(w.pos_dev);
    w.pos_dev = nullptr;
    w.pos_ph = w.pos_pw = 0;
    NB_CUDA(cudaMalloc((void**)&w.pos_dev, tab.size() * 4));
    NB_CUDA(cudaMemcpyAsync(w.pos_dev, tab.data(), tab.size() * 4, cudaMemcpyHostToDevice, st));
    NB_CUDA(cudaStreamSynchronize(st));   // `tab` is a host temporary (once per token-grid shape)
    w.pos_ph = ph; w.pos_pw = pw;
    return 0;
}

int da_encode(cudaStream_t st, const nb200_model* m, const DaW& w, const float* x, const DptGeom& g, const DptBufs& b, __half* Apatch) {
    if (da_patch_im2col(st, x, g.B, g.H, g.W, Apatch, w.kpad)) return 1;
    if (da_linear(st, m, w.patch, Apatch, (long long)g.B * g.P, w.kpad, b.T, ACT_NONE)) return 1;
    if (da_assemble_tokens(st, b.T, m->at<float>(w.cls), w.pos_dev, b.X32, g.B, g.P, w.vit.dim)) return 1;
    return vit_encoder(st, m, w.vit, b, g, nullptr, 0, 0);
}

static int depth_anything_forward(nb200_model* m, DaW& w, cudaStream_t st, const float* x, int B, int H, int W, float* depth) {
    NB_CHECK(H % 14 == 0 && W % 14 == 0 && H >= 14 && W >= 14, "input height and width must be multiples of 14 (batch_preprocess)");
    const DptGeom g = dpt_geom(B, H, W, 14);
    if (da_prepare_pos(w, st, g.ph, g.pw)) return 1;
    __half* Apatch;
    DptBufs b;
    if (m->carve([&](Arena& a) {
            Apatch = a.take<__half>((size_t)B * g.P * w.kpad);
            dpt_plan(a, w.vit, w.dpt, g, b);
        })) return 1;
    if (da_encode(st, m, w, x, g, b, Apatch)) return 1;
    // ---- DPT head (dpt.py DPTHead.forward)
    if (dpt_fuse(st, m, w.dpt, w.vit.dim, b, g)) return 1;
    return dpt_output(st, m, w.dpt, b, g, depth);
}

std::unique_ptr<NetW> pack_depth_anything(Packer& pk, int encoder, bool v1) {
    return pack_dinov2_dpt(pk, encoder, "", v1);
}

}  // namespace nb200

using namespace nb200;

// DepthAnythingV2.forward (what DepthAnythingModel._forward calls, iw3/depth_anything_model.py:113-119)
extern "C" int nb200_depth_anything_forward(nb200_model* m, const float* x, int B, int H, int W, float* depth, void* stream) {
    NB_CHECK(m && x && depth, "null pointer");
    DaW* w = net_as<DaW>(m);
    NB_CHECK(w, "model is not a Depth-Anything network");
    NB_CHECK(B > 0, "empty batch");
    return depth_anything_forward(m, *w, (cudaStream_t)stream, x, B, H, W, depth);
}

// Host-only: the position table of a ph x pw token grid, as da_prepare_pos builds it for the forward (include/nunif_b200.h).
extern "C" int nb200_vit_pos_table_f32(const float* table, int grid, int dim, int ph, int pw, float* out) {
    NB_CHECK(table && out, "null pointer");
    NB_CHECK(grid > 0 && dim > 0 && ph > 0 && pw > 0, "bad shape");
    interp_pos_table(table, grid, dim, ph, pw, out);
    return 0;
}

// ---- test entry points of the encoder-edge and DPT kernels that only a model forward reaches otherwise
// (include/nunif_b200.h).  Every check runs before the first CUDA call.
extern "C" int nb200_da_patch_im2col_f16(const float* x, int B, int H, int W, int kpad, void* A, void* stream) {
    NB_CHECK(x && A, "null pointer");
    NB_CHECK(B > 0 && H > 0 && W > 0, "bad shape");
    NB_CHECK(H % 14 == 0 && W % 14 == 0, "height and width must be multiples of the 14-pixel patch");
    NB_CHECK(kpad >= 3 * 14 * 14, "kpad below the 588 patch columns");
    return da_patch_im2col((cudaStream_t)stream, x, B, H, W, (__half*)A, kpad);
}

extern "C" int nb200_zoe_patch_im2col_f16(const float* x, int B, int H, int W, void* A, void* stream) {
    NB_CHECK(x && A, "null pointer");
    NB_CHECK(B > 0 && H > 0 && W > 0, "bad shape");
    NB_CHECK(H % 16 == 0 && W % 16 == 0, "height and width must be multiples of the 16-pixel patch");
    return zoe_patch_im2col((cudaStream_t)stream, x, B, H, W, (__half*)A);
}

extern "C" int nb200_vit_assemble_tokens_f32(const void* T, const float* cls, const float* pos, float* x32, int B, int P, int dim,
                                             void* stream) {
    NB_CHECK(T && cls && x32, "null pointer");
    NB_CHECK(B > 0 && P > 0 && dim > 0, "bad shape");
    if (!pos) return zoe_assemble_tokens((cudaStream_t)stream, (const __half*)T, cls, x32, B, P, dim);
    return da_assemble_tokens((cudaStream_t)stream, (const __half*)T, cls, pos, x32, B, P, dim);
}

extern "C" int nb200_zoe_add_cast_f16(float* x32, const void* delta, void* out, long long n, void* stream) {
    NB_CHECK(x32 && out, "null pointer");
    NB_CHECK(n > 0, "bad shape");
    return zoe_add_cast((cudaStream_t)stream, x32, (const __half*)delta, (__half*)out, n);
}

extern "C" int nb200_zoe_readout_concat_f16(const void* F, int B, int P, int dim, void* A, void* stream) {
    NB_CHECK(F && A, "null pointer");
    NB_CHECK(B > 0 && P > 0 && dim > 0, "bad shape");
    return zoe_readout_concat((cudaStream_t)stream, (const __half*)F, B, P, dim, (__half*)A);
}

extern "C" int nb200_dpt_depth_to_space4_f16(const void* T, int B, int h, int w, int c, int cpad, void* out, void* stream) {
    NB_CHECK(T && out, "null pointer");
    NB_CHECK(B > 0 && h > 0 && w > 0 && c > 0, "bad shape");
    return da_depth_to_space4((cudaStream_t)stream, (const __half*)T, B, h, w, c, (__half*)out, cpad);
}

extern "C" int nb200_dpt_im2col_s2_f16(const void* x, int B, int h, int w, int C, void* A, void* stream) {
    NB_CHECK(x && A, "null pointer");
    NB_CHECK(B > 0 && h > 0 && w > 0 && C > 0, "bad shape");
    return da_im2col_s2((cudaStream_t)stream, (const __half*)x, B, h, w, C, (__half*)A);
}

extern "C" int nb200_dpt_relu_add_f16(const void* x, const void* x0, void* y, void* s, long long n, void* stream) {
    NB_CHECK(x && y, "null pointer");
    NB_CHECK(!x0 == !s, "x0 and s go together");
    NB_CHECK(n > 0, "bad shape");
    return da_relu_add((cudaStream_t)stream, (const __half*)x, (const __half*)x0, (__half*)y, (__half*)s, n);
}

extern "C" int nb200_dpt_head_final_f32(const void* x, long long npix, int C, const float* w, float bias, float* depth, void* stream) {
    NB_CHECK(x && w && depth, "null pointer");
    NB_CHECK(npix > 0, "bad shape");
    return da_head_final((cudaStream_t)stream, (const __half*)x, npix, C, w, bias, depth);
}
