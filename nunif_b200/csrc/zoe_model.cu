// ZoeD_N (BEiT-L/16 encoder + MiDaS DPT head + ZoeDepth metric bins head) container: weight packing from the upstream
// checkpoint keys of ZoeD_M12_N.pt (`core.core.pretrained.*`, `core.core.scratch.*`, `conv2`, `seed_bin_regressor`,
// `seed_projector`, `projectors`, `attractors`, `conditional_log_binomial`; what torch.hub "nagadomi/ZoeDepth_iw3" ZoeD_N
// loads, iw3/zoedepth_model.py:151-157) and the forward pass.  The BEiT encoder (with the relative-position bias in the flash
// attention) and the MiDaS DPT head (with the project readout) run on the ViT encoder and DPT neck shared with Depth-Anything
// in depth_model.cu (vit_dpt.h); this file holds what is ZoeD_N's own: the BEiT qkv and relative-position tables, the 16-px
// patch embedding, the token assembly and the metric bins head (zoe_kernels.cu).
// Restated architecture + parity anchor: oracle/zoedepth.py.
//
// The configuration (embedding dim, depth, DPT widths, training grid of the relative-position table) is read off the
// tensor sizes, so the reduced test configuration (synth.ZOED_MINI) runs the same code.
// Pack-time algebra as in depth_model.cu: gamma_1 / gamma_2 folded into attn.proj / mlp.fc2, act_postprocess{1,2}.3 (1x1 conv)
// folded into the following ConvTranspose2d; q_bias | 0 | v_bias become one qkv bias vector (BEiT has no key bias).
#include "vit_dpt.h"
#include "gemm.h"
#include "depth_kernels.h"
#include "zoe_kernels.h"
#include <cmath>

namespace nb200 {

// the metric bins head (zoedepth_v1.py: conv2, seed regressor, seed projector, 4 projector / attractor pairs, conditional
// log-binomial), shared by ZoeD_N and ZoeD_Any
struct ZoeBinsW {
    bool normed = false;      // bin_centers_type "normed" (ZoeD_Any_K: SeedBinRegressor + AttractorLayer), else "softplus"
    float min_depth = 1e-3f, max_depth = 10.f;
    int feat = 0;
    int ald = 16;             // row stride of the attractor pre-activation: n_attractors (softplus) or 2 n_attractors (normed), padded
    Lin conv2, seed1, seed2, sproj1, sproj2, proj1[4], proj2[4], att1[4], att2[4], clb1;
    size_t clb2w = 0, clb2b = 0;
    int n_att[4] = {16, 8, 4, 1};
};

struct NB_HIDDEN ZoeW : NetW {
    std::unique_ptr<DaW> da;  // ZoeD_Any: the Depth-Anything V1 encoder + DPT head (the BEiT fields below are then unused)
    int old_grid = 24;
    VitW vit;
    DptW dpt;
    Lin patch;
    size_t cls = 0;
    ZoeBinsW head;
    std::vector<std::vector<float>> tables;   // per block: learned relative_position_bias_table [(2g-1)^2 + 3][heads]
    // expanded bias of the last token grid: [depth][heads][N][ldb] fp32, log2(e) folded in
    int bias_ph = 0, bias_pw = 0, ldb = 0;
    float* bias_dev = nullptr;
    ~ZoeW() override { if (bias_dev) cudaFree(bias_dev); }
};

// attn.qkv.weight [3 dim][dim] + (q_bias | 0 | v_bias)
static Lin pack_beit_qkv(Packer& pk, const std::string& p, int dim) {
    Lin l;
    l.N = 3 * dim; l.K = dim;
    const float* w = pk.get(p + "attn.qkv.weight", (int64_t)3 * dim * dim);
    const float* qb = pk.get(p + "attn.q_bias", dim);
    const float* vb = pk.get(p + "attn.v_bias", dim);
    if (!w || !qb || !vb) return l;
    std::vector<float> bv((size_t)3 * dim, 0.f);
    memcpy(bv.data(), qb, (size_t)dim * 4);
    memcpy(bv.data() + 2 * (size_t)dim, vb, (size_t)dim * 4);
    l.w = pk.add_f16(std::vector<float>(w, w + (size_t)3 * dim * dim));
    l.b = pk.add_f32(bv);
    return l;
}

// metric bins head (zoedepth_v1.py): n_bins 64, bin_embedding_dim 128, attractors 16 / 8 / 4 / 1; F = bottleneck width
static void pack_zoe_bins(Packer& pk, ZoeBinsW& w, int F, bool normed, float min_depth, float max_depth) {
    w.feat = F;
    w.normed = normed;
    w.min_depth = min_depth;
    w.max_depth = max_depth;
    {   // AttractorLayer (normed) predicts 2 values per attractor and keeps the first, AttractorLayerUnnormed one
        const int64_t n = key_numel(pk, "attractors.0._net.2.bias");
        if (!pk.err.empty()) return;
        if (n != (normed ? 32 : 16)) {
            pk.err = "attractors.0._net.2 has " + std::to_string(n) + " outputs: a \"" + (normed ? "normed" : "softplus") +
                     "\" bins head (" + (normed ? "ZoeD_Any_K" : "ZoeD_N, ZoeD_Any_N") + ") has " + (normed ? "2 x 16" : "16") +
                     " (is this the checkpoint of the other ZoeD_Any model?)";
            return;
        }
    }
    w.ald = normed ? 32 : 16;
    w.conv2 = pack_conv(pk, "conv2", F, F, 1, 1);
    w.seed1 = pack_conv(pk, "seed_bin_regressor._net.0", 256, F, 1, 1);
    w.seed2 = pack_conv(pk, "seed_bin_regressor._net.2", 64, 256, 1, 1);
    w.sproj1 = pack_conv(pk, "seed_projector._net.0", 128, F, 1, 1);
    w.sproj2 = pack_conv(pk, "seed_projector._net.2", 128, 128, 1, 1);
    for (int i = 0; i < 4; ++i) {
        const std::string s = std::to_string(i);
        w.proj1[i] = pack_conv(pk, "projectors." + s + "._net.0", 128, F, 1, 1);
        w.proj2[i] = pack_conv(pk, "projectors." + s + "._net.2", 128, 128, 1, 1);
        w.att1[i] = pack_conv(pk, "attractors." + s + "._net.0", 128, 128, 1, 1);
        w.att2[i] = pack_conv(pk, "attractors." + s + "._net.2", (normed ? 2 : 1) * w.n_att[i], 128, 1, 1, 0, /*cout_pad=*/w.ald);
    }
    // ConditionalLogBinomial mlp: (32 + 1 + 128 = 161 -> K padded to 192) -> 80 (N padded to 96) -> GELU -> 4
    // input channels are re-ordered [embedding 128 | activation 32 | relative depth | 31 zeros] so that zoe_clb_concat moves
    // whole 16-byte groups (the reference concatenates [activation | relative depth | embedding])
    {
        Lin l;
        l.N = 96; l.K = 192;
        const float* cw = pk.get("conditional_log_binomial.mlp.0.weight", (int64_t)80 * 161);
        const float* cb = pk.get("conditional_log_binomial.mlp.0.bias", 80);
        if (cw && cb) {
            std::vector<float> wv((size_t)96 * 192, 0.f), bv(96, 0.f);
            for (int n = 0; n < 80; ++n) {
                for (int j = 0; j < 128; ++j) wv[(size_t)n * 192 + j] = cw[(size_t)n * 161 + 33 + j];
                for (int j = 0; j < 33; ++j) wv[(size_t)n * 192 + 128 + j] = cw[(size_t)n * 161 + j];
                bv[n] = cb[n];
            }
            l.w = pk.add_f16(wv);
            l.b = pk.add_f32(bv);
        }
        w.clb1 = l;
    }
    if (const float* c2 = pk.get("conditional_log_binomial.mlp.2.weight", 4 * 80)) {
        std::vector<float> v(c2, c2 + 320);
        for (auto& x : v) x = round_f16(x);   // the reference runs this conv in fp16
        w.clb2w = pk.add_f32(v);
    }
    w.clb2b = pack_vec_f32(pk, "conditional_log_binomial.mlp.2.bias", 4);
}

std::unique_ptr<NetW> pack_zoedepth(Packer& pk) {
    auto z = std::make_unique<ZoeW>();
    ZoeW& w = *z;
    const std::string bb = "core.core.pretrained.model.", pp = "core.core.pretrained.", sc = "core.core.scratch.";
    VitW& v = w.vit;
    v.dim = (int)key_numel(pk, bb + "cls_token");
    if (!pk.err.empty()) return z;
    const int dim = v.dim;
    if (dim < 64 || dim % 64) { pk.err = "ZoeDepth: embedding dim must be a multiple of 64 (head dim 64)"; return z; }
    v.heads = dim / 64;
    v.depth = 0;
    while (pk.src.count(bb + "blocks." + std::to_string(v.depth) + ".norm1.weight")) ++v.depth;
    if (v.depth < 4 || v.depth % 4) { pk.err = "ZoeDepth: the encoder depth must be a positive multiple of 4"; return z; }
    for (int i = 0; i < 4; ++i) {
        v.hooks[i] = v.depth / 4 * (i + 1) - 1;     // BEiT-L: blocks 5, 11, 17, 23 (MiDaS dpt_depth.py hooks)
        w.dpt.oc[i] = (int)key_numel(pk, pp + "act_postprocess" + std::to_string(i + 1) + ".3.bias");
        if (pk.err.empty() && (w.dpt.oc[i] < 32 || w.dpt.oc[i] % 32)) pk.err = "ZoeDepth: reassemble widths must be multiples of 32";
    }
    if (!pk.err.empty()) return z;
    w.dpt.feat = (int)(key_numel(pk, sc + "layer1_rn.weight") / ((int64_t)w.dpt.oc[0] * 9));
    const int F = w.dpt.feat;
    if (F < 64 || F % 64) { pk.err = "ZoeDepth: fusion width must be a multiple of 64"; return z; }
    {
        const int64_t rows = key_numel(pk, bb + "blocks.0.attn.relative_position_bias_table") / v.heads;
        const int s = (int)std::lround(std::sqrt((double)(rows - 3)));
        if (rows < 4 || (int64_t)s * s + 3 != rows || s % 2 == 0) { pk.err = "ZoeDepth: relative_position_bias_table must be [(2g-1)^2 + 3, heads]"; return z; }
        w.old_grid = (s + 1) / 2;
    }
    {   // patch embedding: Conv2d(3, dim, 16, 16) as a Linear over im2col rows (K = 768)
        Lin l;
        l.N = dim; l.K = 768;
        const float* pw = pk.get(bb + "patch_embed.proj.weight", (int64_t)dim * 768);
        const float* pb = pk.get(bb + "patch_embed.proj.bias", dim);
        if (pw && pb) {
            l.w = pk.add_f16(std::vector<float>(pw, pw + (size_t)dim * 768));
            l.b = pk.add_f32(std::vector<float>(pb, pb + dim));
        }
        w.patch = l;
    }
    w.cls = pack_vec_f32(pk, bb + "cls_token", dim);
    const int64_t trows = (int64_t)(2 * w.old_grid - 1) * (2 * w.old_grid - 1) + 3;
    for (int i = 0; i < v.depth; ++i) {
        const std::string p = bb + "blocks." + std::to_string(i) + ".";
        v.blocks.push_back(pack_vit_block(pk, p, dim, pack_beit_qkv(pk, p, dim), "gamma_1", "gamma_2"));
        const float* t = pk.get(p + "attn.relative_position_bias_table", trows * v.heads);
        w.tables.emplace_back(t ? std::vector<float>(t, t + trows * v.heads) : std::vector<float>());
        pk.mark(p + "attn.relative_position_index");   // a buffer of the timm module; recomputed for the actual grid
    }
    // the hooks are the raw residual stream: the final norm is unused by DPT
    for (const char* k : {"norm.weight", "norm.bias", "fc_norm.weight", "fc_norm.bias", "head.weight", "head.bias"}) pk.mark(bb + k);
    DptKeys k;
    for (int i = 0; i < 4; ++i) {
        const std::string p = pp + "act_postprocess" + std::to_string(i + 1) + ".";
        k.readout[i] = p + "0.project.0";
        k.project[i] = p + "3";
        k.resize[i] = p + "4";
    }
    k.scratch = sc;
    k.out_conv[0] = sc + "output_conv.0";
    k.out_conv[1] = sc + "output_conv.2";
    k.out_conv[2] = sc + "output_conv.4";
    pack_dpt(pk, w.dpt, dim, k);
    pack_zoe_bins(pk, w.head, F, false, 1e-3f, 10.f);
    return z;
}

// MiDaS beit.py _get_rel_pos_bias: the (2g-1) x (2g-1) learned sub-table -> (2ph-1) x (2pw-1) by ATen's bilinear resample
// (align_corners=False, no antialias), the 3 class-token rows appended unchanged.  out: [(2ph-1)(2pw-1) + 3][heads]
static void zoe_resample_table(const float* tab, int g, int heads, int ph, int pw, float* out) {
    const int S = 2 * g - 1, nh = 2 * ph - 1, nw = 2 * pw - 1;
    const float sy = (float)S / (float)nh, sx = (float)S / (float)nw;
    for (int y = 0; y < nh; ++y) {
        float fy = sy * ((float)y + 0.5f) - 0.5f;
        if (fy < 0.f) fy = 0.f;
        const int y0 = (int)fy, y1 = y0 + (y0 < S - 1 ? 1 : 0);
        const float ly = fy - (float)y0, hy = 1.f - ly;
        for (int x = 0; x < nw; ++x) {
            float fx = sx * ((float)x + 0.5f) - 0.5f;
            if (fx < 0.f) fx = 0.f;
            const int x0 = (int)fx, x1 = x0 + (x0 < S - 1 ? 1 : 0);
            const float lx = fx - (float)x0, hx = 1.f - lx;
            const float* a = &tab[((size_t)y0 * S + x0) * heads];
            const float* b = &tab[((size_t)y0 * S + x1) * heads];
            const float* c = &tab[((size_t)y1 * S + x0) * heads];
            const float* d = &tab[((size_t)y1 * S + x1) * heads];
            float* o = out + ((size_t)y * nw + x) * heads;
            for (int h = 0; h < heads; ++h) o[h] = hy * (hx * a[h] + lx * b[h]) + ly * (hx * c[h] + lx * d[h]);
        }
    }
    memcpy(out + (size_t)nh * nw * heads, &tab[(size_t)S * S * heads], (size_t)3 * heads * 4);
}

static int zoe_prepare_bias(ZoeW& w, cudaStream_t st, int ph, int pw) {
    if (w.bias_dev && w.bias_ph == ph && w.bias_pw == pw) return 0;
    const int heads = w.vit.heads, depth = w.vit.depth;
    const int N = ph * pw + 1, ldb = (N + 63) / 64 * 64;
    const size_t rows = (size_t)(2 * ph - 1) * (2 * pw - 1) + 3, per_layer = (size_t)heads * N * ldb;
    std::vector<float> host(rows * heads * depth);
    for (int i = 0; i < depth; ++i) zoe_resample_table(w.tables[i].data(), w.old_grid, heads, ph, pw, host.data() + (size_t)i * rows * heads);
    if (w.bias_dev) cudaFree(w.bias_dev);
    w.bias_dev = nullptr; w.bias_ph = w.bias_pw = 0;
    float* tdev = nullptr;
    NB_CUDA(cudaMalloc((void**)&w.bias_dev, per_layer * depth * 4));
    NB_CUDA(cudaMalloc((void**)&tdev, host.size() * 4));
    cudaError_t e = cudaMemsetAsync(w.bias_dev, 0, per_layer * depth * 4, st);
    if (e == cudaSuccess) e = cudaMemcpyAsync(tdev, host.data(), host.size() * 4, cudaMemcpyHostToDevice, st);
    int rc = 0;
    for (int i = 0; i < depth && e == cudaSuccess && !rc; ++i)
        rc = zoe_expand_rel_bias(st, tdev + (size_t)i * rows * heads, ph, pw, heads, w.bias_dev + (size_t)i * per_layer, ldb);
    if (e == cudaSuccess) e = cudaStreamSynchronize(st);   // `host` / `tdev` are temporaries (once per token-grid shape)
    cudaFree(tdev);
    if (e != cudaSuccess) return fail(std::string("zoe_prepare_bias: ") + cudaGetErrorString(e));
    if (rc) return 1;
    w.bias_ph = ph; w.bias_pw = pw; w.ldb = ldb;
    return 0;
}

// ZoeD_Any_N / ZoeD_Any_K (Depth-Anything metric_depth ZoeDepth over DepthAnythingCore): the Depth-Anything V1 encoder and DPT
// head under `core.core.` (hooks: the last four blocks through the final norm), the bins head of ZoeD_N ("softplus", indoor) or
// the "normed" one (outdoor, max_depth 80).  The widths are read off the tensor sizes.
std::unique_ptr<NetW> pack_zoedepth_any(Packer& pk, bool normed) {
    auto z = std::make_unique<ZoeW>();
    z->da = pack_dinov2_dpt(pk, -1, "core.core.", true);
    if (pk.err.empty()) pack_zoe_bins(pk, z->head, z->da->dpt.feat, normed, 1e-3f, normed ? 80.f : 10.f);
    return z;
}

// workspace of the bins head
struct ZoeBinsBufs {
    __half *XB, *S1, *S2, *Ea, *E[2], *Yb, *A1, *A2, *CC, *G;
    float *BIN[2], *SORTED;
};
static void zoe_bins_plan(Arena& a, const ZoeBinsW& w, const DptGeom& g, ZoeBinsBufs& z) {
    const size_t B = g.B, lv3 = B * g.lh[3] * g.lw[3], lvp = B * g.hp * g.wp, npix = B * g.H * g.W;
    z.XB = a.take<__half>(lv3 * w.feat);
    z.S1 = a.take<__half>(lv3 * 256);
    z.S2 = a.take<__half>(lv3 * 64);
    z.Ea = a.take<__half>(lvp * 128);
    for (auto& e : z.E) e = a.take<__half>(lvp * 128);
    z.Yb = a.take<__half>(lvp * 128);
    z.A1 = a.take<__half>(lvp * 128);
    z.A2 = a.take<__half>(lvp * w.ald);
    for (auto& e : z.BIN) e = a.take<float>(lvp * 64);
    z.SORTED = w.normed ? a.take<float>(lvp * 64) : nullptr;
    z.CC = a.take<__half>(npix * 192);
    z.G = a.take<__half>(npix * 96);
}

// zoedepth_v1.py ZoeDepth.forward after the core: b.R[3] (bottleneck), b.PATH (r4..r1), b.O2 (out_conv activation) and rel ->
// metric depth.  Taps 11..14: the bin centres of each attractor level (fp32 [pix][64]; [0, 1] units for a normed head), tap 15
// (normed only): the sorted, scaled and clipped centres of the last level.
static int zoe_bins_forward(nb200_model* m, cudaStream_t st, const ZoeBinsW& w, const DptBufs& b, const DptGeom& g, const float* rel,
                            const ZoeBinsBufs& z, float* depth) {
    const int B = g.B, H = g.H, W = g.W, F = w.feat, hp = g.hp, wp = g.wp, h4 = g.lh[3], w4 = g.lw[3];
    const size_t npix = (size_t)B * H * W;
    auto c1x1 = [&](const Lin& l, const __half* A, int h, int ww, int cin, __half* out, int act) {
        return da_conv(st, m, l, A, B, h, ww, cin, cin, out, act, nullptr, false);
    };
    if (c1x1(w.conv2, b.R[3], h4, w4, F, z.XB, ACT_NONE)) return 1;
    if (c1x1(w.seed1, z.XB, h4, w4, F, z.S1, ACT_RELU)) return 1;
    if (w.normed) {                                                                         // SeedBinRegressor: ReLU, normalise, cumsum
        if (c1x1(w.seed2, z.S1, h4, w4, 256, z.S2, ACT_RELU)) return 1;
        if (zoe_seed_normed(st, z.S2, (long long)B * h4 * w4, w.min_depth, w.max_depth, z.BIN[0])) return 1;
    } else {                                                                                // SeedBinRegressorUnnormed: softplus
        if (c1x1(w.seed2, z.S1, h4, w4, 256, z.S2, ACT_NONE)) return 1;
        if (zoe_softplus(st, z.S2, z.BIN[0], (long long)B * h4 * w4 * 64)) return 1;
    }
    if (c1x1(w.sproj1, z.XB, h4, w4, F, z.Ea, ACT_RELU)) return 1;
    if (c1x1(w.sproj2, z.Ea, h4, w4, 128, z.E[0], ACT_NONE)) return 1;
    const int lh[4] = {g.lh[2], g.lh[1], g.lh[0], hp}, lw[4] = {g.lw[2], g.lw[1], g.lw[0], wp};
    int prev_h = h4, prev_w = w4, cur = 0;
    for (int i = 0; i < 4; ++i) {
        const int nh = lh[i], nw = lw[i], nxt = cur ^ 1;
        if (c1x1(w.proj1[i], b.PATH[i], nh, nw, F, z.Ea, ACT_RELU)) return 1;
        if (c1x1(w.proj2[i], z.Ea, nh, nw, 128, z.E[nxt], ACT_NONE)) return 1;
        if (zoe_add_upsampled(st, z.E[nxt], z.E[cur], B, prev_h, prev_w, 128, nh, nw, z.Yb)) return 1;
        if (c1x1(w.att1[i], z.Yb, nh, nw, 128, z.A1, ACT_RELU)) return 1;
        if (w.normed) {
            // the reference sorts the scaled centres at every level but passes only the last level's on
            if (c1x1(w.att2[i], z.A1, nh, nw, 128, z.A2, ACT_RELU)) return 1;
            if (zoe_attractor_normed(st, z.A2, w.ald, w.n_att[i], z.BIN[cur], B, prev_h, prev_w, nh, nw, w.min_depth, w.max_depth,
                                     z.BIN[nxt], i == 3 ? z.SORTED : nullptr)) return 1;
        } else {
            if (c1x1(w.att2[i], z.A1, nh, nw, 128, z.A2, ACT_NONE)) return 1;
            if (zoe_attractor(st, z.A2, w.ald, w.n_att[i], z.BIN[cur], B, prev_h, prev_w, nh, nw, z.BIN[nxt])) return 1;
        }
        prev_h = nh; prev_w = nw; cur = nxt;
        if (tap_copy(st, 11 + i, z.BIN[cur], (size_t)B * nh * nw * 64 * 4)) return 1;       // taps 11..14: bin centres fp32 [pix][64]
    }
    const float* centres = w.normed ? z.SORTED : z.BIN[cur];
    if (w.normed && tap_copy(st, 15, centres, (size_t)B * hp * wp * 64 * 4)) return 1;      // tap 15: sorted centres (normed)
    if (zoe_clb_concat(st, b.O2, rel, z.E[cur], B, hp, wp, H, W, z.CC)) return 1;
    if (da_linear(st, m, w.clb1, z.CC, (long long)npix, 192, z.G, ACT_GELU)) return 1;
    return zoe_clb_final(st, z.G, 96, m->at<float>(w.clb2w), m->at<float>(w.clb2b), centres, B, hp, wp, H, W, depth);
}

// ZoeDepth.forward(x)['metric_depth'] of ZoeD_N (BEiT-L/16 encoder, MiDaS DPT head) or ZoeD_Any (Depth-Anything V1 encoder and
// DPT head); taps 0..10 are the points of the core the bins head reads.
static int zoedepth_forward(nb200_model* m, ZoeW& w, cudaStream_t st, const float* x, int B, int H, int W, float* depth) {
    DaW* any = w.da.get();
    if (any) NB_CHECK(H % 14 == 0 && W % 14 == 0 && H >= 14 && W >= 14, "input height and width must be multiples of 14 (batch_preprocess, prep_mod 14)");
    else NB_CHECK(H % 32 == 0 && W % 32 == 0 && H >= 32 && W >= 32, "input height and width must be multiples of 32 (batch_preprocess)");
    const DptGeom g = dpt_geom(B, H, W, any ? 14 : 16);
    const VitW& vit = any ? any->vit : w.vit;
    const DptW& dpt = any ? any->dpt : w.dpt;
    const int dim = vit.dim, P = g.P, N = g.N, F = dpt.feat;
    const int h1 = g.lh[0], w1 = g.lw[0], h2 = g.lh[1], w2 = g.lw[1], h3 = g.lh[2], w3 = g.lw[2], h4 = g.lh[3], w4 = g.lw[3];
    const int hp = g.hp, wp = g.wp;   // path_1 resolution = 8 x the token grid
    const long long M = (long long)B * N;
    if (any ? da_prepare_pos(*any, st, g.ph, g.pw) : zoe_prepare_bias(w, st, g.ph, g.pw)) return 1;
    const size_t npix = (size_t)B * H * W;
    __half* Apatch;
    float* REL;
    DptBufs b;
    ZoeBinsBufs z;
    if (m->carve([&](Arena& a) {
            Apatch = a.take<__half>((size_t)B * P * (any ? any->kpad : 768));
            dpt_plan(a, vit, dpt, g, b);
            REL = a.take<float>(npix);
            zoe_bins_plan(a, w.head, g, z);
        })) return 1;

    if (any) {
        // ---- encoder (dinov2 get_intermediate_layers(x, 4, return_class_token=True): the last four blocks, final norm)
        if (da_encode(st, m, *any, x, g, b, Apatch)) return 1;
    } else {
        // ---- encoder (timm beit.py Beit.forward_features with the MiDaS relative-position resample; hooks, no final norm)
        if (zoe_patch_im2col(st, x, B, H, W, Apatch)) return 1;
        if (da_linear(st, m, w.patch, Apatch, (long long)B * P, 768, b.T, ACT_NONE)) return 1;
        if (zoe_assemble_tokens(st, b.T, m->at<float>(w.cls), b.X32, B, P, dim)) return 1;
        if (vit_encoder(st, m, w.vit, b, g, w.bias_dev, (size_t)w.vit.heads * N * w.ldb, w.ldb)) return 1;
    }
    for (int i = 0; i < 4; ++i)                                                             // taps 0..3: hooked hidden states
        if (tap_copy(st, i, b.FE[i], (size_t)M * dim * 2)) return 1;
    // ---- DPT reassemble (readout "project" for ZoeD_N, "ignore" for ZoeD_Any), 1x1 conv, resize, fusion
    if (dpt_fuse(st, m, dpt, dim, b, g)) return 1;
    for (int i = 0; i < 4; ++i)                                                             // taps 4..7: path_4 .. path_1 (NHWC)
        if (tap_copy(st, 4 + i, b.PATH[i], (size_t)B * (i == 0 ? h3 * w3 : i == 1 ? h2 * w2 : i == 2 ? h1 * w1 : hp * wp) * F * 2)) return 1;
    if (tap_copy(st, 8, b.R[3], (size_t)B * h4 * w4 * F * 2)) return 1;                    // tap 8: bottleneck (layer4_rn)
    // ---- output_conv: relative depth + the 32-channel activation the bins head is conditioned on
    if (dpt_output(st, m, dpt, b, g, REL)) return 1;
    if (tap_copy(st, 9, b.O2, npix * 32 * 2)) return 1;                                     // tap 9: out_conv activation (NHWC, 32)
    if (tap_copy(st, 10, REL, npix * 4)) return 1;                                          // tap 10: relative depth fp32
    return zoe_bins_forward(m, st, w.head, b, g, REL, z, depth);
}

}  // namespace nb200

using namespace nb200;

// Host-only: the relative-position table resample of the BEiT blocks (MiDaS beit.py _get_rel_pos_bias) for a ph x pw token grid.
// table [(2g-1)^2 + 3][heads] -> out [(2ph-1)(2pw-1) + 3][heads].  No GPU needed (tests/test_host_logic.py).
extern "C" int nb200_zoe_rel_pos_table(const float* table, int g, int heads, int ph, int pw, float* out) {
    NB_CHECK(table && out, "null pointer");
    NB_CHECK(g > 0 && heads > 0 && ph > 0 && pw > 0, "bad shape");
    zoe_resample_table(table, g, heads, ph, pw, out);
    return 0;
}

// ZoeDepth.forward(x)['metric_depth'] (what zoedepth_model._forward calls, iw3/zoedepth_model.py:23-27)
extern "C" int nb200_zoedepth_forward(nb200_model* m, const float* x, int B, int H, int W, float* depth, void* stream) {
    NB_CHECK(m && x && depth, "null pointer");
    ZoeW* w = net_as<ZoeW>(m);
    NB_CHECK(w, "model is not a ZoeDepth network");
    NB_CHECK(B > 0, "empty batch");
    return zoedepth_forward(m, *w, (cudaStream_t)stream, x, B, H, W, depth);
}
