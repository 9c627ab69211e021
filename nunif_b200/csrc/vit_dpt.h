// The ViT encoder and DPT head that Depth-Anything (depth_model.cu) and ZoeD_N / ZoeD_Any (zoe_model.cu) share: their weights,
// packers, workspace and forward stages, defined in depth_model.cu.
#pragma once
#include "model.h"

namespace nb200 {

struct VitBlockW {
    Lin qkv, proj, fc1, fc2;
    size_t n1w = 0, n1b = 0, n2w = 0, n2b = 0;
};
struct VitW {
    int dim = 0, depth = 0, heads = 0, hooks[4] = {};
    std::vector<VitBlockW> blocks;
    bool hook_norm = false;         // the hooked hidden states go through the final LayerNorm normw / normb
    size_t normw = 0, normb = 0;
};
struct DaRefineW {
    Lin out_conv, c[2][2];   // resConfUnit{1,2}.conv{1,2}
};
struct DptW {
    int oc[4] = {}, feat = 0;
    int c0pad = 0;      // channel stride of the first reassembled map (oc[0] rounded up to a multiple of 32)
    Lin readout[4];     // ProjectReadout Linear(2 dim, dim) + GELU; N == 0: the class token is ignored
    Lin reasm[4], resize3, rn[4], oc1, oc2;
    DaRefineW ref[4];   // refinenet1..4
    size_t oc3w = 0;
    float oc3b = 0.f;
};
// state_dict key names of one DPT neck; readout[i] empty: no readout projection
struct DptKeys {
    std::string readout[4], project[4], resize[4];   // resize[2] unused (identity)
    std::string scratch;                              // prefix of layerN_rn and refinenetN
    std::string out_conv[3];                          // 3x3 feat -> feat/2, 3x3 feat/2 -> 32, 1x1 32 -> 1
};

// Depth-Anything V2 / V1: the DINOv2 encoder and the DPT head (also ZoeD_Any's core)
struct NB_HIDDEN DaW : NetW {
    int kpad = 640, pos_grid = 37;
    VitW vit;
    DptW dpt;
    Lin patch;
    size_t cls = 0;
    std::vector<float> pos_host;   // learned table [1 + grid*grid][dim]
    // interpolated position table of the last token grid
    int pos_ph = 0, pos_pw = 0;
    float* pos_dev = nullptr;
    ~DaW() override { if (pos_dev) cudaFree(pos_dev); }
};

// one pre-norm ViT block (prefix p) around an already packed qkv; the LayerScale gammas p + gamma1 / gamma2 are folded into
// attn.proj / mlp.fc2
NB_HIDDEN VitBlockW pack_vit_block(Packer& pk, const std::string& p, int dim, const Lin& qkv, const char* gamma1, const char* gamma2);
// the DPT neck (dpt.py DPTHead / MiDaS dpt_depth.py): d.oc and d.feat are set by the caller
NB_HIDDEN void pack_dpt(Packer& pk, DptW& d, int dim, const DptKeys& k);
// the element count of a state_dict tensor (0 and a packer error when it is missing)
NB_HIDDEN int64_t key_numel(Packer& pk, const std::string& name);
// encoder: 0 = ViT-S, 1 = ViT-B, 2 = ViT-L (Depth-Anything dpt.py model_configs), -1 = read the widths off the tensor sizes
// (ZoeD_Any, whose reduced test configuration runs the same code).  pre: key prefix of `pretrained.*` / `depth_head.*`
// ("core.core." inside ZoeD_Any).  last4: the hooks are the last four blocks (Depth-Anything V1 get_intermediate_layers(x, 4)),
// else the V2 intermediate_layer_idx table.
NB_HIDDEN std::unique_ptr<DaW> pack_dinov2_dpt(Packer& pk, int encoder, const std::string& pre, bool last4);

// B images of H x W as a ph x pw token grid (P patches + the class token) and the DPT levels: lv[0..3] = 4x, 2x, 1x and
// (ceil) 1/2x the token grid; path_1 / output_conv1 at hp x wp = 8x
struct DptGeom {
    int B, H, W, ph, pw, P, N, hp, wp;
    int lh[4], lw[4];
};
NB_HIDDEN DptGeom dpt_geom(int B, int H, int W, int patch);

// the workspace buffers of the encoder and the DPT neck
struct DptBufs {
    __half* T;                 // patch GEMM output, readout concat, reassemble-0 GEMM output
    float* X32;                // residual stream
    __half *Hn, *QKV, *ATT, *HID, *D, *FE[4];
    __half* Y;                 // readout GEMM output (only with a readout)
    __half *L[4], *L4lin, *L4col, *R[4];
    __half *t_relu, *t_c1, *t_sum, *t_u, *t_up;
    __half* PATH[4];           // path_4 .. path_1
    __half *O1, *O1u, *O2;
};
NB_HIDDEN void dpt_plan(Arena& a, const VitW& v, const DptW& d, const DptGeom& g, DptBufs& b);

NB_HIDDEN int da_linear(cudaStream_t st, const nb200_model* m, const Lin& l, const __half* A, long long M, int lda, __half* out, int act);
// NHWC conv3x3 pad 1 (or 1x1 when taps == 1) on [B][H][W][Cin] -> [B][H][W][N]
NB_HIDDEN int da_conv(cudaStream_t st, const nb200_model* m, const Lin& l, const __half* A, int B, int H, int W, int Ci, int Cin,
                      __half* out, int act, const __half* res, bool k3);
// The ViT blocks over the tokens in b.X32; the hidden state after block v.hooks[i] goes to b.FE[i].  bias: per-layer
// attention bias (layer i at bias + i * bias_layer, row stride ldb), or null.
NB_HIDDEN int vit_encoder(cudaStream_t st, const nb200_model* m, const VitW& v, const DptBufs& b, const DptGeom& g, const float* bias,
                          size_t bias_layer, int ldb);
// DPT reassemble (readout, 1x1 conv, resize), layerN_rn and the four fusion blocks: b.FE -> b.R, b.PATH
NB_HIDDEN int dpt_fuse(cudaStream_t st, const nb200_model* m, const DptW& d, int dim, const DptBufs& b, const DptGeom& g);
// scratch.output_conv: path_1 -> the 32-channel activation b.O2 and the relative depth rel fp32 [B][H][W]
NB_HIDDEN int dpt_output(cudaStream_t st, const nb200_model* m, const DptW& d, const DptBufs& b, const DptGeom& g, float* rel);
// the position table of a ph x pw token grid, rebuilt when the grid changes
NB_HIDDEN int da_prepare_pos(DaW& w, cudaStream_t st, int ph, int pw);
// dinov2 vision_transformer.py prepare_tokens_with_masks + blocks: x -> the hooked, normed hidden states b.FE
// (Apatch: B * P * kpad fp16)
NB_HIDDEN int da_encode(cudaStream_t st, const nb200_model* m, const DaW& w, const float* x, const DptGeom& g, const DptBufs& b,
                        __half* Apatch);

}  // namespace nb200
