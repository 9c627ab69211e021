// The window-attention block WABlock that sbs.row_flow_v3, sbs.mlbw and iw3.depth_aa are built from (wa_block.cu).
#pragma once
#include "model.h"
#include "gemm.h"

namespace nb200 {

struct WaBlockW {
    Lin qkv, proj, mlp0, mlp3;
    size_t bias = 0;              // fp32 [N][N], N = ws * ws
    int ws = 0, heads = 0;
    int pad_y = 0, pad_x = 0;     // ws / 2 in each direction the block is shifted in, else 0
    int act = ACT_NONE;           // after the 3x3: ACT_LRELU01 or ACT_NONE
};

// p: the block's prefix, e.g. "blocks.1."
NB_HIDDEN WaBlockW pack_wa_block(Packer& pk, const std::string& p, int C, int ws, int heads, int pad_y, int pad_x, int act);

// the workspace of the blocks over a [B][H][W][C] token grid: the residual stream X and the blocks' temporaries
struct WaBufs {
    __half *X, *QKV, *ATT, *T, *TP;
};
NB_HIDDEN void wa_plan(Arena& a, WaBufs& w, int B, int H, int W, int C);

// one block, in place on w.X
NB_HIDDEN int wa_block(cudaStream_t st, const nb200_model* m, const WaBlockW& b, const WaBufs& w, int B, int H, int W);

// The test entry points of the three networks' input and output stages (the kernels a forward launches between its blocks)
// check the geometry their forward computes: an image of B x H x W at (ph1, pw1) inside a padded Hp x Wp grid.
NB_HIDDEN int stereo_geometry(int B, int H, int W, int ph1, int pw1, int Hp, int Wp);

}  // namespace nb200
