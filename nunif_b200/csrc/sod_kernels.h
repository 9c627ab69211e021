// iw3.sod_v1 (iw3/models/sod_v1.py): U^2-Net-p (nunif/utils/u2netp.py) on 192 x 192 NHWC fp16, and the convergence
// estimate of iw3/convergence_estimator.py.  Packed by sod_model.cu, run by sod.cu.
#pragma once
#include "common.cuh"
#include <string>
#include <vector>

namespace nb200 {

constexpr int SOD_SIZE = 192;   // SODV1's i2i_in_size: both inputs are resized to it, every level size is then even

// One REBNCONV (3x3 conv, padding = dilation, BatchNorm folded in, ReLU): weights fp16 [cout][9][cin_pad] (K = (tap, c)),
// bias fp32 holding the fp16-rounded folded bias.  cin_pad is cin rounded up to 16 (the first conv's 6 channels).
struct SodConv {
    size_t w = 0, b = 0;
    int cin = 0, cin_pad = 0, cout = 0, dil = 1;
    std::string name;
};

struct SodW {
    std::vector<SodConv> convs;   // in forward order (sod_layer_list)
    size_t side = 0;              // fp32 [6][9][64] fp16-rounded side1..6 weights (tap-major), then 6 biases
    size_t head = 0;              // fp32 [7]: outconv weight [6] and bias, fp16-rounded
};

// The REBNCONVs of U2NETP(in_ch=6) in the order the forward runs them: stage1..6, stage5d..1d; inside a block rebnconvin,
// rebnconv1..n, rebnconv(n-1)d..1d.  RSU7/6/5/4 (n = 7..4) dilate only the innermost conv (2); RSU4F (n = 0 here) uses
// 1, 2, 4, 8, then 4, 2, 1.
struct SodStage { const char* name; int n; int in_ch; };
static const SodStage SOD_STAGES[11] = {
    {"stage1", 7, 6},   {"stage2", 6, 64},   {"stage3", 5, 64},   {"stage4", 4, 64},  {"stage5", 0, 64}, {"stage6", 0, 64},
    {"stage5d", 0, 128}, {"stage4d", 4, 128}, {"stage3d", 5, 128}, {"stage2d", 6, 128}, {"stage1d", 7, 128}};

inline void sod_layer_list(std::vector<SodConv>& out) {
    out.clear();
    auto add = [&](const std::string& name, int cin, int cout, int dil) {
        SodConv c;
        c.name = name; c.cin = cin; c.cin_pad = (cin + 15) / 16 * 16; c.cout = cout; c.dil = dil;
        out.push_back(c);
    };
    for (const SodStage& s : SOD_STAGES) {
        const std::string p = std::string("u2netp.") + s.name + ".rebnconv";
        add(p + "in", s.in_ch, 64, 1);
        add(p + "1", 64, 16, 1);
        if (s.n == 0) {
            add(p + "2", 16, 16, 2);
            add(p + "3", 16, 16, 4);
            add(p + "4", 16, 16, 8);
            add(p + "3d", 32, 16, 4);
            add(p + "2d", 32, 16, 2);
        } else {
            for (int k = 2; k < s.n; ++k) add(p + std::to_string(k), 16, 16, 1);
            add(p + std::to_string(s.n), 16, 16, 2);
            for (int k = s.n - 1; k >= 2; --k) add(p + std::to_string(k) + "d", 32, 16, 1);
        }
        add(p + "1d", 32, 64, 1);
    }
}

// SODV1.infer up to the sigmoid: rgb [B][3][H][W], depth [B][1][h][w] fp32 -> saliency [B][1][192][192] (fp32 holding the
// fp16 sigmoid) and depth192 [B][1][192][192] fp32 (the bilinear resize of depth).
int sod_forward(cudaStream_t st, const uint8_t* blob, const SodW& w, const float* rgb, int B, int H, int W, const float* depth,
                int h, int wd, float* saliency, float* depth192);

}  // namespace nb200
