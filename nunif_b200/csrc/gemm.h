// Host interface of the wgmma implicit-GEMM (see gemm_wgmma.cuh).
#pragma once
#include "common.cuh"

namespace nb200 {

// CG_TCONV3: a (3,1,1) convolution over time with dilation `dil` and zero padding `dil`; A is viewed as [B][T = Hi][Wi][Ci]
// (Wi = the pixels of one frame), taps t - dil, t, t + dil
enum : int { CG_LINEAR_FLAT = 0, CG_LINEAR_2D = 1, CG_CONV3 = 2, CG_DOWN2 = 3, CG_TCONV3 = 5 };
// ConvGemm::act (the epilogue's activation) and ConvGemm::out_mode
enum : int { ACT_NONE = 0, ACT_LRELU01 = 1, ACT_GELU = 2, ACT_RELU = 3 };
enum : int { OUT_NHWC = 0, OUT_PIXSHUF2 = 1, OUT_SPLIT = 2 };

struct ConvGemm {
    const __half* A = nullptr;  // NHWC fp16 activations [B][Hi][Wi][Ci]
    int B = 1, Hi = 1, Wi = 1;
    int Ci = 0;                 // channel stride of A (elements per pixel)
    int Cin = 0;                // channels consumed (<= Ci)
    long long a_row_stride = 0; // elements between image rows (0 = Wi*Ci); lets A be a cropped view
    long long a_img_stride = 0; // elements between images     (0 = Hi*a_row_stride)
    int kind = CG_LINEAR_FLAT;
    int pad = 0;                // CG_CONV3: zero padding (0 = valid conv, 1 = 'same'); the halo comes from the TMA's out-of-bounds zero fill
    int dil = 1;                // CG_TCONV3: temporal dilation (1..127); the time padding is the same out-of-bounds zero fill
    const __half* Wt = nullptr; // packed weights [N][taps*Cin_tap], K ordered (ky, kx, c)
    int N = 0;
    const float* bias = nullptr;
    int act = 0;
    __half* out = nullptr;      // NHWC fp16, channel stride ldo
    int ldo = 0;
    int out_mode = 0, cout = 0; // OUT_PIXSHUF2: N = 4*cout ordered (dy, dx, co); OUT_SPLIT: N = nsplit*cout
    long long split_stride = 0; // OUT_SPLIT: elements between the dense [M][cout] output planes
    int a_planes = 1;           // CG_LINEAR_FLAT: A is `a_planes` dense [M][Cin] planes (K = a_planes*Cin, plane-major)
    long long a_plane_stride = 0;
    const __half* res = nullptr;
    int ldr = 0, res_H = 0, res_W = 0, res_cy = 0, res_cx = 0, res_before_act = 0;
    // OUT_PIXSHUF2 only, instead of res: a second A operand [B][2 Ho][2 Wo][ld2] whose first Cin2 channels at each output
    // pixel are K columns [taps*Cin, taps*Cin + Cin2) of Wt (a Linear of the skip folded into the GEMM)
    const __half* A2 = nullptr;
    int Cin2 = 0, ld2 = 0;
};

int conv_gemm(cudaStream_t st, const ConvGemm& g);

}  // namespace nb200
