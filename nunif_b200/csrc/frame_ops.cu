// Frame-edge conversions of the iw3 path (SURVEY.md 8a rows B2, B15):
//   * uint8/uint16 HWC  <-> fp32 CHW in [0,1]   (nunif/utils/video.py:218-223,236-246, iw3/utils.py:274-289)
//   * DepthAnything batch_preprocess (iw3/depth_anything_model.py:69-110): short side -> lower_bound (multiple of 14),
//     antialiased bilinear resize (ATen _upsample_bilinear2d_aa, align_corners=False), clamp, ImageNet normalise -
//     one fused kernel over the output (the reference makes 1 resize + 3 elementwise passes).
// All HBM-bound: the conversions move 3+12 B/px, the preprocess reads the 24.9 MB fp32 frame once.
#include "common.cuh"
#include "aa_resize.cuh"
#include <cmath>
#include "../../include/nunif_b200.h"

namespace nb200 {

template <typename T>
__global__ void __launch_bounds__(256) hwc_to_chw_kernel(const T* __restrict__ x, float* __restrict__ out, size_t plane, size_t total,
                                                          float maxv) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;   // pixel index over B*H*W
    if (i >= total) return;
    const size_t b = i / plane, p = i - b * plane;
    const T* s = x + i * 3;
    float* o = out + b * 3 * plane + p;
    // true division like x / iinfo.max (video.py:223, iw3/utils.py:287)
    o[0] = __fdiv_rn((float)s[0], maxv);
    o[plane] = __fdiv_rn((float)s[1], maxv);
    o[2 * plane] = __fdiv_rn((float)s[2], maxv);
}

template <typename T>
__global__ void __launch_bounds__(256) chw_to_hwc_kernel(const float* __restrict__ x, T* __restrict__ out, size_t plane, size_t total,
                                                          float scale, float maxv) {
    const size_t i = (size_t)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const size_t b = i / plane, p = i - b * plane;
    const float* s = x + b * 3 * plane + p;
    T* o = out + i * 3;
#pragma unroll
    for (int c = 0; c < 3; ++c) {
        // (x * scale).round_().to(dtype) (video.py:244): round half to even; out-of-range values saturate here
        // (the reference's cast is undefined for them - frames are clamped to [0,1] before this point)
        float v = rintf(__fmul_rn(s[c * plane], scale));
        v = fminf(fmaxf(v, 0.f), maxv);
        o[c] = (T)v;
    }
}

struct DaPrepParams {
    const float* x;
    float* out;
    int B, H, W, oh, ow;  // oh x ow = resized frame; the output is (oh + 2*pad_h) x (ow + 2*pad_w), reflection padded
    int pad_h, pad_w;
    float sy, sx;         // in/out scale (align_corners=False)
    float mean[3], stdv[3];
    int plain;            // 1: the resize alone (no clamp, no normalisation)
};

// ATen UpSampleKernel (_upsample_bilinear2d_aa, csrc/aa_resize.cuh), align_corners=False.
__global__ void __launch_bounds__(128) da_preprocess_kernel(DaPrepParams p) {
    const int px = blockIdx.x * blockDim.x + threadIdx.x, py = blockIdx.y, b = blockIdx.z;
    const int OW = p.ow + 2 * p.pad_w, OH = p.oh + 2 * p.pad_h;
    if (px >= OW) return;
    // reflection padding (ZoeDepth, reflection_pad2d.py:57-68) copies resized pixels: evaluate the resize at the mirrored index
    // (reflection_pad2d_loop pads in steps of at most size-1, which is the periodic mirror extension for any pad)
    int ox = px - p.pad_w, oy = py - p.pad_h;
    if (p.pad_w > 0) { const int m = 2 * (p.ow - 1); ox = ((ox % m) + m) % m; ox = ox < p.ow ? ox : m - ox; }
    if (p.pad_h > 0) { const int m = 2 * (p.oh - 1); oy = ((oy % m) + m) % m; oy = oy < p.oh ? oy : m - oy; }
    const AaTaps ty = aa_taps(p.sy, oy, p.H), tx = aa_taps(p.sx, ox, p.W);
    const float sum_y = aa_weight_sum(ty), sum_x = aa_weight_sum(tx);
    const size_t plane = (size_t)p.H * p.W;
    for (int c = 0; c < 3; ++c) {
        const float* src = p.x + ((size_t)b * 3 + c) * plane;
        float acc = aa_sample(ty, tx, sum_y, sum_x, [&](int y, int x) { return __ldg(src + (size_t)y * p.W + x); });
        if (!p.plain) {
            acc = clamp01(acc);                                                // depth_anything_model.py:104 / zoedepth_model.py:75
            acc = __fdiv_rn(__fsub_rn(acc, p.mean[c]), p.stdv[c]);             // :107-109 / :78-80
        }
        p.out[(((size_t)b * 3 + c) * OH + py) * OW + px] = acc;
    }
}

// torch.rot90(x, k, (-2, -1)) of one H x W plane per blockIdx.z -> W x H.  k = 1: out[i][j] = x[j][W-1-i];
// k = 3: out[i][j] = x[H-1-j][i].  A 32 x 32 tile goes through shared memory so that reads and writes are both coalesced.
__global__ void __launch_bounds__(256) rot90_kernel(const float* __restrict__ x, float* __restrict__ out, int H, int W, int k) {
    __shared__ float tile[32][33];
    const int x0 = blockIdx.x * 32, y0 = blockIdx.y * 32, tx = threadIdx.x, ty = threadIdx.y;
    const size_t plane = (size_t)H * W;
    const float* src = x + blockIdx.z * plane;
    float* dst = out + blockIdx.z * plane;
    for (int r = ty; r < 32; r += 8) {
        const int yy = y0 + r, xx = x0 + tx;
        if (yy < H && xx < W) tile[r][tx] = src[(size_t)yy * W + xx];
    }
    __syncthreads();
    // thread (tx, r) writes the element that came from input (y0 + tx, x0 + r)
    const int yy = y0 + tx;
    if (yy >= H) return;
    for (int r = ty; r < 32; r += 8) {
        const int xx = x0 + r;
        if (xx >= W) break;
        const size_t o = k == 1 ? (size_t)(W - 1 - xx) * H + yy : (size_t)xx * H + (H - 1 - yy);
        dst[o] = tile[tx][r];
    }
}

}  // namespace nb200

using namespace nb200;

extern "C" int nb200_rot90(const float* x, int planes, int H, int W, int k, float* out, void* stream) {
    NB_CHECK(x && out && x != out, "null or aliased pointer");
    NB_CHECK(planes > 0 && planes <= 65535 && H > 0 && W > 0, "bad shape");
    NB_CHECK(k == 1 || k == 3, "k must be 1 or 3");
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope ps(st, PC_OTHER, (double)planes * H * W * 8);
    rot90_kernel<<<dim3(cdiv(W, 32), cdiv(H, 32), planes), dim3(32, 8), 0, st>>>(x, out, H, W, k);
    NB_LAUNCHED();
    return 0;
}

extern "C" int nb200_hwc_to_chw_f32(const void* x, int bits, int B, int H, int W, float* out, void* stream) {
    NB_CHECK(x && out, "null pointer");
    NB_CHECK(bits == 8 || bits == 16, "bits must be 8 or 16");
    NB_CHECK(B > 0 && H > 0 && W > 0, "bad shape");
    const size_t plane = (size_t)H * W, total = plane * B;
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope ps(st, PC_OTHER, (double)total * (3.0 * bits / 8 + 12));
    if (bits == 8) hwc_to_chw_kernel<uint8_t><<<(unsigned)cdiv64((int64_t)total, 256), 256, 0, st>>>((const uint8_t*)x, out, plane, total, 255.f);
    else hwc_to_chw_kernel<uint16_t><<<(unsigned)cdiv64((int64_t)total, 256), 256, 0, st>>>((const uint16_t*)x, out, plane, total, 65535.f);
    NB_LAUNCHED();
    return 0;
}

extern "C" int nb200_chw_f32_to_hwc(const float* x, int bits, int B, int H, int W, void* out, void* stream) {
    NB_CHECK(x && out, "null pointer");
    NB_CHECK(bits == 8 || bits == 16, "bits must be 8 or 16");
    NB_CHECK(B > 0 && H > 0 && W > 0, "bad shape");
    const size_t plane = (size_t)H * W, total = plane * B;
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope ps(st, PC_OTHER, (double)total * (3.0 * bits / 8 + 12));
    if (bits == 8) chw_to_hwc_kernel<uint8_t><<<(unsigned)cdiv64((int64_t)total, 256), 256, 0, st>>>(x, (uint8_t*)out, plane, total, 255.f, 255.f);
    else chw_to_hwc_kernel<uint16_t><<<(unsigned)cdiv64((int64_t)total, 256), 256, 0, st>>>(x, (uint16_t*)out, plane, total, 65535.f, 65535.f);
    NB_LAUNCHED();
    return 0;
}

// iw3/depth_anything_model.py:69-101 (integers; Python float == C double)
extern "C" int nb200_da_preprocess_size(int H, int W, int lower_bound, int max_aspect_ratio, int limit_resolution,
                                        int* new_h, int* new_w) {
    NB_CHECK(new_h && new_w, "null pointer");
    NB_CHECK(H > 0 && W > 0 && lower_bound > 0 && max_aspect_ratio > 0, "bad argument");
    const int mult = 14, min_res = 224;
    if (limit_resolution && lower_bound > (W < H ? W : H)) {
        lower_bound = W < H ? W : H;
        lower_bound -= lower_bound % mult;
        if (lower_bound < min_res) lower_bound = min_res;
    }
    const double sf = W < H ? (double)lower_bound / (double)W : (double)lower_bound / (double)H;
    int nh = (int)((double)H * sf), nw = (int)((double)W * sf);
    if (nh < nw) { const int cap = max_aspect_ratio * nh; if (nw > cap) nw = cap; }
    else { const int cap = max_aspect_ratio * nw; if (nh > cap) nh = cap; }
    nh -= nh % mult;
    nw -= nw % mult;
    if (nh < lower_bound) nh = lower_bound;
    if (nw < lower_bound) nw = lower_bound;
    *new_h = nh;
    *new_w = nw;
    return 0;
}

static int launch_prep(const float* x, int B, int H, int W, int frame_h, int frame_w, int pad_h, int pad_w, const float* mean,
                       const float* stdv, float* out, void* stream, int plain = 0) {
    DaPrepParams p;
    p.plain = plain;
    p.x = x; p.out = out; p.B = B; p.H = H; p.W = W; p.oh = frame_h; p.ow = frame_w; p.pad_h = pad_h; p.pad_w = pad_w;
    p.sy = (float)H / (float)frame_h;   // area_pixel_compute_scale, align_corners=False, no scale_factor given
    p.sx = (float)W / (float)frame_w;
    for (int c = 0; c < 3; ++c) { p.mean[c] = mean[c]; p.stdv[c] = stdv[c]; }
    cudaStream_t st = (cudaStream_t)stream;
    const int OH = frame_h + 2 * pad_h, OW = frame_w + 2 * pad_w;
    ProfScope ps(st, PC_OTHER, (double)B * 3 * ((double)H * W + (double)OH * OW) * 4);
    da_preprocess_kernel<<<dim3(cdiv(OW, 128), OH, B), 128, 0, st>>>(p);
    NB_LAUNCHED();
    return 0;
}

extern "C" int nb200_da_preprocess(const float* x, int B, int H, int W, int new_h, int new_w, float* out, void* stream) {
    NB_CHECK(x && out, "null pointer");
    NB_CHECK(B > 0 && H > 0 && W > 0 && new_h > 0 && new_w > 0, "bad shape");
    const float mean[3] = {0.485f, 0.456f, 0.406f}, stdv[3] = {0.229f, 0.224f, 0.225f};
    return launch_prep(x, B, H, W, new_h, new_w, 0, 0, mean, stdv, out, stream);
}

// F.interpolate(x, (new_h, new_w), mode="bilinear", antialias=True, align_corners=False) alone (iw3/forward_inpaint.py:74-81)
extern "C" int nb200_resize_bilinear_aa(const float* x, int B, int H, int W, int new_h, int new_w, float* out, void* stream) {
    NB_CHECK(x && out, "null pointer");
    NB_CHECK(B > 0 && H > 0 && W > 0 && new_h > 0 && new_w > 0, "bad shape");
    const float zero[3] = {0.f, 0.f, 0.f}, one[3] = {1.f, 1.f, 1.f};
    return launch_prep(x, B, H, W, new_h, new_w, 0, 0, zero, one, out, stream, 1);
}

// iw3/zoedepth_model.py:30-71 (integers; Python float == C double, round() == round-half-even)
extern "C" int nb200_zoe_preprocess_size(int H, int W, int h_height, int v_height, int mod, int* new_h, int* new_w, int* pad_h,
                                         int* pad_w, int* frame_h, int* frame_w) {
    NB_CHECK(new_h && new_w && pad_h && pad_w && frame_h && frame_w, "null pointer");
    NB_CHECK(H > 0 && W > 0 && h_height > 0 && v_height > 0 && mod > 0, "bad argument");
    const int target = W > H ? h_height : v_height;
    int nh, nw;
    if (target < H) {
        nh = target;
        nw = (int)((double)nh / (double)H * (double)W);
        if (nw % mod) nw += mod - nw % mod;
        if (nh % mod) nh += mod - nh % mod;
    } else {
        nh = H; nw = W;
        if (nw % mod) nw -= nw % mod;
        if (nh % mod) nh -= nh % mod;
    }
    const int psh = (int)(std::sqrt((double)H * 0.5) * 3.0), psw = (int)(std::sqrt((double)W * 0.5) * 3.0);
    const double sh = (double)psh / (double)(H + psh * 2), sw = (double)psw / (double)(W + psw * 2);
    int ph, pw, fh, fw;
    if (nh > nw) {
        ph = (int)std::nearbyint((double)nh * sh);
        fh = nh - ph * 2;
        fw = (int)((double)W * ((double)fh / (double)H));
        fw += fw % 2;
        pw = (nh - fw) / 2;
    } else {
        ph = (int)std::nearbyint((double)nh * sh);
        pw = (int)std::nearbyint((double)nw * sw);
        fh = nh - ph * 2;
        fw = nw - pw * 2;
    }
    NB_CHECK(fh > 0 && fw > 0, "frame too small for the reflection padding");
    *new_h = nh; *new_w = nw; *pad_h = ph; *pad_w = pw; *frame_h = fh; *frame_w = fw;
    return 0;
}

// ZoeDepth batch_preprocess body (zoedepth_model.py:62-82): AA resize to frame_h x frame_w, reflection pad, clamp,
// normalise with mean = std = 0.5 -> out [B][3][frame_h + 2*pad_h][frame_w + 2*pad_w]
extern "C" int nb200_zoe_preprocess(const float* x, int B, int H, int W, int frame_h, int frame_w, int pad_h, int pad_w, float* out,
                                    void* stream) {
    NB_CHECK(x && out, "null pointer");
    NB_CHECK(B > 0 && H > 0 && W > 0 && frame_h > 0 && frame_w > 0 && pad_h >= 0 && pad_w >= 0, "bad shape");
    NB_CHECK((pad_h == 0 || frame_h > 1) && (pad_w == 0 || frame_w > 1), "cannot reflect a 1-pixel frame");
    const float mean[3] = {0.5f, 0.5f, 0.5f}, stdv[3] = {0.5f, 0.5f, 0.5f};
    return launch_prep(x, B, H, W, frame_h, frame_w, pad_h, pad_w, mean, stdv, out, stream);
}
