// Planar YUV <-> integer RGB for the frame pipeline's two ends: the work of PyAV's
// to_ndarray(format="rgb24" | "rgb48le", src_colorspace, src_color_range, dst_color_range=JPEG) on decoded frames and of
// frame.reformat(format=pix_fmt, dst_colorspace, dst_color_range) on the frames handed to the encoder
// (nunif/utils/video.py:621-639 guess_rgb24_options, :763-850 configure_colorspace), which the reference runs on the CPU
// through libswscale.
//
// One frame is one buffer: Y [H][W], then U and V [ch][cw] (cw = ceil(W / sx), ch = ceil(H / sy)), each row pitch equal
// to its width, frames frame_stride elements apart (the tail past the three planes is padding; rgb_to_yuv zeroes it).
// 8-bit planes are uint8, 10- and 16-bit planes uint16 holding the code in the low bits (the *le formats).
//
// One thread per chroma sample: it reads its U / V once and converts the sx x sy luma block they cover.  yuv -> rgb
// replicates the chroma over the block (swscale's unscaled yuv2rgb path); rgb -> yuv writes the block's luma and the mean
// of its full-resolution Cb / Cr (fewer samples at an odd right / bottom edge).  Round to nearest even, clamp to the code
// range.  The arithmetic is fp64: fp32's 24-bit significand leaves a 16-bit rgb48 code about 1/256 of a code of
// headroom, so about one rgb48 sample in a hundred would round differently from the conversion's definition; the few fp64
// operations per sample stay far below the time the kernels' memory traffic takes on an H100.
#include "common.cuh"
#include "../../include/nunif_b200.h"

namespace nb200 {

namespace {

// yuv -> rgb: out = ys * (Y - yo) + {rv * V', gu * U' + gv * V', bu * U'} with U' = U - co, V' = V - co, already scaled to
// the output code range.  rgb -> yuv: {Y, U, V} = {yo, co, co} + m (3 x 3) * (R, G, B) on input codes.
struct YuvCoef {
    double yo, co;
    double ys, rv, gu, gv, bu;
    double m[9];
    double out_max;
};

template <typename T>
__device__ __forceinline__ T code(double v, double vmax) {
    return (T)rint(fmin(fmax(v, 0.0), vmax));
}

template <int SX, int SY, typename TI, typename TO>
__global__ void __launch_bounds__(256) yuv_to_rgb_kernel(const TI* __restrict__ planes, int64_t frame_stride, int H, int W,
                                                         int cw, int ch, YuvCoef p, TO* __restrict__ out) {
    const int cx = blockIdx.x * blockDim.x + threadIdx.x, cy = blockIdx.y * blockDim.y + threadIdx.y, b = blockIdx.z;
    if (cx >= cw || cy >= ch) return;
    const TI* Yp = planes + (int64_t)b * frame_stride;
    const TI* Up = Yp + (int64_t)H * W;
    const TI* Vp = Up + (int64_t)cw * ch;
    const double u = (double)__ldg(Up + (int64_t)cy * cw + cx) - p.co, v = (double)__ldg(Vp + (int64_t)cy * cw + cx) - p.co;
    const double dr = p.rv * v, dg = fma(p.gu, u, p.gv * v), db = p.bu * u;
    TO* o = out + (int64_t)b * H * W * 3;
#pragma unroll
    for (int dy = 0; dy < SY; ++dy) {
        const int y = cy * SY + dy;
        if (SY > 1 && y >= H) break;
#pragma unroll
        for (int dx = 0; dx < SX; ++dx) {
            const int x = cx * SX + dx;
            if (SX > 1 && x >= W) break;
            const int64_t i = (int64_t)y * W + x;
            const double yv = p.ys * ((double)__ldg(Yp + i) - p.yo);
            o[i * 3 + 0] = code<TO>(yv + dr, p.out_max);
            o[i * 3 + 1] = code<TO>(yv + dg, p.out_max);
            o[i * 3 + 2] = code<TO>(yv + db, p.out_max);
        }
    }
}

template <int SX, int SY, typename TI, typename TO>
__global__ void __launch_bounds__(256) rgb_to_yuv_kernel(const TI* __restrict__ rgb, int H, int W, int cw, int ch,
                                                         int64_t frame_stride, YuvCoef p, TO* __restrict__ planes) {
    const int cx = blockIdx.x * blockDim.x + threadIdx.x, cy = blockIdx.y * blockDim.y + threadIdx.y, b = blockIdx.z;
    if (cx >= cw || cy >= ch) return;
    const TI* in = rgb + (int64_t)b * H * W * 3;
    TO* Yp = planes + (int64_t)b * frame_stride;
    TO* Up = Yp + (int64_t)H * W;
    TO* Vp = Up + (int64_t)cw * ch;
    double su = 0.0, sv = 0.0;
    int n = 0;
#pragma unroll
    for (int dy = 0; dy < SY; ++dy) {
        const int y = cy * SY + dy;
        if (SY > 1 && y >= H) break;
#pragma unroll
        for (int dx = 0; dx < SX; ++dx) {
            const int x = cx * SX + dx;
            if (SX > 1 && x >= W) break;
            const int64_t i = (int64_t)y * W + x;
            const double r = __ldg(in + i * 3 + 0), g = __ldg(in + i * 3 + 1), bl = __ldg(in + i * 3 + 2);
            Yp[i] = code<TO>(p.yo + fma(p.m[0], r, fma(p.m[1], g, p.m[2] * bl)), p.out_max);
            su += fma(p.m[3], r, fma(p.m[4], g, p.m[5] * bl));
            sv += fma(p.m[6], r, fma(p.m[7], g, p.m[8] * bl));
            ++n;
        }
    }
    const int64_t c = (int64_t)cy * cw + cx;
    const double inv = n == 4 ? 0.25 : n == 2 ? 0.5 : 1.0;
    Up[c] = code<TO>(p.co + su * inv, p.out_max);
    Vp[c] = code<TO>(p.co + sv * inv, p.out_max);
    // padding after V (odd widths of the subsampled layouts): zero it so that the frame buffer is deterministic
    const int64_t used = (int64_t)H * W + 2 * (int64_t)cw * ch;
    for (int64_t k = c; used + k < frame_stride; k += (int64_t)cw * ch) Yp[used + k] = 0;
}

// planar RGB reorder (gbrp*): G, B, R planes of W x H, each code rescaled to the output depth
template <typename TI, typename TO>
__global__ void __launch_bounds__(256) rgb_to_gbr_kernel(const TI* __restrict__ rgb, int64_t hw, int64_t frame_stride,
                                                         double scale, double out_max, TO* __restrict__ planes) {
    const int64_t i = (int64_t)blockIdx.x * blockDim.x + threadIdx.x, b = blockIdx.y;
    if (i >= hw) return;
    const TI* in = rgb + (b * hw + i) * 3;
    TO* o = planes + b * frame_stride;
    o[i] = code<TO>(__ldg(in + 1) * scale, out_max);
    o[hw + i] = code<TO>(__ldg(in + 2) * scale, out_max);
    o[2 * hw + i] = code<TO>(__ldg(in + 0) * scale, out_max);
}

int sub_x(int layout) { return layout == NB200_YUV444 || layout == NB200_GBR ? 1 : 2; }
int sub_y(int layout) { return layout == NB200_YUV420 ? 2 : 1; }

bool kr_kb(int matrix, double& kr, double& kb) {
    switch (matrix) {
        case NB200_MATRIX_BT601: kr = 0.299; kb = 0.114; return true;      // ITU-R BT.601
        case NB200_MATRIX_BT709: kr = 0.2126; kb = 0.0722; return true;    // ITU-R BT.709
        case NB200_MATRIX_BT2020: kr = 0.2627; kb = 0.0593; return true;   // ITU-R BT.2020 non-constant luminance
        default: return false;
    }
}

// code offsets and spans of a YUV depth: limited range puts Y in [16, 235] and Cb / Cr in [16, 240] (x 2^(bits-8)),
// full range uses the whole code range with the chroma zero at 2^(bits-1)
void yuv_range(int bits, int range, double& yo, double& co, double& yspan, double& cspan) {
    const double s = (double)(1 << (bits - 8)), vmax = (double)((1 << bits) - 1);
    co = (double)(1 << (bits - 1));
    if (range == NB200_RANGE_LIMITED) { yo = 16 * s; yspan = 219 * s; cspan = 224 * s; }
    else { yo = 0; yspan = cspan = vmax; }
}

bool valid_bits(int bits) { return bits == 8 || bits == 10 || bits == 16; }

template <int SX, int SY, typename TI, typename TO>
void launch_yuv2rgb(const void* planes, int64_t fs, int B, int H, int W, int cw, int ch, const YuvCoef& p, void* out,
                    cudaStream_t st) {
    const dim3 block(32, 8), grid(cdiv(cw, 32), cdiv(ch, 8), B);
    yuv_to_rgb_kernel<SX, SY, TI, TO><<<grid, block, 0, st>>>((const TI*)planes, fs, H, W, cw, ch, p, (TO*)out);
}

template <int SX, int SY, typename TI, typename TO>
void launch_rgb2yuv(const void* rgb, int B, int H, int W, int cw, int ch, int64_t fs, const YuvCoef& p, void* planes,
                    cudaStream_t st) {
    const dim3 block(32, 8), grid(cdiv(cw, 32), cdiv(ch, 8), B);
    rgb_to_yuv_kernel<SX, SY, TI, TO><<<grid, block, 0, st>>>((const TI*)rgb, H, W, cw, ch, fs, p, (TO*)planes);
}

}  // namespace

}  // namespace nb200

using namespace nb200;

extern "C" int nb200_yuv_to_rgb(const void* planes, int layout, int bits, int matrix, int range, int frame_stride, int B,
                                int H, int W, int rgb_bits, void* out, void* stream) {
    NB_CHECK(planes && out, "null pointer");
    NB_CHECK(B > 0 && H > 0 && W > 0, "bad shape");
    NB_CHECK(layout == NB200_YUV420 || layout == NB200_YUV422 || layout == NB200_YUV444,
             "layout must be NB200_YUV420, NB200_YUV422 or NB200_YUV444");
    NB_CHECK(bits == 8 || bits == 10, "YUV bits must be 8 or 10");
    NB_CHECK(rgb_bits == 8 || rgb_bits == 16, "rgb_bits must be 8 (rgb24) or 16 (rgb48)");
    NB_CHECK(range == NB200_RANGE_LIMITED || range == NB200_RANGE_FULL, "bad range");
    double kr, kb;
    NB_CHECK(kr_kb(matrix, kr, kb), "bad matrix");
    const int sx = sub_x(layout), sy = sub_y(layout), cw = cdiv(W, sx), ch = cdiv(H, sy);
    NB_CHECK((int64_t)frame_stride >= (int64_t)H * W + 2 * (int64_t)cw * ch, "frame_stride smaller than the three planes");
    double yo, co, yspan, cspan;
    yuv_range(bits, range, yo, co, yspan, cspan);
    const double kg = 1.0 - kr - kb, omax = (double)((1 << rgb_bits) - 1), cs = omax / cspan;
    YuvCoef p{};
    p.yo = yo;
    p.co = co;
    p.ys = omax / yspan;
    p.rv = cs * 2 * (1 - kr);
    p.gu = -cs * 2 * kb * (1 - kb) / kg;
    p.gv = -cs * 2 * kr * (1 - kr) / kg;
    p.bu = cs * 2 * (1 - kb);
    p.out_max = omax;
    cudaStream_t st = (cudaStream_t)stream;
    const size_t ib = bits > 8 ? 2 : 1, ob = rgb_bits > 8 ? 2 : 1;
    ProfScope ps(st, PC_OTHER, (double)B * ((double)H * W * (ib + 3 * ob) + 2.0 * cw * ch * ib));
#define NB_Y2R(SX, SY)                                                                                             \
    if (bits > 8 && rgb_bits > 8) launch_yuv2rgb<SX, SY, uint16_t, uint16_t>(planes, frame_stride, B, H, W, cw, ch, p, out, st); \
    else if (bits > 8) launch_yuv2rgb<SX, SY, uint16_t, uint8_t>(planes, frame_stride, B, H, W, cw, ch, p, out, st);          \
    else if (rgb_bits > 8) launch_yuv2rgb<SX, SY, uint8_t, uint16_t>(planes, frame_stride, B, H, W, cw, ch, p, out, st);      \
    else launch_yuv2rgb<SX, SY, uint8_t, uint8_t>(planes, frame_stride, B, H, W, cw, ch, p, out, st);
    if (layout == NB200_YUV420) { NB_Y2R(2, 2) }
    else if (layout == NB200_YUV422) { NB_Y2R(2, 1) }
    else { NB_Y2R(1, 1) }
#undef NB_Y2R
    NB_LAUNCHED();
    return 0;
}

extern "C" int nb200_rgb_to_yuv(const void* rgb, int rgb_bits, int B, int H, int W, int layout, int bits, int matrix,
                                int range, int frame_stride, void* planes, void* stream) {
    NB_CHECK(rgb && planes, "null pointer");
    NB_CHECK(B > 0 && H > 0 && W > 0, "bad shape");
    NB_CHECK(rgb_bits == 8 || rgb_bits == 16, "rgb_bits must be 8 (rgb24) or 16 (rgb48)");
    NB_CHECK(layout == NB200_YUV420 || layout == NB200_YUV422 || layout == NB200_YUV444 || layout == NB200_GBR,
             "layout must be NB200_YUV420, NB200_YUV422, NB200_YUV444 or NB200_GBR");
    NB_CHECK(valid_bits(bits) && (bits != 16 || layout == NB200_GBR), "bits must be 8 or 10 (16 only for NB200_GBR)");
    const int sx = sub_x(layout), sy = sub_y(layout), cw = cdiv(W, sx), ch = cdiv(H, sy);
    NB_CHECK((int64_t)frame_stride >= (int64_t)H * W + 2 * (int64_t)cw * ch, "frame_stride smaller than the three planes");
    const double imax = (double)((1 << rgb_bits) - 1), omax = (double)((1 << bits) - 1);
    cudaStream_t st = (cudaStream_t)stream;
    const size_t ib = rgb_bits > 8 ? 2 : 1, ob = bits > 8 ? 2 : 1;
    ProfScope ps(st, PC_OTHER, (double)B * ((double)H * W * (3 * ib + ob) + 2.0 * cw * ch * ob));
    if (layout == NB200_GBR) {
        NB_CHECK(frame_stride == 3 * H * W, "NB200_GBR frames are exactly three planes");
        const int64_t hw = (int64_t)H * W;
        const dim3 grid((unsigned)cdiv64(hw, 256), B);
        const double scale = omax / imax, om = omax;
        if (rgb_bits > 8 && bits > 8) rgb_to_gbr_kernel<<<grid, 256, 0, st>>>((const uint16_t*)rgb, hw, frame_stride, scale, om, (uint16_t*)planes);
        else if (rgb_bits > 8) rgb_to_gbr_kernel<<<grid, 256, 0, st>>>((const uint16_t*)rgb, hw, frame_stride, scale, om, (uint8_t*)planes);
        else if (bits > 8) rgb_to_gbr_kernel<<<grid, 256, 0, st>>>((const uint8_t*)rgb, hw, frame_stride, scale, om, (uint16_t*)planes);
        else rgb_to_gbr_kernel<<<grid, 256, 0, st>>>((const uint8_t*)rgb, hw, frame_stride, scale, om, (uint8_t*)planes);
        NB_LAUNCHED();
        return 0;
    }
    NB_CHECK(range == NB200_RANGE_LIMITED || range == NB200_RANGE_FULL, "bad range");
    double kr, kb;
    NB_CHECK(kr_kb(matrix, kr, kb), "bad matrix");
    double yo, co, yspan, cspan;
    yuv_range(bits, range, yo, co, yspan, cspan);
    const double kg = 1.0 - kr - kb, ys = yspan / imax, us = cspan / imax / (2 * (1 - kb)), vs = cspan / imax / (2 * (1 - kr));
    const double m[9] = {ys * kr, ys * kg, ys * kb,
                         -us * kr, -us * kg, us * (1 - kb),
                         vs * (1 - kr), -vs * kg, -vs * kb};
    YuvCoef p{};
    p.yo = yo;
    p.co = co;
    for (int i = 0; i < 9; ++i) p.m[i] = m[i];
    p.out_max = omax;
#define NB_R2Y(SX, SY)                                                                                             \
    if (rgb_bits > 8 && bits > 8) launch_rgb2yuv<SX, SY, uint16_t, uint16_t>(rgb, B, H, W, cw, ch, frame_stride, p, planes, st); \
    else if (rgb_bits > 8) launch_rgb2yuv<SX, SY, uint16_t, uint8_t>(rgb, B, H, W, cw, ch, frame_stride, p, planes, st);          \
    else if (bits > 8) launch_rgb2yuv<SX, SY, uint8_t, uint16_t>(rgb, B, H, W, cw, ch, frame_stride, p, planes, st);              \
    else launch_rgb2yuv<SX, SY, uint8_t, uint8_t>(rgb, B, H, W, cw, ch, frame_stride, p, planes, st);
    if (layout == NB200_YUV420) { NB_R2Y(2, 2) }
    else if (layout == NB200_YUV422) { NB_R2Y(2, 1) }
    else { NB_R2Y(1, 1) }
#undef NB_R2Y
    NB_LAUNCHED();
    return 0;
}
