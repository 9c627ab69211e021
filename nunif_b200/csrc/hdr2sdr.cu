// HDR10 (PQ) / HLG BT.2020 -> BT.709 / BT.601 SDR tone map of rgb48 frames (nunif/utils/video.py:309-416 hdr2sdr, steps 1-6),
// one fused pass over x [B][H][W][3] uint16 -> the uint16 rgb48 frame hdr2sdr returns, or that frame / 65535 as fp32 BCHW
// (what nb200_hwc_to_chw_f32 makes of it): the reference runs ~30 ATen kernels over fp32 CHW per frame.
//
// Numerics follow the reference's ops one by one as ATen evaluates them on CUDA: every op rounds to fp32 once (_rn
// intrinsics, so nothing is contracted into an FMA), powf / expf are the accurate libdevice functions ATen calls, a
// division by a Python scalar is a multiply by its fp32 reciprocal (ATen div_true with a CPU scalar), every Python-double
// constant enters as one fp32 scalar (compound constants such as C*B are folded in double first), pow(x, 2.0) is x*x.
// The one step that cannot be matched bit for bit is the 3x3 colour matrix (torch.mm, cuBLAS: unspecified summation order);
// it is evaluated as fma(m2, s2, fma(m1, s1, m0*s0)).  The final cast truncates.
#include "common.cuh"
#include "../../include/nunif_b200.h"

namespace nb200 {

namespace {

constexpr int kThreads = 256;       // one pixel per thread; a block's 256 pixels are 1536 B = 96 uint4

struct Hdr2SdrParams {
    float m[9];                     // BT.2020 -> target RGB matrix, row-major
    float exposure, white;          // fp32 scalars of the Python floats of the selected transfer
    float sat_gain, one_minus_gain; // HLG saturation blend: gain and fl(1.0 - gain) folded in double
    int saturate;                   // hlg_saturation_gain < 1.0
};

template <bool HLG>
__device__ __forceinline__ float hable(float v) {
    // video.py:356-358; E = 0.02 (PQ) / 0.01 (HLG).  C*B, D*E, D*F and E/F are Python-double products
    constexpr double E = HLG ? 0.01 : 0.02;
    const float A = (float)0.15, B = (float)0.50, CB = (float)(0.10 * 0.50), DE = (float)(0.20 * E), DF = (float)(0.20 * 0.30),
                EF = (float)(E / 0.30);
    const float num = __fadd_rn(__fmul_rn(v, __fadd_rn(__fmul_rn(A, v), CB)), DE);
    const float den = __fadd_rn(__fmul_rn(v, __fadd_rn(__fmul_rn(A, v), B)), DF);
    return __fsub_rn(__fdiv_rn(num, den), EF);
}

// inverse EOTF of one channel (video.py:328-344)
template <bool HLG>
__device__ __forceinline__ float to_linear(float x) {
    if (!HLG) {
        constexpr double m1 = 2610.0 / 16384, m2 = 2523.0 / 4096 * 128;
        const float c1 = (float)(3424.0 / 4096), c2 = (float)(2413.0 / 4096 * 32), c3 = (float)(2392.0 / 4096 * 32);
        const float xp = powf(x, (float)(1.0 / m2));
        const float t = fmaxf(__fsub_rn(xp, c1), 0.f);
        return powf(__fdiv_rn(t, __fsub_rn(c2, __fmul_rn(c3, xp))), (float)(1.0 / m1));
    } else {
        const float a_inv = 1.f / (float)0.17883277, b = (float)0.28466892, c = (float)0.55991073;
        return x <= 0.5f ? __fmul_rn(__fmul_rn(x, x), 1.f / 3.f)
                         : __fmul_rn(__fadd_rn(expf(__fmul_rn(__fsub_rn(x, c), a_inv)), b), 1.f / 12.f);
    }
}

// BT.709 / BT.601 OETF between the two clamps (video.py:388-398), then the truncating cast to uint16
__device__ __forceinline__ uint16_t oetf_u16(float v) {
    v = clamp01(v);
    v = v < (float)0.018 ? __fmul_rn(v, 4.5f) : __fsub_rn(__fmul_rn((float)1.099, powf(v, (float)0.45)), (float)0.099);
    return (uint16_t)__float2uint_rz(__fmul_rn(clamp01(v), 65535.f));
}

template <bool HLG, bool OUT_F32>
__global__ void __launch_bounds__(kThreads) hdr2sdr_kernel(const uint16_t* __restrict__ x, void* __restrict__ out, int64_t total,
                                                         int64_t plane, Hdr2SdrParams p, int vec) {
    __shared__ __align__(16) uint16_t tile[kThreads * 3];
    const int64_t p0 = (int64_t)blockIdx.x * kThreads;
    const int n = (int)min((int64_t)kThreads, total - p0);
    const int t = threadIdx.x;
    // stage the block's pixels through shared memory: 6-byte pixels are not aligned for a per-thread vector load
    if (vec && n == kThreads) {
        if (t < kThreads * 3 / 8) reinterpret_cast<uint4*>(tile)[t] = __ldg(reinterpret_cast<const uint4*>(x + p0 * 3) + t);
    } else {
        for (int i = t; i < n * 3; i += kThreads) tile[i] = x[p0 * 3 + i];
    }
    __syncthreads();
    uint16_t q[3];
    if (t < n) {
        const float inv = 1.f / 65535.f;   // uint16 / 65535.0 on CUDA: a multiply by the fp32 reciprocal
        const float hw = hable<HLG>(p.white);
        float s[3];
#pragma unroll
        for (int c = 0; c < 3; ++c)
            s[c] = __fdiv_rn(hable<HLG>(__fmul_rn(to_linear<HLG>(__fmul_rn((float)tile[t * 3 + c], inv)), p.exposure)), hw);
        if (HLG && p.saturate) {           // video.py:363-367
            const float luma = __fadd_rn(__fadd_rn(__fmul_rn(s[0], (float)0.2126), __fmul_rn(s[1], (float)0.7152)),
                                         __fmul_rn(s[2], (float)0.0722));
#pragma unroll
            for (int c = 0; c < 3; ++c) s[c] = __fadd_rn(__fmul_rn(s[c], p.sat_gain), __fmul_rn(luma, p.one_minus_gain));
        }
#pragma unroll
        for (int r = 0; r < 3; ++r)
            q[r] = oetf_u16(fmaf(p.m[r * 3 + 2], s[2], fmaf(p.m[r * 3 + 1], s[1], __fmul_rn(p.m[r * 3], s[0]))));
    }
    if (OUT_F32) {
        if (t < n) {
            const int64_t i = p0 + t, b = i / plane;
            float* o = static_cast<float*>(out) + b * 3 * plane + (i - b * plane);
            // nb200_hwc_to_chw_f32 of the uint16 frame: a true division
#pragma unroll
            for (int c = 0; c < 3; ++c) o[c * plane] = __fdiv_rn((float)q[c], 65535.f);
        }
    } else {
        if (t < n) {                      // each thread overwrites only the pixel it read
#pragma unroll
            for (int c = 0; c < 3; ++c) tile[t * 3 + c] = q[c];
        }
        __syncthreads();
        uint16_t* o = static_cast<uint16_t*>(out) + p0 * 3;
        if (vec && n == kThreads) {
            if (t < kThreads * 3 / 8) reinterpret_cast<uint4*>(o)[t] = reinterpret_cast<const uint4*>(tile)[t];
        } else {
            for (int i = t; i < n * 3; i += kThreads) o[i] = tile[i];
        }
    }
}

template <bool HLG>
void launch(const uint16_t* x, void* out, int out_f32, int64_t total, int64_t plane, const Hdr2SdrParams& p, int vec,
            cudaStream_t st) {
    const unsigned grid = (unsigned)cdiv64(total, kThreads);
    if (out_f32) hdr2sdr_kernel<HLG, true><<<grid, kThreads, 0, st>>>(x, out, total, plane, p, vec);
    else hdr2sdr_kernel<HLG, false><<<grid, kThreads, 0, st>>>(x, out, total, plane, p, vec);
}

}  // namespace

}  // namespace nb200

using namespace nb200;

extern "C" int nb200_hdr2sdr(const uint16_t* x, int B, int H, int W, int trc, int colorspace, const double* params_host,
                             int out_float, void* out, void* stream) {
    NB_CHECK(x && out && params_host, "null pointer");
    NB_CHECK((const void*)x != out, "out must not alias x");
    NB_CHECK(B > 0 && H > 0 && W > 0, "bad shape");
    NB_CHECK(trc == NB200_TRC_PQ || trc == NB200_TRC_HLG, "trc must be 16 (PQ) or 18 (HLG)");
    NB_CHECK(colorspace == NB200_SDR_BT709 || colorspace == NB200_SDR_BT601, "colorspace must be BT.709 or BT.601");
    static const double kM[2][9] = {
        {1.6605, -0.5876, -0.0728, -0.1246, 1.1329, -0.0083, -0.0182, -0.1006, 1.1187},   // video.py:373-377
        {1.5540, -0.5143, -0.0397, -0.1017, 1.1147, -0.0130, -0.0163, -0.0886, 1.1049},   // video.py:379-383
    };
    const bool hlg = trc == NB200_TRC_HLG;
    Hdr2SdrParams p;
    for (int i = 0; i < 9; ++i) p.m[i] = (float)kM[colorspace == NB200_SDR_BT601][i];
    p.exposure = (float)params_host[hlg ? 2 : 0];
    p.white = (float)params_host[hlg ? 3 : 1];
    p.sat_gain = (float)params_host[4];
    p.one_minus_gain = (float)(1.0 - params_host[4]);
    p.saturate = params_host[4] < 1.0;
    const int64_t plane = (int64_t)H * W, total = plane * B;
    const int vec = ((uintptr_t)x % 16 == 0) && ((uintptr_t)out % 16 == 0);
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope ps(st, PC_OTHER, (double)total * (6 + (out_float ? 12 : 6)));
    if (hlg) launch<true>(x, out, out_float, total, plane, p, vec, st);
    else launch<false>(x, out, out_float, total, plane, p, vec, st);
    NB_LAUNCHED();
    return 0;
}
