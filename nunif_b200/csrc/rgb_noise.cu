// waifu2x film grain (--grain; waifu2x/ui_utils.py:58-61 images, :167-175 video) through nunif/utils/rgb_noise.py:
// rgb_noise_like (:5-17) and apply_rgb_noise (:20-36), and for video the temporal noise buffer, in one pass per batch.
//
// Noise.  Every normal is a pure function of (seed, counter): Philox4x32-10 keyed by the 64-bit seed at the counter
// (element, 2 * channel + field, frame, offset) - field 0 the full-resolution field, element y * W + x; field 1 the
// half-resolution field of level 2, element hy * (W / 2) + hx - and Box-Muller of the first two words with the accurate
// logf / cospif.  Level 2 is 0.5 * full + 0.5 * half[up(y)][up(x)] with ATen's nearest rule for F.interpolate(size=...):
// up(d) = min(int(d * ((float)in / out)), in - 1).  Each thread recomputes the half-resolution value its pixel maps to.
//
// Apply.  The reference's fp32 ops one by one as ATen evaluates them on CUDA: _rn intrinsics so nothing contracts into
// an FMA; x ** e is powf (libdevice) except where ATen's pow takes another path for the exponent (1, 0.5, 2, 3); every
// Python scalar enters as one fp32 value, compound ones (1 - lds, 1 / gamma, 1 - speed) folded in double first.
//
// Temporal.  b = b * (1 - s) + n * s per frame, in frame order, each thread holding its (channel, y, x) of the buffer in a
// register across the batch: the buffer is read and written once per launch.  The first frame of a launch may copy the
// noise into the buffer instead (the reference's resize_ + copy_ on the first frame and on a shape change).
#include "common.cuh"
#include "../../include/nunif_b200.h"

namespace nb200 {

namespace {

constexpr int kThreads = 128;      // one (y, x) pixel per thread, blockIdx.y = row

// how ATen's pow(Tensor, Scalar) evaluates x ** e for a float tensor (pow_out / pow_tensor_scalar_kernel)
enum PowKind : int { POW_GENERIC = 0, POW_ONE, POW_HALF, POW_TWO, POW_THREE };

int pow_kind(double e) {
    return e == 1.0 ? POW_ONE : e == 0.5 ? POW_HALF : e == 2.0 ? POW_TWO : e == 3.0 ? POW_THREE : POW_GENERIC;
}

__device__ __forceinline__ float aten_pow(float x, float e, int kind) {
    switch (kind) {
    case POW_ONE: return x;
    case POW_HALF: return sqrtf(x);
    case POW_TWO: return __fmul_rn(x, x);
    case POW_THREE: return __fmul_rn(__fmul_rn(x, x), x);
    default: return powf(x, e);
    }
}

struct NoiseField {
    uint2 key;             // the 64-bit seed
    int level, W, hh, hw;  // hh x hw = (H / 2) x (W / 2), the half-resolution field of level 2
    float sy, sx;          // ATen's nearest scales (float)hh / H, (float)hw / W
};

__device__ __forceinline__ float philox_normal(uint2 key, uint32_t elem, uint32_t stream, uint32_t frame, uint32_t offset) {
    const uint4 r = philox4x32_10(make_uint4(elem, stream, frame, offset), key);
    const float u1 = ((float)(r.x >> 9) + 0.5f) * 0x1p-23f;   // (0, 1), exact: k + 0.5 fits 24 bits
    const float a = (float)(r.y >> 8) * 0x1p-23f;             // 2 * u2 in [0, 2), exact
    return __fmul_rn(sqrtf(__fmul_rn(-2.f, logf(u1))), cospif(a));
}

// rgb_noise_like's value at (frame, offset, c, y, x)
__device__ __forceinline__ float noise_at(const NoiseField& f, uint32_t frame, uint32_t offset, int c, int y, int x) {
    const float n = philox_normal(f.key, (uint32_t)y * f.W + x, 2u * c, frame, offset);
    if (f.level == 1) return n;
    const int hy = min((int)__fmul_rn((float)y, f.sy), f.hh - 1), hx = min((int)__fmul_rn((float)x, f.sx), f.hw - 1);
    const float h = philox_normal(f.key, (uint32_t)hy * f.hw + hx, 2u * c + 1, frame, offset);
    return __fadd_rn(__fmul_rn(n, 0.5f), __fmul_rn(0.5f, h));   // noise.mul_(0.5).add_(noise2, alpha=0.5)
}

__global__ void __launch_bounds__(kThreads) rgb_noise_kernel(NoiseField f, uint32_t offset, int B, int C, int H, float* __restrict__ out) {
    const int x = blockIdx.x * kThreads + threadIdx.x, y = blockIdx.y;
    if (x >= f.W) return;
    const size_t plane = (size_t)H * f.W, p = (size_t)y * f.W + x;
    for (int b = 0; b < B; ++b)
        for (int c = 0; c < C; ++c) out[((size_t)b * C + c) * plane + p] = noise_at(f, (uint32_t)b, offset, c, y, x);
}

struct ApplyParams {
    const float* rgb;      // [B][C][H][W]
    const float* noise;    // [B][C][H][W], or null: generate frame b's noise as rgb_noise_like(seed, offset + b)
    float* buffer;         // [C][H][W] temporal noise buffer, or null
    void* out;             // [B][C][H][W] fp32, or [B][H][W][3] uint8 / uint16
    int B, C, H, reset;    // reset: frame 0 copies its noise into the buffer instead of blending
    uint32_t offset;
    float strength, gamma, inv_gamma, lds, one_minus_lds, speed, one_minus_speed;
    int pow_gamma, pow_inv_gamma, light_decay;
};

// OUT_BITS 0: fp32 CHW; 8 / 16: (x * 255 | 65535).round_().to(uint8 | uint16) as HWC, as from_tensor makes the frame
template <int OUT_BITS, bool GEN>
__global__ void __launch_bounds__(kThreads) apply_rgb_noise_kernel(ApplyParams p, NoiseField f) {
    const int x = blockIdx.x * kThreads + threadIdx.x, y = blockIdx.y;
    if (x >= f.W) return;
    const size_t plane = (size_t)p.H * f.W, px = (size_t)y * f.W + x;
    for (int c = 0; c < p.C; ++c) {
        float buf = p.buffer && !p.reset ? p.buffer[c * plane + px] : 0.f;
        for (int b = 0; b < p.B; ++b) {
            const size_t i = ((size_t)b * p.C + c) * plane + px;
            float n = GEN ? noise_at(f, 0u, p.offset + (uint32_t)b, c, y, x) : __ldg(p.noise + i);
            if (p.buffer) {        // ui_utils.py:168-174
                buf = (b == 0 && p.reset) ? n : __fadd_rn(__fmul_rn(buf, p.one_minus_speed), __fmul_rn(n, p.speed));
                n = buf;
            }
            // rgb_noise.py:25-35
            float o = aten_pow(__ldg(p.rgb + i), p.gamma, p.pow_gamma);
            const float corr = __fmul_rn(n, o);
            const float ld = p.light_decay
                ? aten_pow(__fadd_rn(__fmul_rn(__fsub_rn(1.f, o), p.lds), p.one_minus_lds), p.gamma, p.pow_gamma) : 1.f;
            o = __fadd_rn(o, __fmul_rn(corr, __fmul_rn(ld, p.strength)));
            o = isnan(o) ? o : clamp01(o);    // clamp_ keeps NaN
            const float v = aten_pow(o, p.inv_gamma, p.pow_inv_gamma);
            if (OUT_BITS == 0) {
                static_cast<float*>(p.out)[i] = v;
            } else {
                constexpr float maxv = OUT_BITS == 8 ? 255.f : 65535.f;
                // round half to even; out-of-range values saturate as in nb200_chw_f32_to_hwc
                const float q = fminf(fmaxf(rintf(__fmul_rn(v, maxv)), 0.f), maxv);
                const size_t o3 = ((size_t)b * plane + px) * 3 + c;
                if (OUT_BITS == 8) static_cast<uint8_t*>(p.out)[o3] = (uint8_t)q;
                else static_cast<uint16_t*>(p.out)[o3] = (uint16_t)q;
            }
        }
        if (p.buffer) p.buffer[c * plane + px] = buf;
    }
}

template <int OUT_BITS>
void launch_apply(const ApplyParams& p, const NoiseField& f, dim3 grid, cudaStream_t st) {
    if (p.noise) apply_rgb_noise_kernel<OUT_BITS, false><<<grid, kThreads, 0, st>>>(p, f);
    else apply_rgb_noise_kernel<OUT_BITS, true><<<grid, kThreads, 0, st>>>(p, f);
}

int make_field(uint64_t seed, int level, int H, int W, NoiseField* f) {
    NB_CHECK(level == 1 || level == 2, "level must be 1 or 2");
    // the reference's level 2 draws an (H // 2) x (W // 2) field and cannot upsample an empty one
    NB_CHECK(level == 1 || (H >= 2 && W >= 2), "level 2 needs H >= 2 and W >= 2");
    f->key = make_uint2((uint32_t)seed, (uint32_t)(seed >> 32));
    f->level = level;
    f->W = W;
    f->hh = H / 2;
    f->hw = W / 2;
    f->sy = (float)f->hh / (float)H;
    f->sx = (float)f->hw / (float)W;
    return 0;
}

}  // namespace

}  // namespace nb200

using namespace nb200;

extern "C" int nb200_rgb_noise(uint64_t seed, uint32_t offset, int level, int B, int C, int H, int W, float* out, void* stream) {
    NB_CHECK(out, "null pointer");
    NB_CHECK(B > 0 && C > 0 && H > 0 && W > 0 && H <= 65535, "bad shape");
    NB_CHECK((int64_t)H * W <= INT32_MAX, "frame too large");
    NoiseField f;
    if (make_field(seed, level, H, W, &f)) return 1;
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope ps(st, PC_OTHER, (double)B * C * H * W * 4);
    rgb_noise_kernel<<<dim3(cdiv(W, kThreads), H), kThreads, 0, st>>>(f, offset, B, C, H, out);
    NB_LAUNCHED();
    return 0;
}

extern "C" int nb200_apply_rgb_noise(const float* rgb, int B, int C, int H, int W, const float* noise, uint64_t seed,
                                     uint32_t offset, int level, float* buffer, int buffer_reset, const double* params_host,
                                     int light_decay, int out_bits, void* out, void* stream) {
    NB_CHECK(rgb && out && params_host, "null pointer");
    NB_CHECK((const void*)rgb != out && (const void*)noise != out && (const void*)buffer != out, "out must not alias an input");
    NB_CHECK(B > 0 && C > 0 && H > 0 && W > 0 && H <= 65535, "bad shape");
    NB_CHECK((int64_t)H * W <= INT32_MAX, "frame too large");
    NB_CHECK(out_bits == 0 || out_bits == 8 || out_bits == 16, "out_bits must be 0 (float), 8 or 16");
    NB_CHECK(out_bits == 0 || C == 3, "uint8 / uint16 output needs 3 channels");
    const double strength = params_host[0], gamma = params_host[1], lds = params_host[2], speed = params_host[3];
    NB_CHECK(gamma > 0, "gamma must be positive");
    NB_CHECK(lds >= 0 && lds <= 1, "light_decay_strength must be in [0, 1]");   // rgb_noise.py:23
    NoiseField f{};
    if (noise) {
        f.W = W;               // the field is only read for its width
    } else if (make_field(seed, level, H, W, &f)) {
        return 1;
    }
    ApplyParams p;
    p.rgb = rgb; p.noise = noise; p.buffer = buffer; p.out = out;
    p.B = B; p.C = C; p.H = H; p.reset = buffer_reset != 0; p.offset = offset;
    p.strength = (float)strength;
    p.gamma = (float)gamma;
    p.inv_gamma = (float)(1.0 / gamma);
    p.lds = (float)lds;
    p.one_minus_lds = (float)(1.0 - lds);
    p.speed = (float)speed;
    p.one_minus_speed = (float)(1.0 - speed);
    p.pow_gamma = pow_kind(gamma);
    p.pow_inv_gamma = pow_kind(1.0 / gamma);
    p.light_decay = light_decay != 0;
    const double px = (double)B * C * H * W;
    cudaStream_t st = (cudaStream_t)stream;
    ProfScope ps(st, PC_OTHER, px * (4 + (noise ? 4 : 0) + (out_bits ? out_bits / 8 : 4)) + (buffer ? 8.0 * C * H * W : 0.0));
    const dim3 grid(cdiv(W, kThreads), H);
    if (out_bits == 0) launch_apply<0>(p, f, grid, st);
    else if (out_bits == 8) launch_apply<8>(p, f, grid, st);
    else launch_apply<16>(p, f, grid, st);
    NB_LAUNCHED();
    return 0;
}
