// Disparity mapper of iw3/mapper.py on the device: one evaluator of the nb200_mapper descriptor
// (include/nunif_b200.h), shared by the per-frame min/max pass (dilation.cu) and the EMA normaliser
// and standalone mapper (ema_scaler.cu).  The host parses the name and rounds every constant to fp32
// the way the reference does; here each function runs in fp32 in the reference's op order.
// __fmul_rn / __fadd_rn keep nvcc from contracting a multiply and an add into an FMA that torch does
// not do.
#pragma once
#include "common.cuh"
#include "../../include/nunif_b200.h"

namespace nb200 {

static_assert(sizeof(nb200_mapper) == 528, "nb200_mapper is a fixed-size ABI struct");

enum MapperKind { MK_NONE = 0, MK_POW2, MK_SOFTPLUS, MK_SOFTPLUS2, MK_SOFTPLUS01, MK_INV_SOFTPLUS01, MK_DIV, MK_SHIFT, MK_COUNT };

// resolve_mapper_function (iw3/mapper.py:64-120)
__device__ __forceinline__ float mapper_fn(const nb200_mapper_fn& f, float x) {
    switch (f.kind) {
    case MK_POW2:
        return __fmul_rn(x, x);
    case MK_SOFTPLUS:
    case MK_SOFTPLUS2: {  // :7-11, c = 6: log(1 + exp(x * 12 - 6)) / 6
        float v = logf(1.f + expf(__fmul_rn(x, 12.f) - 6.f)) / 6.f;
        v = (v - f.k[0]) / f.k[1];
        return f.kind == MK_SOFTPLUS2 ? __fmul_rn(v, v) : v;
    }
    case MK_SOFTPLUS01: {  // :14-19 (torch.log(1. + torch.exp(...)), not log1p)
        const float v = logf(1.f + expf(__fmul_rn(x - f.k[0], f.k[1])));
        return (v - f.k[2]) / f.k[3];
    }
    case MK_INV_SOFTPLUS01: {  // :22-26; clamp(min=1e-6) lets a NaN through, like torch.clamp
        float e = expm1f(__fmul_rn(x - f.k[0], f.k[1]));
        e = e < 1e-6f ? 1e-6f : e;
        return (logf(e) - f.k[2]) / f.k[3];
    }
    case MK_DIV:  // :29-32, the expression nb200_minmax_map has always computed
        return ((f.k[0] / (f.k[1] - x)) - f.k[2]) / f.k[3];
    case MK_SHIFT: {  // :39-61: distance = 1 / (A + B * x); (1 - min_distance) + distance; 1 / distance; rescale
        const float distance = f.k[2] + 1.f / __fadd_rn(f.k[0], __fmul_rn(f.k[1], x));
        return (1.f / distance - f.k[3]) / f.k[4];
    }
    default:
        return x;
    }
}

// get_mapper (:129-151): the chain of stages, each one function or the blend a(x) * (1 - w) + b(x) * w
__device__ __forceinline__ float mapper_eval(const nb200_mapper& m, float x) {
    for (int s = 0; s < m.n_stages; ++s) {
        const nb200_mapper_stage& st = m.stage[s];
        const float a = mapper_fn(st.a, x);
        x = st.blend ? __fadd_rn(__fmul_rn(a, st.one_minus_w), __fmul_rn(mapper_fn(st.b, x), st.w)) : a;
    }
    return x;
}

// the descriptor of the float mapper_c entries: mapper_c < 0 -> "none", else distance_to_disparity(x, mapper_c)
// with the constants derived in double from mapper_c, as those entries always have
inline nb200_mapper mapper_from_c(float mapper_c) {
    nb200_mapper m = {};
    if (mapper_c >= 0.f) {
        const double c = (double)mapper_c, c1 = 1.0 + c, min_v = c / c1;
        nb200_mapper_fn& f = m.stage[0].a;
        f.kind = MK_DIV;
        f.k[0] = (float)c; f.k[1] = (float)c1; f.k[2] = (float)min_v; f.k[3] = (float)(1.0 - min_v);
        m.n_stages = 1;
    }
    return m;
}

// empty string if the descriptor can be evaluated, else what is wrong with it
inline const char* mapper_invalid(const nb200_mapper& m) {
    if (m.n_stages < 0 || m.n_stages > NB200_MAPPER_MAX_STAGES) return "n_stages must be in [0, NB200_MAPPER_MAX_STAGES]";
    for (int s = 0; s < m.n_stages; ++s) {
        const nb200_mapper_stage& st = m.stage[s];
        if (st.a.kind < 0 || st.a.kind >= MK_COUNT || (st.blend && (st.b.kind < 0 || st.b.kind >= MK_COUNT))) return "unknown mapper function kind";
    }
    return "";
}

}  // namespace nb200
