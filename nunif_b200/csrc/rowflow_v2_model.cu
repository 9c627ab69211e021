// sbs.row_flow_v2 container (iw3/models/row_flow_v2.py:10-37; state_dict keys `feature.0.*`, `non_overlap.*`,
// `overlap_residual.{0,2,4,6}.*`, buffer `delta_scale`): the whole network is one kernel (rowflow_v2.cu), whose weights are
// one parameter block in the layout rowflow_kernels.h describes.
#include "model.h"
#include "rowflow_kernels.h"

namespace nb200 {

struct NB_HIDDEN Rf2W : NetW {
    size_t params = 0;
};

// B fragments of mma.sync m16n8k16 (.col) for a conv weight [cout][cin][kh][kw] as the implicit GEMM
// k = (ky * kw + kx) * cin + ci, n = co (n >= cout zero): lane (g = lane / 4, t = lane % 4) of k-step ks, n8 tile nt holds
// {B[ks*16 + 2t][n], B[ks*16 + 2t + 1][n]} and {B[ks*16 + 2t + 8][n], B[ks*16 + 2t + 9][n]} with n = nt * 8 + g.
static void rf2_pack_frag(const float* w, int cout, int cin, int kh, int kw, int ntiles, __half* out) {
    const int K = kh * kw * cin, ksteps = K / 16;
    auto B = [&](int k, int n) -> float {
        if (n >= cout) return 0.f;
        const int tap = k / cin, ci = k % cin;
        return w[(((size_t)n * cin + ci) * kh + tap / kw) * kw + tap % kw];
    };
    for (int ks = 0; ks < ksteps; ++ks)
        for (int nt = 0; nt < ntiles; ++nt)
            for (int lane = 0; lane < 32; ++lane) {
                const int g = lane >> 2, t = lane & 3, n = nt * 8 + g, k = ks * 16 + 2 * t;
                __half* o = out + (((size_t)ks * ntiles + nt) * 32 + lane) * 4;
                o[0] = __float2half_rn(B(k, n));
                o[1] = __float2half_rn(B(k + 1, n));
                o[2] = __float2half_rn(B(k + 8, n));
                o[3] = __float2half_rn(B(k + 9, n));
            }
}

std::unique_ptr<NetW> pack_row_flow_v2(Packer& pk) {
    auto r = std::make_unique<Rf2W>();
    const float* fw = pk.get("feature.0.weight", 16 * 3 * 3);                  // Conv2d(3, 16, (1, 3))
    const float* fb = pk.get("feature.0.bias", 16);
    const float* hw = pk.get("non_overlap.weight", 16);                        // Conv2d(16, 1, 1)
    const float* hb = pk.get("non_overlap.bias", 1);
    const float* w1 = pk.get("overlap_residual.0.weight", 16 * 16 * 9);        // Conv2d(16, 16, (1, 9))
    const float* b1 = pk.get("overlap_residual.0.bias", 16);
    const float* w2 = pk.get("overlap_residual.2.weight", 32 * 16 * 9);        // Conv2d(16, 32, (1, 9))
    const float* b2 = pk.get("overlap_residual.2.bias", 32);
    const float* w3 = pk.get("overlap_residual.4.weight", 32 * 32 * 9);        // Conv2d(32, 32, (1, 9))
    const float* b3 = pk.get("overlap_residual.4.bias", 32);
    const float* w4 = pk.get("overlap_residual.6.weight", 32 * 9);             // Conv2d(32, 1, 3)
    const float* b4 = pk.get("overlap_residual.6.bias", 1);
    pk.mark("delta_scale");   // the driver computes 1 / (W // 2 - 1) itself (backward_warp.py:201)
    if (!fw || !fb || !hw || !hb || !w1 || !b1 || !w2 || !b2 || !w3 || !b3 || !w4 || !b4) return r;
    r->params = pk.reserve(RF2_PARAM_BYTES);
    uint8_t* p = pk.blob.data() + r->params;
    rf2_pack_frag(w1, 16, 16, 1, 9, 2, reinterpret_cast<__half*>(p + RF2_FRAG1));
    rf2_pack_frag(w2, 32, 16, 1, 9, 4, reinterpret_cast<__half*>(p + RF2_FRAG2));
    rf2_pack_frag(w3, 32, 32, 1, 9, 4, reinterpret_cast<__half*>(p + RF2_FRAG3));
    rf2_pack_frag(w4, 1, 32, 3, 3, 1, reinterpret_cast<__half*>(p + RF2_FRAG4));
    // autocast runs every conv with fp16 weights and biases: the scalar ones are stored fp16-rounded
    float* f = reinterpret_cast<float*>(p + RF2_F32);
    for (int i = 0; i < 144; ++i) f[RF2_FW + i] = round_f16(fw[i]);
    for (int i = 0; i < 16; ++i) f[RF2_FB + i] = round_f16(fb[i]);
    for (int i = 0; i < 16; ++i) f[RF2_HW + i] = round_f16(hw[i]);
    for (int i = 0; i < 16; ++i) f[RF2_B1 + i] = round_f16(b1[i]);
    for (int i = 0; i < 32; ++i) f[RF2_B2 + i] = round_f16(b2[i]);
    for (int i = 0; i < 32; ++i) f[RF2_B3 + i] = round_f16(b3[i]);
    f[RF2_HB] = round_f16(hb[0]);
    f[RF2_B4] = round_f16(b4[0]);
    return r;
}

}  // namespace nb200

using namespace nb200;

// RowFlowV2.forward with delta_output=True (iw3/models/row_flow_v2.py:80-86) - the x component of the returned delta
extern "C" int nb200_row_flow_v2_delta(nb200_model* m, const float* x, int B, int h, int w, float* delta, void* stream) {
    NB_CHECK(m && x && delta, "null pointer");
    const Rf2W* r = net_as<Rf2W>(m);
    NB_CHECK(r, "model is not sbs.row_flow_v2");
    NB_CHECK(B > 0 && h > 0 && w > 0, "bad shape");
    return rf2_forward((cudaStream_t)stream, m->blob + r->params, x, B, h, w, delta);
}
