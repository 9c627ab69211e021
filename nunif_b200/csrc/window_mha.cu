// Kernels of the window-attention block WABlock that sbs.row_flow_v3, sbs.mlbw and iw3.depth_aa are built from
// (iw3/models/row_flow_v3.py:13-29, mlbw.py:18-34, depth_aa.py:11-26): the WindowMHA2d core between its qkv and head_proj
// Linears, and the replication pad of conv_mlp.  Everything else of the block runs on the wgmma GEMM (wa_block.cu).
#include "window_mha.h"

namespace nb200 {

namespace {

// One thread per (window, head, query), WPB windows per CTA; K and V of each window are staged in shared memory.  Window
// (wy, wx) starts at token (wy * WS - pad_y, wx * WS - pad_x): tokens outside the grid belong to the zero padding.
template <int WS, int HD, int HEADS>
__global__ void __launch_bounds__(128) window_mha_kernel(const __half* __restrict__ qkv, const float* __restrict__ qkv_bias,
                                                          const float* __restrict__ bias, __half* __restrict__ out, int H, int W,
                                                          int pad_y, int pad_x, int nwx, int nwy, long long nwin) {
    constexpr int N = WS * WS, C = HD * HEADS, TPW = N * HEADS, WPB = 128 / TPW, VPT = C / 8;   // VPT: 16-byte vectors per token
    static_assert(HD == 16 || HD == 32, "head dim 16 or 32");
    constexpr float scale = HD == 16 ? 0.25f : 0.17677669529663687f;                              // 1/sqrt(HD)
    __shared__ __align__(16) __half sK[WPB][N][C];
    __shared__ __align__(16) __half sV[WPB][N][C];
    __shared__ float sBias[N * N];
    if (threadIdx.x == 0) NB_PDL_TRIGGER();
    for (int i = threadIdx.x; i < N * N; i += blockDim.x) sBias[i] = bias[i];
    const int wl = threadIdx.x / TPW, r = threadIdx.x % TPW;
    const long long win = (long long)blockIdx.x * WPB + wl;
    const bool active = wl < WPB && win < nwin;
    int y0 = 0, x0 = 0, b = 0;
    if (active) {
        const int wx = (int)(win % nwx), wy = (int)((win / nwx) % nwy);
        b = (int)(win / ((long long)nwx * nwy));
        y0 = wy * WS - pad_y;
        x0 = wx * WS - pad_x;
        for (int i = r; i < N * 2 * VPT; i += TPW) {
            const int j = i / (2 * VPT), v = i % (2 * VPT);
            const int y = y0 + j / WS, x = x0 + j % WS;
            uint4 val;
            if (y >= 0 && y < H && x >= 0 && x < W) {
                val = __ldg(reinterpret_cast<const uint4*>(qkv + (((size_t)b * H + y) * W + x) * (3 * C) + C) + v);
            } else {                                                   // a token of the zero padding: k | v = projection bias
                __align__(16) __half2 h[4];
#pragma unroll
                for (int k = 0; k < 4; ++k) h[k] = __floats2half2_rn(qkv_bias[C + v * 8 + 2 * k], qkv_bias[C + v * 8 + 2 * k + 1]);
                val = *reinterpret_cast<const uint4*>(h);
            }
            if (v < VPT) *reinterpret_cast<uint4*>(&sK[wl][j][v * 8]) = val;
            else *reinterpret_cast<uint4*>(&sV[wl][j][(v - VPT) * 8]) = val;
        }
    }
    __syncthreads();
    if (!active) return;
    const int head = r / N, qi = r % N;
    const int qy = y0 + qi / WS, qx = x0 + qi % WS;
    if (qy < 0 || qy >= H || qx < 0 || qx >= W) return;                // cropped away after the attention (attention.py:158-160)
    const size_t tokq = ((size_t)b * H + qy) * W + qx;
    float q[HD];
    {
        const uint4* qp = reinterpret_cast<const uint4*>(qkv + tokq * (3 * C) + head * HD);
#pragma unroll
        for (int v = 0; v < HD / 8; ++v) {
            const uint4 raw = __ldg(qp + v);
            const __half2* hh = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
            for (int k = 0; k < 4; ++k) {
                const float2 f = __half22float2(hh[k]);
                q[v * 8 + 2 * k] = f.x;
                q[v * 8 + 2 * k + 1] = f.y;
            }
        }
    }
    float s[N], mx = -1e30f;
#pragma unroll
    for (int j = 0; j < N; ++j) {
        const __half2* kp = reinterpret_cast<const __half2*>(&sK[wl][j][head * HD]);
        float acc = 0.f;
#pragma unroll
        for (int k = 0; k < HD / 2; ++k) {
            const float2 f = __half22float2(kp[k]);
            acc = fmaf(q[2 * k], f.x, acc);
            acc = fmaf(q[2 * k + 1], f.y, acc);
        }
        s[j] = acc * scale + sBias[qi * N + j];                         // attn_mask is additive (F.scaled_dot_product_attention)
        mx = fmaxf(mx, s[j]);
    }
    float sum = 0.f;
#pragma unroll
    for (int j = 0; j < N; ++j) { s[j] = __expf(s[j] - mx); sum += s[j]; }
    const float inv = 1.f / sum;
    float o[HD];
#pragma unroll
    for (int k = 0; k < HD; ++k) o[k] = 0.f;
#pragma unroll
    for (int j = 0; j < N; ++j) {
        const __half2* vp = reinterpret_cast<const __half2*>(&sV[wl][j][head * HD]);
        const float pj = s[j] * inv;
#pragma unroll
        for (int k = 0; k < HD / 2; ++k) {
            const float2 f = __half22float2(vp[k]);
            o[2 * k] = fmaf(pj, f.x, o[2 * k]);
            o[2 * k + 1] = fmaf(pj, f.y, o[2 * k + 1]);
        }
    }
    __half* op = out + tokq * C + head * HD;
#pragma unroll
    for (int v = 0; v < HD / 8; ++v) {
        __align__(16) __half2 hv[4];
#pragma unroll
        for (int k = 0; k < 4; ++k) hv[k] = __floats2half2_rn(o[v * 8 + 2 * k], o[v * 8 + 2 * k + 1]);
        *reinterpret_cast<uint4*>(op + v * 8) = *reinterpret_cast<const uint4*>(hv);
    }
}

template <int WS, int HD, int HEADS>
int launch_window_mha(cudaStream_t st, const __half* qkv, const float* qkv_bias, const float* bias, __half* out, int H, int W, int pad_y,
                      int pad_x, int nwx, int nwy, long long nwin) {
    constexpr int WPB = 128 / (WS * WS * HEADS);
    window_mha_kernel<WS, HD, HEADS><<<(unsigned)cdiv64(nwin, WPB), 128, 0, st>>>(qkv, qkv_bias, bias, out, H, W, pad_y, pad_x, nwx, nwy, nwin);
    NB_LAUNCHED();
    return 0;
}

__global__ void __launch_bounds__(256) reppad1_kernel(const uint4* __restrict__ x, uint4* __restrict__ out, int B, int H, int W, int V) {
    if (threadIdx.x == 0) NB_PDL_TRIGGER();
    const long long total = (long long)B * (H + 2) * (W + 2) * V;
    const long long i = (long long)blockIdx.x * blockDim.x + threadIdx.x;
    if (i >= total) return;
    const int v = (int)(i % V);
    long long t = i / V;
    const int X = (int)(t % (W + 2));
    t /= W + 2;
    const int Y = (int)(t % (H + 2)), b = (int)(t / (H + 2));
    const int sy = min(max(Y - 1, 0), H - 1), sx = min(max(X - 1, 0), W - 1);
    out[i] = __ldg(x + (((size_t)b * H + sy) * W + sx) * V + v);
}

}  // namespace

int window_mha(cudaStream_t st, const __half* qkv, const float* qkv_bias, const float* bias, __half* out, int B, int H, int W, int C,
               int ws, int heads, int pad_y, int pad_x) {
    if (rec_on(REC_AUX))
        rec_launch("wmha", {{"B", B}, {"H", H}, {"W", W}, {"C", C}, {"ws", ws}, {"heads", heads}, {"pad_y", pad_y},
                            {"pad_x", pad_x}});
    NB_CHECK(H % ws == 0 && W % ws == 0, "token grid must be a multiple of the window");
    // a shifted direction pads ws / 2 on both sides; the padded grid must still tile into whole windows (not so for odd ws)
    NB_CHECK((pad_y == 0 || pad_y == ws / 2) && (pad_x == 0 || pad_x == ws / 2), "padding must be 0 or ws / 2");
    NB_CHECK((H + 2 * pad_y) % ws == 0 && (W + 2 * pad_x) % ws == 0, "padded token grid must be a multiple of the window");
    NB_CHECK(qkv_bias || (pad_y == 0 && pad_x == 0), "padding needs the qkv bias");
    NB_CHECK(C % heads == 0, "channels must split evenly into heads");
    const int nwx = (W + 2 * pad_x) / ws, nwy = (H + 2 * pad_y) / ws, hd = C / heads;
    const long long nwin = (long long)B * nwx * nwy;
    if (ws == 3 && hd == 32 && heads == 2) return launch_window_mha<3, 32, 2>(st, qkv, qkv_bias, bias, out, H, W, pad_y, pad_x, nwx, nwy, nwin);
    if (ws == 4 && hd == 32 && heads == 2) return launch_window_mha<4, 32, 2>(st, qkv, qkv_bias, bias, out, H, W, pad_y, pad_x, nwx, nwy, nwin);
    if (ws == 4 && hd == 32 && heads == 4) return launch_window_mha<4, 32, 4>(st, qkv, qkv_bias, bias, out, H, W, pad_y, pad_x, nwx, nwy, nwin);
    if (ws == 8 && hd == 16 && heads == 2) return launch_window_mha<8, 16, 2>(st, qkv, qkv_bias, bias, out, H, W, pad_y, pad_x, nwx, nwy, nwin);
    return fail("window_mha: no kernel for " + std::to_string(ws) + "x" + std::to_string(ws) + " windows with " + std::to_string(heads) +
                " heads of " + std::to_string(hd));
}

int reppad1(cudaStream_t st, const __half* x, int B, int H, int W, int C, __half* out) {
    if (rec_on(REC_AUX)) rec_launch("reppad", {{"B", B}, {"H", H}, {"W", W}, {"C", C}});
    NB_CHECK(C % 8 == 0, "channels must be a multiple of 8");
    const long long total = (long long)B * (H + 2) * (W + 2) * (C / 8);
    reppad1_kernel<<<(unsigned)cdiv64(total, 256), 256, 0, st>>>(reinterpret_cast<const uint4*>(x), reinterpret_cast<uint4*>(out), B, H, W, C / 8);
    NB_LAUNCHED();
    return 0;
}

}  // namespace nb200

// Test entry points of the WABlock kernels (include/nunif_b200.h)
extern "C" int nb200_window_mha_f16(const void* qkv, const float* qkv_bias, const float* bias, void* out, int B, int H, int W, int C,
                                    int ws, int heads, int pad_y, int pad_x, void* stream) {
    NB_CHECK(qkv && bias && out && B > 0 && H > 0 && W > 0 && C > 0 && ws > 0 && heads > 0, "bad arguments");
    return nb200::window_mha((cudaStream_t)stream, (const __half*)qkv, qkv_bias, bias, (__half*)out, B, H, W, C, ws, heads, pad_y, pad_x);
}

extern "C" int nb200_reppad1_f16(const void* x, int B, int H, int W, int C, void* out, void* stream) {
    NB_CHECK(x && out && B > 0 && H > 0 && W > 0 && C > 0, "bad arguments");
    return nb200::reppad1((cudaStream_t)stream, (const __half*)x, B, H, W, C, (__half*)out);
}
