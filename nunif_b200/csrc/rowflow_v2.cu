// `sbs.row_flow_v2` delta network (iw3/models/row_flow_v2.py:10-86, _forward_delta_only) in one fused kernel.
//
// The 28-pixel pre_pad, the inner ReplicationPad2d's and the final crop of _forward_delta_only equal "valid" convolutions
// over the input extended by clamp-to-edge indexing, 14 columns left / right and 1 row above / below: the receptive field is
// +-14 columns and +-1 row, so no inner pad is reached inside the cropped region.  Intermediate columns outside the image are
// computed from the clamped input (they are not replicas of edge activations).  Everything before the final 3x3 conv works
// on one row, so row -1 equals row 0 and the 3x3 sees a replicate pad of layer 4.
//
// One CTA = a strip of RF2_ROWS output rows x RF2_T output columns of one image.  It walks the strip's rows (plus one above
// and one below), and for each row computes, in shared memory as fp16 [column][channel]:
//   feature  1x3 conv 3 -> 16 + ReLU        136 columns (CUDA cores)
//   conv #1  1x9 conv 16 -> 16 + ReLU       128 columns (mma.sync m16n8k16, K = 9 * 16)
//   conv #2  1x9 conv 16 -> 32 + ReLU       128 columns (K = 9 * 16)
//   conv #3  1x9 conv 32 -> 32 + ReLU       128 columns (K = 9 * 32), kept for three rows
// and, one row behind, the 3x3 conv 32 -> 1 (mma, N = 8 with one live column, K = 9 * 32) plus the 1x1 head 16 -> 1 and the
// fp16 add non_overlap + overlap_residual.  Every mma layer computes 8 m16 tiles (128 columns); the columns that only see
// clamped input shrink layer by layer: feature 136, conv #1 128, conv #2 120, conv #3 112, 3x3 110 = RF2_T, the columns the
// CTA stores.  4 warps, each owns m tiles w and w + 4.  Only x and delta touch HBM.
//
// Numerics follow the reference under CUDA autocast: x and the weights are fp16, every conv accumulates in fp32 and its output
// is rounded to fp16, then the fp16 bias is added and the sum rounded again (ATen's cuDNN path adds the bias with a separate
// fp16 add), ReLU on fp16, and non_overlap + overlap_residual is an fp16 add.
#include "common.cuh"
#include "rowflow_kernels.h"

namespace nb200 {

namespace {

constexpr int NC = 128;          // computed columns per layer (8 m16 tiles)
constexpr int BW = 136;          // buffer columns: a 1x9 conv over NC columns reads NC + 8
constexpr int S16 = 24;          // pixel stride (halves) of the 16-channel buffers: 48 B rows make ldmatrix conflict-free
constexpr int S32 = 40;          // pixel stride of the 32-channel buffers (80 B)
constexpr int THREADS = 128;

// smem layout (bytes)
constexpr int OFF_BUFF = RF2_PARAM_BYTES;
constexpr int OFF_BUF1 = OFF_BUFF + BW * S16 * 2;
constexpr int OFF_BUF2 = OFF_BUF1 + BW * S16 * 2;
constexpr int OFF_C3 = OFF_BUF2 + BW * S32 * 2;
constexpr int OFF_NOV = OFF_C3 + 3 * BW * S32 * 2;
constexpr int SMEM_BYTES = OFF_NOV + 3 * NC * 4;
static_assert(RF2_PARAM_BYTES % 16 == 0 && OFF_C3 % 16 == 0 && OFF_NOV % 16 == 0, "16-byte aligned smem regions");

__device__ __forceinline__ float r16(float v) { return __half2float(__float2half_rn(v)); }

__device__ __forceinline__ void ldsm_x4(uint32_t (&a)[4], const __half* p) {
    const uint32_t s = (uint32_t)__cvta_generic_to_shared(p);
    asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0,%1,%2,%3}, [%4];\n"
                 : "=r"(a[0]), "=r"(a[1]), "=r"(a[2]), "=r"(a[3]) : "r"(s));
}

__device__ __forceinline__ void mma16816(float (&c)[4], const uint32_t (&a)[4], uint2 b) {
    asm volatile("mma.sync.aligned.m16n8k16.row.col.f32.f16.f16.f32 {%0,%1,%2,%3}, {%4,%5,%6,%7}, {%8,%9}, {%0,%1,%2,%3};\n"
                 : "+f"(c[0]), "+f"(c[1]), "+f"(c[2]), "+f"(c[3])
                 : "r"(a[0]), "r"(a[1]), "r"(a[2]), "r"(a[3]), "r"(b.x), "r"(b.y));
}

// One warp, two m16 tiles (columns m0 .. m0 + 15 and m0 + 64 .. m0 + 79): acc[mt][nt] += sum over the k-steps of
// A[col][k] * B[k][n], k-step ks = (row * TAPS + tap) * CIN/16 + chunk reading channels chunk*16 .. +15 of column col + tap of
// src[row].  The weights are B fragments in lane order, [ks][nt][lane] (rf2 packing in rowflow_v2_model.inl).
template <int CIN, int NT, int TAPS, int ROWS>
__device__ __forceinline__ void conv_mma(float (&acc)[2][NT][4], const __half* const (&src)[ROWS], int stride, int m0,
                                         const uint2* __restrict__ frag, int lane) {
    const int prow = m0 + (lane & 15), koff = (lane >> 4) * 8;
#pragma unroll
    for (int ry = 0; ry < ROWS; ++ry)
#pragma unroll
        for (int tap = 0; tap < TAPS; ++tap)
#pragma unroll
            for (int ch = 0; ch < CIN / 16; ++ch) {
                const int ks = (ry * TAPS + tap) * (CIN / 16) + ch;
                uint32_t a0[4], a1[4];
                ldsm_x4(a0, src[ry] + (prow + tap) * stride + ch * 16 + koff);
                ldsm_x4(a1, src[ry] + (prow + 64 + tap) * stride + ch * 16 + koff);
#pragma unroll
                for (int nt = 0; nt < NT; ++nt) {
                    const uint2 b = frag[(ks * NT + nt) * 32 + lane];
                    mma16816(acc[0][nt], a0, b);
                    mma16816(acc[1][nt], a1, b);
                }
            }
}

// conv output -> fp16, + fp16 bias -> fp16, ReLU; stored at [col][n] of dst
template <int NT>
__device__ __forceinline__ void store_relu(const float (&acc)[2][NT][4], const float* __restrict__ bias, __half* dst, int stride,
                                           int m0, int lane) {
    const int g = lane >> 2, t4 = lane & 3;
#pragma unroll
    for (int mt = 0; mt < 2; ++mt)
#pragma unroll
        for (int nt = 0; nt < NT; ++nt) {
            const int n = nt * 8 + 2 * t4, col = m0 + mt * 64 + g;
            const float b0 = bias[n], b1 = bias[n + 1];
            const float* c = acc[mt][nt];
            *reinterpret_cast<__half2*>(dst + col * stride + n) =
                __floats2half2_rn(fmaxf(r16(c[0]) + b0, 0.f), fmaxf(r16(c[1]) + b1, 0.f));
            *reinterpret_cast<__half2*>(dst + (col + 8) * stride + n) =
                __floats2half2_rn(fmaxf(r16(c[2]) + b0, 0.f), fmaxf(r16(c[3]) + b1, 0.f));
        }
}

template <int MT, int NT>
__device__ __forceinline__ void zero(float (&acc)[MT][NT][4]) {
#pragma unroll
    for (int i = 0; i < MT; ++i)
#pragma unroll
        for (int j = 0; j < NT; ++j)
#pragma unroll
            for (int k = 0; k < 4; ++k) acc[i][j][k] = 0.f;
}

__global__ void __launch_bounds__(THREADS, 2) rf2_kernel(const float* __restrict__ x, float* __restrict__ delta,
                                                         const uint4* __restrict__ params, int h, int w) {
    extern __shared__ __align__(16) unsigned char smem[];
    const int tid = threadIdx.x, lane = tid & 31, warp = tid >> 5;
    const int x0 = blockIdx.x * RF2_T, y0 = blockIdx.y * RF2_ROWS, b = blockIdx.z;
    const int y1 = min(y0 + RF2_ROWS, h);
    {
        uint4* d = reinterpret_cast<uint4*>(smem);
        for (int i = tid; i < RF2_PARAM_BYTES / 16; i += THREADS) d[i] = __ldg(params + i);
        // the columns past NC of each activation buffer are read by the garbage rows of the last m tile only; keep them finite
        for (int i = RF2_PARAM_BYTES / 16 + tid; i < OFF_NOV / 16; i += THREADS) d[i] = make_uint4(0, 0, 0, 0);
    }
    const uint2* frag1 = reinterpret_cast<const uint2*>(smem + RF2_FRAG1);
    const uint2* frag2 = reinterpret_cast<const uint2*>(smem + RF2_FRAG2);
    const uint2* frag3 = reinterpret_cast<const uint2*>(smem + RF2_FRAG3);
    const uint2* frag4 = reinterpret_cast<const uint2*>(smem + RF2_FRAG4);
    const float* fp = reinterpret_cast<const float*>(smem + RF2_F32);
    const float *fw = fp + RF2_FW, *fb = fp + RF2_FB, *hw = fp + RF2_HW, *b1 = fp + RF2_B1, *b2 = fp + RF2_B2, *b3 = fp + RF2_B3;
    __half* bufF = reinterpret_cast<__half*>(smem + OFF_BUFF);
    __half* buf1 = reinterpret_cast<__half*>(smem + OFF_BUF1);
    __half* buf2 = reinterpret_cast<__half*>(smem + OFF_BUF2);
    __half* c3 = reinterpret_cast<__half*>(smem + OFF_C3);
    float* nov = reinterpret_cast<float*>(smem + OFF_NOV);
    __syncthreads();
    const float hb = fp[RF2_HB], b4 = fp[RF2_B4];
    const int m0 = warp * 16;
    const size_t plane = (size_t)h * w;
    const float* xb = x + (size_t)b * 3 * plane;

    // conv #3 rows r = y0 - 1 .. y1; the output row r - 1 follows once rows r - 2 .. r are in c3
    for (int r = y0 - 1; r <= y1; ++r) {
        const int ry = min(max(r, 0), h - 1);
        const int slot = (r - y0 + 1) % 3;
        // feature: buffer column j is image column x0 - 13 + j, reading x0 - 14 + j .. x0 - 12 + j (clamped)
        for (int j = tid; j < BW; j += THREADS) {
            float in[3][3];
#pragma unroll
            for (int k = 0; k < 3; ++k) {
                const int xx = min(max(x0 - 14 + j + k, 0), w - 1);
#pragma unroll
                for (int ci = 0; ci < 3; ++ci) in[ci][k] = r16(__ldg(xb + ci * plane + (size_t)ry * w + xx));
            }
            __align__(16) __half o[16];
#pragma unroll
            for (int oc = 0; oc < 16; ++oc) {
                float acc = 0.f;
#pragma unroll
                for (int ci = 0; ci < 3; ++ci)
#pragma unroll
                    for (int k = 0; k < 3; ++k) acc = fmaf(in[ci][k], fw[(oc * 3 + ci) * 3 + k], acc);
                o[oc] = __float2half_rn(fmaxf(r16(acc) + fb[oc], 0.f));
            }
            uint4* dst = reinterpret_cast<uint4*>(bufF + j * S16);
            dst[0] = reinterpret_cast<const uint4*>(o)[0];
            dst[1] = reinterpret_cast<const uint4*>(o)[1];
        }
        __syncthreads();
        // non_overlap (1x1 head) at the output columns j <-> feature column j + 13; conv #1: column j <-> image x0 - 9 + j
        if (tid < RF2_T) {
            const __half* f = bufF + (tid + 13) * S16;
            float acc = 0.f;
#pragma unroll
            for (int c = 0; c < 16; ++c) acc = fmaf(__half2float(f[c]), hw[c], acc);
            nov[slot * NC + tid] = r16(r16(acc) + hb);
        }
        {
            float acc[2][2][4];
            zero(acc);
            const __half* const src[1] = {bufF};
            conv_mma<16, 2, 9, 1>(acc, src, S16, m0, frag1, lane);
            store_relu<2>(acc, b1, buf1, S16, m0, lane);
        }
        __syncthreads();
        {   // conv #2: column j <-> image x0 - 5 + j
            float acc[2][4][4];
            zero(acc);
            const __half* const src[1] = {buf1};
            conv_mma<16, 4, 9, 1>(acc, src, S16, m0, frag2, lane);
            store_relu<4>(acc, b2, buf2, S32, m0, lane);
        }
        __syncthreads();
        {   // conv #3: column j <-> image x0 - 1 + j
            float acc[2][4][4];
            zero(acc);
            const __half* const src[1] = {buf2};
            conv_mma<32, 4, 9, 1>(acc, src, S32, m0, frag3, lane);
            store_relu<4>(acc, b3, c3 + slot * BW * S32, S32, m0, lane);
        }
        __syncthreads();
        if (r >= y0 + 1) {   // 3x3 conv 32 -> 1 over conv #3 rows r - 2, r - 1, r, + non_overlap of row r - 1
            float acc[2][1][4];
            zero(acc);
            const __half* const src[3] = {c3 + ((r - y0 + 2) % 3) * BW * S32, c3 + ((r - y0) % 3) * BW * S32, c3 + slot * BW * S32};
            conv_mma<32, 1, 3, 3>(acc, src, S32, m0, frag4, lane);
            const int yo = r - 1;
            if ((lane & 3) == 0) {
                const float* nv = nov + ((r - y0) % 3) * NC;
                float* drow = delta + ((size_t)b * h + yo) * w;
#pragma unroll
                for (int mt = 0; mt < 2; ++mt)
#pragma unroll
                    for (int hi = 0; hi < 2; ++hi) {
                        const int j = m0 + mt * 64 + (lane >> 2) + hi * 8;
                        if (j < RF2_T && x0 + j < w) {
                            const float res = r16(r16(acc[mt][0][hi * 2]) + b4);
                            drow[x0 + j] = r16(nv[j] + res);
                        }
                    }
            }
        }
    }
}

}  // namespace

int rf2_forward(cudaStream_t st, const void* params, const float* x, int B, int h, int w, float* delta) {
    NB_CHECK(B <= 65535 && cdiv(h, RF2_ROWS) <= 65535, "batch or height too large for the row_flow_v2 grid");
    if (ensure_dyn_smem((const void*)rf2_kernel, SMEM_BYTES)) return 1;
    // algorithmic HBM traffic: x (3 planes) in, delta out
    ProfScope ps(st, PC_OTHER, (double)B * h * w * 16);
    dim3 grid(cdiv(w, RF2_T), cdiv(h, RF2_ROWS), B);
    rf2_kernel<<<grid, THREADS, SMEM_BYTES, st>>>(x, delta, reinterpret_cast<const uint4*>(params), h, w);
    NB_LAUNCHED();
    return 0;
}

}  // namespace nb200
