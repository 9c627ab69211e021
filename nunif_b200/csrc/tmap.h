// Tensor-map (TMA descriptor) construction shared by the TMA kernels (gemm.cu).
#pragma once
#include "common.cuh"
#include <cuda.h>

namespace nb200 {
// fp16 tiled tensor map; dims/strides innermost first, strides_bytes has rank-1 entries; swizzle_bytes in {128, 64, 32}
int encode(CUtensorMap* m, const void* base, int rank, const cuuint64_t* dims, const cuuint64_t* strides_bytes,
           const cuuint32_t* box, int swizzle_bytes);
}  // namespace nb200
