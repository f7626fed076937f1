// k2_lora.cu -- merging a low-rank (LoRA) weight delta into a packed fp16 weight matrix:
//   out[n, k] = fp16_rn( float(base[n, k]) + scale * sum_j up[n, j] * down[j, k] )
// Run once per adapter load, never per denoising step (declared in include/k2b200.h).
#include "../../include/k2b200.h"
#include "k2_common.cuh"
#include "k2_internal.h"

namespace k2 {
namespace {

constexpr int LM_TC = 64;   // output columns per CTA: 8 column groups of 8 (one 16-byte fp16 vector each)
constexpr int LM_TR = 64;   // output rows per CTA: 32 row lanes x 2
constexpr int LM_RK = 16;   // slice of the rank staged in shared memory per pass

// One thread owns 2 rows x 8 columns of the output tile.  Every output element is summed by one thread over j = 0, 1, ...,
// rank-1 in that order (slices are consumed in ascending order, and the zero padding of the last slice adds exact zeros), so
// the result does not depend on the grid.  base and out may alias (in-place merge): each element is read before it is written
// by the same thread, so neither pointer is __restrict__.
__global__ void __launch_bounds__(256) lora_merge_kernel(const __half* base, int ldb, const float* __restrict__ up,
                                                         const float* __restrict__ down, int rows, int cols, int rank,
                                                         float scale, __half* out, int ldo, int vec) {
  __shared__ float su[LM_TR][LM_RK + 1];  // +1: the 4 row lanes of a warp read 4 different rows of one column
  __shared__ __align__(16) float sd[LM_RK][LM_TC];
  const int tx = threadIdx.x & 7, ty = threadIdx.x >> 3;
  const int r0 = blockIdx.y * LM_TR, c0 = blockIdx.x * LM_TC;
  float acc[2][8];
#pragma unroll
  for (int i = 0; i < 2; ++i)
#pragma unroll
    for (int e = 0; e < 8; ++e) acc[i][e] = 0.f;
  for (int j0 = 0; j0 < rank; j0 += LM_RK) {
    __syncthreads();
    for (int i = threadIdx.x; i < LM_TR * LM_RK; i += blockDim.x) {
      const int r = i / LM_RK, j = i - r * LM_RK;
      su[r][j] = (r0 + r < rows && j0 + j < rank) ? up[static_cast<long long>(r0 + r) * rank + j0 + j] : 0.f;
    }
    for (int i = threadIdx.x; i < LM_RK * LM_TC; i += blockDim.x) {
      const int j = i / LM_TC, c = i - j * LM_TC;
      sd[j][c] = (j0 + j < rank && c0 + c < cols) ? down[static_cast<long long>(j0 + j) * cols + c0 + c] : 0.f;
    }
    __syncthreads();
#pragma unroll
    for (int j = 0; j < LM_RK; ++j) {
      const float4 da = *reinterpret_cast<const float4*>(&sd[j][tx * 8]);
      const float4 db = *reinterpret_cast<const float4*>(&sd[j][tx * 8 + 4]);
      const float d[8] = {da.x, da.y, da.z, da.w, db.x, db.y, db.z, db.w};
#pragma unroll
      for (int i = 0; i < 2; ++i) {
        const float u = su[ty + 32 * i][j];
#pragma unroll
        for (int e = 0; e < 8; ++e) acc[i][e] = fmaf(u, d[e], acc[i][e]);
      }
    }
  }
  const int c = c0 + tx * 8;
#pragma unroll
  for (int i = 0; i < 2; ++i) {
    const int r = r0 + ty + 32 * i;
    if (r >= rows || c >= cols) continue;
    const __half* br = base + static_cast<long long>(r) * ldb;
    __half* orow = out + static_cast<long long>(r) * ldo;
    // an exactly zero delta leaves the stored bits alone (this keeps a -0 weight -0, so scale 0 is the identity)
    auto merge = [&](__half b, float a) {
      const float dlt = scale * a;
      return dlt != 0.f ? __float2half_rn(__half2float(b) + dlt) : b;
    };
    if (vec && c + 8 <= cols) {
      uint4 raw = *reinterpret_cast<const uint4*>(br + c);
      __half* h = reinterpret_cast<__half*>(&raw);
#pragma unroll
      for (int e = 0; e < 8; ++e) h[e] = merge(h[e], acc[i][e]);
      *reinterpret_cast<uint4*>(orow + c) = raw;
    } else {
#pragma unroll
      for (int e = 0; e < 8; ++e)
        if (c + e < cols) orow[c + e] = merge(br[c + e], acc[i][e]);
    }
  }
}

}  // namespace
}  // namespace k2

using namespace k2;

extern "C" int k2_lora_merge(const void* base, int ldb, const float* up, const float* down, int rows, int cols, int rank,
                             float scale, void* out, int ldo, k2_stream_t stream) {
  K2_REQUIRE(base && up && down && out, "lora_merge: null pointer");
  K2_REQUIRE(rows >= 1 && cols >= 1 && rank >= 1, "lora_merge: rows, cols and rank must be >= 1");
  K2_REQUIRE(ldb >= cols && ldo >= cols, "lora_merge: row strides must be >= cols");
  K2_REQUIRE((rows + LM_TR - 1) / LM_TR <= 65535, "lora_merge: too many rows");
  const int vec = (ldb % 8 == 0) && (ldo % 8 == 0) &&
                  (((reinterpret_cast<uintptr_t>(base) | reinterpret_cast<uintptr_t>(out)) & 15) == 0);
  const dim3 grid((cols + LM_TC - 1) / LM_TC, (rows + LM_TR - 1) / LM_TR);
  lora_merge_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __half*>(base), ldb, up, down, rows, cols, rank, scale, reinterpret_cast<__half*>(out), ldo, vec);
  K2_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}
