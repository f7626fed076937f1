// k2_text_encoder.cu -- the two entry points the Kandinsky 2.1 text encoder (multilingual CLIP: XLM-RoBERTa-large plus a
// Linear, kandinsky2/model/text_encoders.py) needs on top of the flat-row GEMM, LayerNorm, GELU and k2_attention_small:
//   k2_xlmr_embed       int32 token ids -> fp16 rows LayerNorm(word[id] + type_row + pos[p]): the fp32 sum of the three fp16
//                       table rows, the float64 two-pass statistics of k2_layernorm_f16, ONE fp16 rounding.  The position p
//                       is computed on the device from the row's ids (transformers' create_position_ids_from_input_ids:
//                       pad_id + the count of non-pad ids up to and including t, pad_id on a pad id), so one replayed CUDA
//                       graph serves every prompt.  An id outside [0, V) or a position >= P writes a NaN row and reads no
//                       table.
//   k2_masked_mean_f16  fp16 hidden rows -> fp32 mean over the kept tokens (the M-CLIP pooling): fp32 sum in ascending t,
//                       one division by the count; a row with no kept token is 0 / 0 = NaN.
// Parity: tests/test_gpu_text_encoder_kernels.py (float64 references, fp16-ulp bounds).
#include <math.h>

#include "../../include/k2b200.h"
#include "k2_common.cuh"
#include "k2_internal.h"

namespace k2 {
namespace {

constexpr int XE_THREADS = 256;
constexpr int XE_MAX_H = 8192;   // the row lives in dynamic shared memory as fp32: 32 KB

template <typename T>
__device__ __forceinline__ T block_sum(T v, T* sred) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = v;
  __syncthreads();
  v = T(0);
#pragma unroll
  for (int w = 0; w < XE_THREADS / 32; ++w) v += sred[w];
  __syncthreads();  // sred is reused by the next call
  return v;
}

// One block per token row m = b T + t.  Pass 0 counts the non-pad ids of ids[b, 0..t] for the position; pass 1 forms the fp32
// row in shared memory and its double sum; pass 2 the centred sum of squares; pass 3 writes fp16(fma(x_hat, gamma, beta)).
__global__ void __launch_bounds__(XE_THREADS) xlmr_embed_kernel(const int* __restrict__ ids, int ldi, int T, int pad_id,
                                                                const __half* __restrict__ word, int V,
                                                                const __half* __restrict__ pos, int P,
                                                                const __half* __restrict__ type_row,
                                                                const float* __restrict__ g, const float* __restrict__ be,
                                                                float eps, __half* __restrict__ y, long long ldy, int H) {
  extern __shared__ float srow[];
  __shared__ double sred_d[XE_THREADS / 32];
  __shared__ int sred_i[XE_THREADS / 32];
  const int b = blockIdx.x / T, t = blockIdx.x - b * T;
  const int* ir = ids + static_cast<long long>(b) * ldi;
  const int id = ir[t];
  int cnt = 0;
  for (int s = threadIdx.x; s <= t; s += blockDim.x) cnt += ir[s] != pad_id;
  cnt = block_sum(cnt, sred_i);
  const long long p = id == pad_id ? static_cast<long long>(pad_id) : static_cast<long long>(pad_id) + cnt;
  __half* yr = y + static_cast<long long>(blockIdx.x) * ldy;
  if (id < 0 || id >= V || p >= P) {
    for (int c = threadIdx.x; c < H; c += blockDim.x) yr[c] = __ushort_as_half(0x7e00);
    return;
  }
  const __half* wr = word + static_cast<long long>(id) * H;
  const __half* pr = pos + p * H;
  double s = 0.0;
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    const float v = (__half2float(wr[c]) + __half2float(type_row[c])) + __half2float(pr[c]);
    srow[c] = v;
    s += static_cast<double>(v);
  }
  const double mean = block_sum(s, sred_d) / H;
  double q = 0.0;
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    const double d = static_cast<double>(srow[c]) - mean;
    q = fma(d, d, q);
  }
  const double rstd = 1.0 / sqrt(block_sum(q, sred_d) / H + static_cast<double>(eps));
  for (int c = threadIdx.x; c < H; c += blockDim.x) {
    const float xh = static_cast<float>((static_cast<double>(srow[c]) - mean) * rstd);
    yr[c] = __float2half_rn(fmaf(xh, g[c], be[c]));
  }
}

// One thread per (row b, column c): the kept rows' fp32 sum in ascending t, then one division by their count.
__global__ void __launch_bounds__(256) masked_mean_kernel(const __half* __restrict__ h, long long ldh,
                                                          const unsigned char* __restrict__ mask, int ldm, int T, int H,
                                                          float* __restrict__ y, long long ldy) {
  const int b = blockIdx.y;
  const int c = blockIdx.x * blockDim.x + threadIdx.x;
  if (c >= H) return;
  const unsigned char* mr = mask + static_cast<long long>(b) * ldm;
  const __half* hr = h + static_cast<long long>(b) * T * ldh + c;
  float s = 0.f;
  int n = 0;
  for (int t = 0; t < T; ++t) {
    if (mr[t]) {
      s += __half2float(hr[static_cast<long long>(t) * ldh]);
      ++n;
    }
  }
  y[static_cast<long long>(b) * ldy + c] = s / static_cast<float>(n);
}

}  // namespace
}  // namespace k2

using namespace k2;

extern "C" {

int k2_xlmr_embed(const int* ids, int ldi, int B, int T, int pad_id, const void* word, int V, const void* pos, int P,
                  const void* type_row, const float* gamma, const float* beta, float eps, void* out, int ldo, int H,
                  k2_stream_t stream) {
  K2_REQUIRE(ids && word && pos && type_row && gamma && beta && out && B > 0 && T > 0 && V > 0 && P > 0 && H > 0,
             "xlmr_embed: bad arguments");
  K2_REQUIRE(pad_id >= 0, "xlmr_embed: pad_id must be >= 0");
  K2_REQUIRE(H <= XE_MAX_H, "xlmr_embed: hidden size must be at most 8192");
  K2_REQUIRE(ldi >= T && ldo >= H, "xlmr_embed: row strides (ldi >= T, ldo >= H)");
  K2_REQUIRE(eps > 0.f, "xlmr_embed: eps must be positive");
  K2_REQUIRE(((reinterpret_cast<uintptr_t>(ids) | reinterpret_cast<uintptr_t>(gamma) | reinterpret_cast<uintptr_t>(beta)) &
              3) == 0 &&
                 ((reinterpret_cast<uintptr_t>(word) | reinterpret_cast<uintptr_t>(pos) |
                   reinterpret_cast<uintptr_t>(type_row) | reinterpret_cast<uintptr_t>(out)) & 1) == 0,
             "xlmr_embed: alignment");
  const long long rows = static_cast<long long>(B) * T;
  K2_REQUIRE(rows <= 0x7fffffffLL, "xlmr_embed: too many rows");
  xlmr_embed_kernel<<<static_cast<unsigned int>(rows), XE_THREADS, static_cast<size_t>(H) * sizeof(float),
                      static_cast<cudaStream_t>(stream)>>>(
      ids, ldi, T, pad_id, reinterpret_cast<const __half*>(word), V, reinterpret_cast<const __half*>(pos), P,
      reinterpret_cast<const __half*>(type_row), gamma, beta, eps, reinterpret_cast<__half*>(out), ldo, H);
  K2_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int k2_masked_mean_f16(const void* hidden, int ldh, const unsigned char* mask, int ldm, int B, int T, int H, float* out,
                       int ldo, k2_stream_t stream) {
  K2_REQUIRE(hidden && mask && out && B > 0 && T > 0 && H > 0, "masked_mean_f16: bad arguments");
  K2_REQUIRE(ldh >= H && ldm >= T && ldo >= H, "masked_mean_f16: row strides (ldh >= H, ldm >= T, ldo >= H)");
  K2_REQUIRE(B <= 65535, "masked_mean_f16: at most 65535 rows");
  K2_REQUIRE((reinterpret_cast<uintptr_t>(hidden) & 1) == 0 && (reinterpret_cast<uintptr_t>(out) & 3) == 0,
             "masked_mean_f16: alignment");
  const dim3 grid(static_cast<unsigned int>((H + 255) / 256), static_cast<unsigned int>(B));
  masked_mean_kernel<<<grid, 256, 0, static_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const __half*>(hidden), ldh, mask,
                                                                          ldm, T, H, out, ldo);
  K2_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
