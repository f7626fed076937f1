// k2_clip_text.cu -- the two entry points the CLIP ViT-bigG/14 text tower (kandinsky2/model/clip_text.py) needs on top of the
// flat-row GEMM, LayerNorm, GELU and causal k2_attention_small the diffusion prior already uses:
//   k2_clip_text_embed  int32 token ids -> fp16 rows tok[id] + pos[t] with ONE rounding (the fp16 model's inputs_embeds +
//                       position_embeds), 16-byte vector loads; an id outside [0, V) writes a NaN row and reads nothing.
//   k2_clip_text_pool   the pooled position of every sequence, computed on the device from the ids (eos_id < 0: the first
//                       argmax, transformers' eos_token_id == 2 rule; else the first position equal to eos_id, 0 if none),
//                       and that row of the final-LayerNorm output widened exactly to fp32.  On the device so that a replayed
//                       CUDA graph keeps its addresses while the ids change per call.
// Parity: tests/test_gpu_clip_text_kernels.py (both bit-exact against the torch composition).
#include <limits.h>

#include "../../include/k2b200.h"
#include "k2_common.cuh"
#include "k2_internal.h"

namespace k2 {
namespace {

// One block per row m = b T + t; each thread writes 8 consecutive columns (one uint4) per iteration.
__global__ void __launch_bounds__(128) clip_text_embed_kernel(const int* __restrict__ ids, int ldi, int T,
                                                              const __half* __restrict__ tok, int V,
                                                              const __half* __restrict__ pos, int H, __half* __restrict__ y,
                                                              long long ldy) {
  const int b = blockIdx.x / T, t = blockIdx.x - b * T;
  const int id = ids[static_cast<long long>(b) * ldi + t];
  uint4* yr = reinterpret_cast<uint4*>(y + static_cast<long long>(blockIdx.x) * ldy);
  const int n8 = H >> 3;
  if (id < 0 || id >= V) {
    const __half2 nan2 = __halves2half2(__ushort_as_half(0x7e00), __ushort_as_half(0x7e00));
    uint4 v;
    v.x = v.y = v.z = v.w = *reinterpret_cast<const unsigned int*>(&nan2);
    for (int c = threadIdx.x; c < n8; c += blockDim.x) yr[c] = v;
    return;
  }
  const uint4* tr = reinterpret_cast<const uint4*>(tok + static_cast<long long>(id) * H);
  const uint4* pr = reinterpret_cast<const uint4*>(pos + static_cast<long long>(t) * H);
  for (int c = threadIdx.x; c < n8; c += blockDim.x) {
    const uint4 a = tr[c], p = pr[c];
    const __half2* a2 = reinterpret_cast<const __half2*>(&a);
    const __half2* p2 = reinterpret_cast<const __half2*>(&p);
    uint4 o;
    __half2* o2 = reinterpret_cast<__half2*>(&o);
#pragma unroll
    for (int j = 0; j < 4; ++j) {
      const float2 fa = __half22float2(a2[j]), fp = __half22float2(p2[j]);
      o2[j] = __floats2half2_rn(fa.x + fp.x, fa.y + fp.y);
    }
    yr[c] = o;
  }
}

// One block of 256 threads per sequence b: a block reduction over the T ids picks the pooled position, then the block widens
// that hidden row.  Key per position (smaller wins): argmax rule (eos_id < 0) -> (INT_MAX - id, t); equality rule -> t where
// id == eos_id, ULLONG_MAX elsewhere (all ULLONG_MAX -> position 0).  Ties go to the first position, as torch.argmax.
__global__ void __launch_bounds__(256) clip_text_pool_kernel(const int* __restrict__ ids, int ldi, int T, int eos_id,
                                                             const __half* __restrict__ h, long long ldh, int H,
                                                             float* __restrict__ y, long long ldy, int* __restrict__ index_out) {
  __shared__ unsigned long long sred[8];
  __shared__ int spos;
  const int b = blockIdx.x;
  const int* ir = ids + static_cast<long long>(b) * ldi;
  unsigned long long best = ULLONG_MAX;
  for (int t = threadIdx.x; t < T; t += blockDim.x) {
    const int id = ir[t];
    unsigned long long key;
    if (eos_id < 0)   // the largest id first (INT_MAX - id in [0, 2^32)), then the lowest t
      key = (static_cast<unsigned long long>(0x7fffffffLL - id) << 32) | static_cast<unsigned int>(t);
    else
      key = id == eos_id ? static_cast<unsigned long long>(t) : ULLONG_MAX;
    best = key < best ? key : best;
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    const unsigned long long other = __shfl_xor_sync(0xffffffffu, best, o);
    best = other < best ? other : best;
  }
  if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = best;
  __syncthreads();
  if (threadIdx.x == 0) {
    unsigned long long m = sred[0];
    for (int w = 1; w < 8; ++w) m = sred[w] < m ? sred[w] : m;
    const int p = m == ULLONG_MAX ? 0 : static_cast<int>(m & 0xffffffffULL);
    spos = p;
    if (index_out) index_out[b] = p;
  }
  __syncthreads();
  const __half* hr = h + (static_cast<long long>(b) * T + spos) * ldh;
  float* yr = y + static_cast<long long>(b) * ldy;
  for (int c = threadIdx.x; c < H; c += blockDim.x) yr[c] = __half2float(hr[c]);
}

}  // namespace
}  // namespace k2

using namespace k2;

extern "C" {

int k2_clip_text_embed(const int* ids, int ldi, int B, int T, const void* tok, int V, const void* pos, int H, void* out, int ldo,
                       k2_stream_t stream) {
  K2_REQUIRE(ids && tok && pos && out && B > 0 && T > 0 && V > 0 && H > 0, "clip_text_embed: bad arguments");
  K2_REQUIRE(H % 8 == 0, "clip_text_embed: hidden size must be a multiple of 8");
  K2_REQUIRE(ldi >= T && ldo >= H && ldo % 8 == 0, "clip_text_embed: row strides (ldi >= T, ldo >= H, ldo a multiple of 8)");
  K2_REQUIRE((reinterpret_cast<uintptr_t>(ids) & 3) == 0 && aligned16(tok) && aligned16(pos) && aligned16(out),
             "clip_text_embed: alignment");
  const long long rows = static_cast<long long>(B) * T;
  K2_REQUIRE(rows <= 0x7fffffffLL, "clip_text_embed: too many rows");
  clip_text_embed_kernel<<<static_cast<unsigned int>(rows), 128, 0, static_cast<cudaStream_t>(stream)>>>(
      ids, ldi, T, reinterpret_cast<const __half*>(tok), V, reinterpret_cast<const __half*>(pos), H,
      reinterpret_cast<__half*>(out), ldo);
  K2_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int k2_clip_text_pool(const int* ids, int ldi, int B, int T, int eos_id, const void* hidden, int ldh, int H, float* out, int ldo,
                      int* index_out, k2_stream_t stream) {
  K2_REQUIRE(ids && hidden && out && B > 0 && T > 0 && H > 0, "clip_text_pool: bad arguments");
  K2_REQUIRE(ldi >= T && ldh >= H && ldo >= H, "clip_text_pool: row strides (ldi >= T, ldh >= H, ldo >= H)");
  K2_REQUIRE(((reinterpret_cast<uintptr_t>(ids) | reinterpret_cast<uintptr_t>(out) |
               reinterpret_cast<uintptr_t>(index_out)) & 3) == 0 &&
                 (reinterpret_cast<uintptr_t>(hidden) & 1) == 0,
             "clip_text_pool: alignment");
  clip_text_pool_kernel<<<B, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      ids, ldi, T, eos_id, reinterpret_cast<const __half*>(hidden), ldh, H, out, ldo, index_out);
  K2_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
