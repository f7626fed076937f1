// k2_prior.cu -- the three small kernels the diffusion prior (SURVEY.md 8f rank 3, kandinsky2/model/prior.py:46-127) needs
// on top of the GEMM (k2_conv_gemm as a flat-row GEMM): LayerNorm on fp16 rows, exact GELU, and a masked multi-head
// attention over a SHORT sequence (81 tokens, head dim 64).
//
// Parity: tests/test_gpu_zz_prior.py (each kernel against torch fp32, the whole prior against tests/golden/prior_tiny.pt = the
// reference's own classes).  Nothing on the measured denoising path calls these entry points; they are not tuned.
#include <math.h>

#include "../../include/k2b200.h"
#include "k2_common.cuh"
#include "k2_internal.h"

namespace k2 {
namespace {

// LayerNorm over the last dimension of fp16 rows, fp32 statistics and affine (prior.py:46-53: "supports fp16 inputs but
// fp32 gains/biases"), fp16 out.  One block per row.
__global__ void __launch_bounds__(256) layernorm_f16_kernel(const __half* __restrict__ x, int ldx,
                                                            const float* __restrict__ g, const float* __restrict__ b,
                                                            __half* __restrict__ y, int ldy, int N, float eps) {
  __shared__ float sred[2][8];
  const __half* xr = x + static_cast<long long>(blockIdx.x) * ldx;
  float s = 0.f, q = 0.f;
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    const float v = __half2float(xr[i]);
    s += v;
    q = fmaf(v, v, q);
  }
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_xor_sync(0xffffffffu, s, o);
    q += __shfl_xor_sync(0xffffffffu, q, o);
  }
  if ((threadIdx.x & 31) == 0) {
    sred[0][threadIdx.x >> 5] = s;
    sred[1][threadIdx.x >> 5] = q;
  }
  __syncthreads();
  s = 0.f;
  q = 0.f;
#pragma unroll
  for (int w = 0; w < 8; ++w) {  // fixed order
    s += sred[0][w];
    q += sred[1][w];
  }
  const float mean = s / N;
  const float var = fmaxf(q / N - mean * mean, 0.f);
  const float rstd = rsqrtf(var + eps);
  __half* yr = y + static_cast<long long>(blockIdx.x) * ldy;
  for (int i = threadIdx.x; i < N; i += blockDim.x)
    yr[i] = __float2half_rn((__half2float(xr[i]) - mean) * rstd * g[i] + b[i]);
}

// nn.GELU() (exact, erf) on fp16, in place or out of place (prior.py:74-83)
__global__ void __launch_bounds__(256) gelu_f16_kernel(const __half2* __restrict__ x, __half2* __restrict__ y, long long n2) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n2;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float2 v = __half22float2(x[i]);
    const float a = 0.5f * v.x * (1.f + erff(v.x * 0.70710678118654752f));
    const float c = 0.5f * v.y * (1.f + erff(v.y * 0.70710678118654752f));
    y[i] = __floats2half2_rn(a, c);
  }
}

// QKVMultiheadAttention (prior.py:86-103) for a short sequence: qkv rows [B, T, heads*192] with per-head [q | k | v]
// (64 each), additive mask = causal AND key-padding (prior.py:251-252: where(mask, 0, -inf)[:, None, :] + triu(-inf, 1)),
// softmax in fp32, out [B, T, heads*64].  One block per (batch, head); K and V of the head in shared memory (rows padded
// to 66 halfs against bank conflicts), one warp per query row, lanes over keys for the scores and over channels for PV.
constexpr int SA_MAXT = 128;
constexpr int SA_PITCH = 66;

__global__ void __launch_bounds__(256) attention_small_kernel(const __half* __restrict__ qkv, int ldq,
                                                              const unsigned char* __restrict__ keep, int causal,
                                                              __half* __restrict__ out, int ldo, int T, int heads,
                                                              float scale) {
  __shared__ __half sK[SA_MAXT * SA_PITCH];
  __shared__ __half sV[SA_MAXT * SA_PITCH];
  __shared__ float sP[8][SA_MAXT];
  const int b = blockIdx.x / heads, h = blockIdx.x % heads;
  const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
  const __half* base = qkv + static_cast<long long>(b) * T * ldq + h * 192;
  for (int i = threadIdx.x; i < T * 64; i += blockDim.x) {
    const int s = i >> 6, c = i & 63;
    sK[s * SA_PITCH + c] = base[static_cast<long long>(s) * ldq + 64 + c];
    sV[s * SA_PITCH + c] = base[static_cast<long long>(s) * ldq + 128 + c];
  }
  __syncthreads();
  for (int t = warp; t < T; t += 8) {
    // q row in registers: lane holds channels 2*lane, 2*lane+1
    const __half2 q2 = *reinterpret_cast<const __half2*>(base + static_cast<long long>(t) * ldq + 2 * lane);
    const float2 qf = __half22float2(q2);
    float sc[SA_MAXT / 32];
    float mx = -INFINITY;
#pragma unroll
    for (int u = 0; u < SA_MAXT / 32; ++u) {
      const int s = u * 32 + lane;
      sc[u] = -INFINITY;
      // every lane needs the full dot product of q with ITS key: q is distributed, so gather it by shuffles
      float acc = 0.f;
      if (u * 32 < T) {
#pragma unroll 8
        for (int c2 = 0; c2 < 32; ++c2) {
          const float qx = __shfl_sync(0xffffffffu, qf.x, c2), qy = __shfl_sync(0xffffffffu, qf.y, c2);
          if (s < T) {
            const float2 kf = __half22float2(*reinterpret_cast<const __half2*>(&sK[s * SA_PITCH + 2 * c2]));
            acc = fmaf(qx, kf.x, fmaf(qy, kf.y, acc));
          }
        }
        const bool ok = s < T && (!causal || s <= t) && (!keep || keep[b * T + s]);
        if (ok) sc[u] = acc * scale;
      }
      mx = fmaxf(mx, sc[u]);
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) mx = fmaxf(mx, __shfl_xor_sync(0xffffffffu, mx, o));
    float sum = 0.f;
#pragma unroll
    for (int u = 0; u < SA_MAXT / 32; ++u) {
      const float p = (sc[u] == -INFINITY) ? 0.f : __expf(sc[u] - mx);
      sum += p;
      if (u * 32 + lane < SA_MAXT) sP[warp][u * 32 + lane] = p;
    }
#pragma unroll
    for (int o = 16; o > 0; o >>= 1) sum += __shfl_xor_sync(0xffffffffu, sum, o);
    __syncwarp();
    const float inv = 1.f / sum;
    float ox = 0.f, oy = 0.f;  // channels 2*lane, 2*lane+1
    for (int s = 0; s < T; ++s) {
      const float p = sP[warp][s];
      const float2 vf = __half22float2(*reinterpret_cast<const __half2*>(&sV[s * SA_PITCH + 2 * lane]));
      ox = fmaf(p, vf.x, ox);
      oy = fmaf(p, vf.y, oy);
    }
    *reinterpret_cast<__half2*>(out + (static_cast<long long>(b) * T + t) * ldo + h * 64 + 2 * lane) =
        __floats2half2_rn(ox * inv, oy * inv);
    __syncwarp();
  }
}

}  // namespace
}  // namespace k2

using namespace k2;

extern "C" {

int k2_layernorm_f16(const void* x, int ldx, const float* gamma, const float* beta, void* y, int ldy, int M, int N, float eps,
                     k2_stream_t stream) {
  K2_REQUIRE(x && gamma && beta && y && M > 0 && N > 0 && ldx >= N && ldy >= N, "layernorm_f16: bad arguments");
  layernorm_f16_kernel<<<M, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __half*>(x), ldx, gamma, beta, reinterpret_cast<__half*>(y), ldy, N, eps);
  K2_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int k2_gelu_f16(const void* x, void* y, long long n, k2_stream_t stream) {
  K2_REQUIRE(x && y && n > 0 && n % 2 == 0, "gelu_f16: n must be a positive even element count");
  K2_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 3) == 0, "gelu_f16: 4-byte alignment");
  long long blocks = (n / 2 + 255) / 256;
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  gelu_f16_kernel<<<static_cast<unsigned int>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __half2*>(x), reinterpret_cast<__half2*>(y), n / 2);
  K2_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int k2_attention_small(const void* qkv, int ldq, const unsigned char* keep_mask, int causal, void* out, int ldo, int B, int T,
                       int heads, float scale, k2_stream_t stream) {
  K2_REQUIRE(qkv && out && B > 0 && heads > 0, "attention_small: bad arguments");
  K2_REQUIRE(T > 0 && T <= SA_MAXT, "attention_small: sequence length must be 1..128");
  K2_REQUIRE(ldq >= heads * 192 && ldo >= heads * 64 && ldq % 2 == 0 && ldo % 2 == 0, "attention_small: row strides");
  K2_REQUIRE(((reinterpret_cast<uintptr_t>(qkv) | reinterpret_cast<uintptr_t>(out)) & 3) == 0, "attention_small: alignment");
  attention_small_kernel<<<B * heads, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __half*>(qkv), ldq, keep_mask, causal, reinterpret_cast<__half*>(out), ldo, T, heads, scale);
  K2_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
