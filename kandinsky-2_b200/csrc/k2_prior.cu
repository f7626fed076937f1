// k2_prior.cu -- the three small kernels the diffusion prior (SURVEY.md 8f rank 3, kandinsky2/model/prior.py:46-127) needs
// on top of the GEMM (k2_conv_gemm as a flat-row GEMM): LayerNorm on fp16 rows, exact GELU, and a masked multi-head
// attention over a SHORT sequence (81 tokens, head dim 64).  Two copies keep torch off the graph-replayed prior step
// (PriorTransformer._step_plan): the token rows written into the sequence with their positional embedding, and the fp16 ->
// fp32 widening in front of out_proj.  Both reproduce the eager forward's roundings bit for bit.
//
// Parity: tests/test_gpu_prior_kernels.py checks each kernel against float64 of the same fp16 inputs, bounds in fp16 ulps
// of the float64 value.  Measured on an H100 (400 W):
//   attention_small  T = 1..128 across every 32-key chunk edge, 1 / 3 / 32 heads, B = 1 / 2 / 8, causal and CLIP prefix or
//                    holed keep masks, scores of +-60, strided views: within 1 ulp plus the first-order fp32 error of the
//                    scores and weights; the largest error is 0.46 of that bound (the fp16 output rounding).
//   layernorm_f16    N = 1..2049, rows offset by up to 1000 std, constant rows (exactly fp16(beta)), a 3e4 channel, variance
//                    below eps: within 1 ulp plus 2^-20 (|gamma x_hat| + |beta|); worst 1.34 ulp, on outputs that cancel.
//   gelu_f16         all 65536 fp16 inputs: within 1 ulp of 0.5 x erfc(-x / sqrt 2); worst 0.50 ulp (all correctly rounded).
//   quick_gelu_f16   (the 2.1 ViT-L/14 towers' QuickGELU; tests/test_gpu_clip_vitl14_kernels.py) all 65536 fp16 inputs:
//                    within 1 ulp of x sigmoid(1.702 x); worst 0.500 ulp, 99.995 % correctly rounded.
// tests/test_gpu_zz_prior.py pins the whole prior to tests/golden/prior_tiny.pt (the reference's own classes), and
// tests/test_gpu_zz_prior_full.py runs the full 2.1 prior against the fp32 oracle.  Nothing on the measured denoising path
// calls these entry points; they are not tuned.
#include <math.h>

#include "../../include/k2b200.h"
#include "k2_common.cuh"
#include "k2_internal.h"

namespace k2 {
namespace {

// Sum over the 256 threads of a block in a fixed order; every thread gets the total.
__device__ __forceinline__ double block_sum_256(double v, double* sred) {
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) v += __shfl_xor_sync(0xffffffffu, v, o);
  if ((threadIdx.x & 31) == 0) sred[threadIdx.x >> 5] = v;
  __syncthreads();
  v = 0.0;
#pragma unroll
  for (int w = 0; w < 8; ++w) v += sred[w];
  __syncthreads();  // sred is reused by the next call
  return v;
}

// LayerNorm over the last dimension of fp16 rows, fp32 gain / bias (prior.py:46-53: "supports fp16 inputs but fp32
// gains/biases"), fp16 out.  One block per row.  The statistics are two passes in double: a sum of up to 8192 fp16 values
// is exact in double (2^-24 .. 2^16 spans 40 bits), so the mean is correctly rounded, and the variance is the centred sum
// of squares.  A
// one-pass q/N - mean^2 in fp32 cancels once |mean| >> std: it misses the one-ulp bound on rows offset by 100 std or more,
// and on rows whose variance is below eps.  The row is at most a few KB and the second and third passes read it from L1.
__global__ void __launch_bounds__(256) layernorm_f16_kernel(const __half* __restrict__ x, int ldx,
                                                            const float* __restrict__ g, const float* __restrict__ b,
                                                            __half* __restrict__ y, int ldy, int N, float eps) {
  __shared__ double sred[8];
  const __half* xr = x + static_cast<long long>(blockIdx.x) * ldx;
  double s = 0.0;
  for (int i = threadIdx.x; i < N; i += blockDim.x) s += static_cast<double>(__half2float(xr[i]));
  const double mean = block_sum_256(s, sred) / N;
  double q = 0.0;
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    const double d = static_cast<double>(__half2float(xr[i])) - mean;
    q = fma(d, d, q);
  }
  const double rstd = 1.0 / sqrt(block_sum_256(q, sred) / N + static_cast<double>(eps));
  __half* yr = y + static_cast<long long>(blockIdx.x) * ldy;
  for (int i = threadIdx.x; i < N; i += blockDim.x) {
    const float xh = static_cast<float>((static_cast<double>(__half2float(xr[i])) - mean) * rstd);
    yr[i] = __float2half_rn(fmaf(xh, g[i], b[i]));
  }
}

// nn.GELU() (exact, erf) on fp16, in place or out of place (prior.py:74-83), as 0.5 x erfc(-x / sqrt 2).  torch's
// 0.5 x (1 + erf(x / sqrt 2)) cancels for x < -3 (1 + erf is the difference of two numbers near 1) and misses by up to 2.2
// fp16 ulps there on an H100; erfc keeps its relative accuracy, and every fp16 input comes out within one ulp of the float64
// value.  +-inf and NaN map as in torch's fp32 GELU: +inf, NaN (-inf * 0), NaN.
__global__ void __launch_bounds__(256) gelu_f16_kernel(const __half2* __restrict__ x, __half2* __restrict__ y, long long n2) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n2;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float2 v = __half22float2(x[i]);
    const float a = 0.5f * v.x * erfcf(v.x * -0.70710678118654752f);
    const float c = 0.5f * v.y * erfcf(v.y * -0.70710678118654752f);
    y[i] = __floats2half2_rn(a, c);
  }
}

// OpenAI CLIP's QuickGELU, x sigmoid(1.702 x), on fp16, in place or out of place (the Kandinsky 2.1 ViT-L/14 towers,
// kandinsky2/model/clip_vitl14.py), as x / (1 + exp(-1.702 x)) in fp32 with one final rounding.  The form keeps its relative
// accuracy everywhere: for x >> 0 the denominator is 1 + (tiny), for x << 0 it is exp(...) with no cancellation, and once
// exp overflows (x < -52) the quotient is -0, which is also the correctly rounded fp16 value.  Over all fp16 inputs it is within
// 0.51 ulp of the float64 value.  +-inf and NaN map as in torch's fp32 x * sigmoid(1.702 x): +inf, NaN (-inf / inf), NaN.
__global__ void __launch_bounds__(256) quick_gelu_f16_kernel(const __half2* __restrict__ x, __half2* __restrict__ y,
                                                             long long n2) {
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < n2;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const float2 v = __half22float2(x[i]);
    const float a = v.x / (1.f + expf(-1.702f * v.x));
    const float c = v.y / (1.f + expf(-1.702f * v.y));
    y[i] = __floats2half2_rn(a, c);
  }
}

// QKVMultiheadAttention (prior.py:86-103) for a short sequence: qkv rows [B, T, heads*192] with per-head [q | k | v]
// (64 each), additive mask = causal AND key-padding (prior.py:251-252: where(mask, 0, -inf)[:, None, :] + triu(-inf, 1)),
// softmax in fp32, out [B, T, heads*64].  A query row with no reachable key has sum = 0 and comes out 0 * inf = NaN, as
// torch's softmax of an all -inf row does; that is the contract, not an accident.  One block per (batch, head); K and V of the head in shared memory (rows padded
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

// Token rows of the prior's sequence, as the eager forward builds them (kandinsky2/model/prior.py PriorTransformer.forward):
// the fp32 projection is rounded to fp16 (`v.half()`), then the fp16 positional row is added in fp32 and rounded again
// (torch's fp16 `seq + pos.half()`).  Two roundings, both round-to-nearest-even, so the rows are bit-identical to the eager
// forward's.  One block per row; ldx = 0 / ldp = 0 broadcast one source / positional row to every output row.
__global__ void __launch_bounds__(256) prior_tokens_kernel(const float* __restrict__ x, long long ldx,
                                                           const __half* __restrict__ pos, long long ldp,
                                                           __half* __restrict__ y, long long ldy, int N) {
  const float* xr = x + blockIdx.x * ldx;
  const __half* pr = pos + blockIdx.x * ldp;
  __half* yr = y + blockIdx.x * ldy;
  for (int c = threadIdx.x; c < N; c += blockDim.x) {
    const float v = __half2float(__float2half_rn(xr[c]));
    yr[c] = __float2half_rn(v + __half2float(pr[c]));
  }
}

// Exact fp16 -> fp32 widening of strided rows (the eager forward's `.float()` in front of the fp32 out_proj).
__global__ void __launch_bounds__(256) f16_to_f32_rows_kernel(const __half* __restrict__ x, long long ldx,
                                                              float* __restrict__ y, long long ldy, int N) {
  const __half* xr = x + blockIdx.x * ldx;
  float* yr = y + blockIdx.x * ldy;
  for (int c = threadIdx.x; c < N; c += blockDim.x) yr[c] = __half2float(xr[c]);
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

int k2_quick_gelu_f16(const void* x, void* y, long long n, k2_stream_t stream) {
  K2_REQUIRE(x && y && n > 0 && n % 2 == 0, "quick_gelu_f16: n must be a positive even element count");
  K2_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 3) == 0,
             "quick_gelu_f16: 4-byte alignment");
  long long blocks = (n / 2 + 255) / 256;
  if (blocks > num_sms() * 8) blocks = num_sms() * 8;
  quick_gelu_f16_kernel<<<static_cast<unsigned int>(blocks), 256, 0, static_cast<cudaStream_t>(stream)>>>(
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

int k2_prior_tokens(const float* x, int ldx, const void* pos, int ldp, void* y, int ldy, int M, int N, k2_stream_t stream) {
  K2_REQUIRE(x && pos && y && M > 0 && N > 0, "prior_tokens: bad arguments");
  K2_REQUIRE((ldx == 0 || ldx >= N) && (ldp == 0 || ldp >= N) && ldy >= N, "prior_tokens: row strides");
  K2_REQUIRE((reinterpret_cast<uintptr_t>(x) & 3) == 0 &&
                 ((reinterpret_cast<uintptr_t>(pos) | reinterpret_cast<uintptr_t>(y)) & 1) == 0,
             "prior_tokens: alignment");
  prior_tokens_kernel<<<M, 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, ldx, reinterpret_cast<const __half*>(pos), ldp, reinterpret_cast<__half*>(y), ldy, N);
  K2_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int k2_f16_to_f32(const void* x, int ldx, float* y, int ldy, int M, int N, k2_stream_t stream) {
  K2_REQUIRE(x && y && M > 0 && N > 0, "f16_to_f32: bad arguments");
  K2_REQUIRE(ldx >= N && ldy >= N, "f16_to_f32: row strides");
  K2_REQUIRE((reinterpret_cast<uintptr_t>(x) & 1) == 0 && (reinterpret_cast<uintptr_t>(y) & 3) == 0, "f16_to_f32: alignment");
  f16_to_f32_rows_kernel<<<M, 256, 0, static_cast<cudaStream_t>(stream)>>>(reinterpret_cast<const __half*>(x), ldx, y, ldy,
                                                                          N);
  K2_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
