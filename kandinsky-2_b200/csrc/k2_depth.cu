// k2_depth.cu -- the DPT depth estimator's neck operations (kandinsky2/model/depth.py) on top of the flat-row GEMM,
// k2_conv_gemm convolutions, LayerNorm, GELU and attention the ViT towers already use:
//   k2_relu_f16 / k2_relu_f32   ReLU on strided rows, bit for bit torch.relu on the GPU (clamp_min(x, 0): NaN passes through
//                               with its bits, everything else is fmaxf(x, 0) -- the same instruction, so -0 maps alike).
//   k2_bilinear_f16             bilinear resize of fp16 NHWC rows, any size to any size, with torch's upsample_bilinear2d
//                               index and weight arithmetic in fp32 and one rounding per output.
//   k2_depth_to_space_f16       the scatter of ConvTranspose2d(kernel = stride = s): the GEMM rows [(n, y, x), (a s + b) C + c]
//                               to pixel (s y + a, s x + b), channel c.  The GEMM adds the bias (tiled s^2 times), so this is a
//                               pure copy and the transposed convolution rounds once, as torch's does.
//   k2_readout_rows_f16         the readout "project" input: per image n and patch token t the row [token_t | CLS_n].
// All four are bandwidth-bound; they move fp16 as 16-byte vectors.  Parity: tests/test_gpu_depth_kernels.py (ReLU over all
// fp16 inputs bit for bit, bilinear against float64, scatter and readout bit for bit against the torch composition).
#include <math.h>

#include "../../include/k2b200.h"
#include "k2_common.cuh"
#include "k2_internal.h"

namespace k2 {
namespace {

inline unsigned int grid_for(long long total) {
  long long blocks = (total + 255) / 256;
  const long long cap = static_cast<long long>(num_sms()) * 16;
  return static_cast<unsigned int>(blocks < cap ? blocks : cap);
}

__device__ __forceinline__ __half relu_h(__half x) {
  const float v = __half2float(x);
  return isnan(v) ? x : __float2half_rn(fmaxf(v, 0.f));
}

__device__ __forceinline__ float relu_f(float v) { return isnan(v) ? v : fmaxf(v, 0.f); }

// V = 8: rows of 16-byte vectors; V = 1: scalar fall-back for widths / strides that are not multiples of 8.
template <int V>
__global__ void __launch_bounds__(256) relu_f16_kernel(const __half* x, long long ldx, __half* y, long long ldy, int M,
                                                       int NV) {
  const long long total = static_cast<long long>(M) * NV;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / NV;
    const int v = static_cast<int>(i - r * NV);
    const __half* xp = x + r * ldx + v * V;
    __half* yp = y + r * ldy + v * V;
    if constexpr (V == 8) {
      uint4 u = *reinterpret_cast<const uint4*>(xp);
      __half* h = reinterpret_cast<__half*>(&u);
#pragma unroll
      for (int k = 0; k < 8; ++k) h[k] = relu_h(h[k]);
      *reinterpret_cast<uint4*>(yp) = u;
    } else {
      *yp = relu_h(*xp);
    }
  }
}

template <int V>
__global__ void __launch_bounds__(256) relu_f32_kernel(const float* x, long long ldx, float* y, long long ldy, int M, int NV) {
  const long long total = static_cast<long long>(M) * NV;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const long long r = i / NV;
    const int v = static_cast<int>(i - r * NV);
    const float* xp = x + r * ldx + v * V;
    float* yp = y + r * ldy + v * V;
    if constexpr (V == 4) {
      float4 u = *reinterpret_cast<const float4*>(xp);
      u.x = relu_f(u.x);
      u.y = relu_f(u.y);
      u.z = relu_f(u.z);
      u.w = relu_f(u.w);
      *reinterpret_cast<float4*>(yp) = u;
    } else {
      *yp = relu_f(*xp);
    }
  }
}

// torch's upsample_bilinear2d (CUDA, accscalar_t = float for half): source index align_corners ? r d : max(r (d + 0.5) - 0.5,
// 0), i0 = (int) src, i1 = i0 + (i0 < in - 1), lambda1 = src - i0, lambda0 = 1 - lambda1, then
// l0y (l0x a + l1x b) + l1y (l0x c + l1x d) in fp32 and one rounding.  One thread per output pixel and 8-channel vector.
__global__ void __launch_bounds__(256) bilinear_f16_kernel(const __half* __restrict__ x, long long ldx, int NB, int Hi, int Wi,
                                                           int CV, __half* __restrict__ y, long long ldy, int Ho, int Wo,
                                                           float rh, float rw, int align) {
  const long long total = static_cast<long long>(NB) * Ho * Wo * CV;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(i % CV);
    const long long pix = i / CV;
    const int ox = static_cast<int>(pix % Wo);
    const int oy = static_cast<int>((pix / Wo) % Ho);
    const int n = static_cast<int>(pix / (static_cast<long long>(Wo) * Ho));
    const float sy = align ? rh * static_cast<float>(oy) : fmaxf(rh * (static_cast<float>(oy) + 0.5f) - 0.5f, 0.f);
    const float sx = align ? rw * static_cast<float>(ox) : fmaxf(rw * (static_cast<float>(ox) + 0.5f) - 0.5f, 0.f);
    const int y0 = static_cast<int>(sy), x0 = static_cast<int>(sx);
    const int yp = y0 < Hi - 1 ? 1 : 0, xp = x0 < Wi - 1 ? 1 : 0;
    const float ly1 = sy - static_cast<float>(y0), ly0 = 1.f - ly1;
    const float lx1 = sx - static_cast<float>(x0), lx0 = 1.f - lx1;
    const __half* base = x + (static_cast<long long>(n) * Hi + y0) * Wi * ldx + v * 8;
    const long long r00 = static_cast<long long>(x0) * ldx, r01 = static_cast<long long>(x0 + xp) * ldx;
    const long long dy = static_cast<long long>(yp) * Wi * ldx;
    uint4 a = __ldg(reinterpret_cast<const uint4*>(base + r00)), b = __ldg(reinterpret_cast<const uint4*>(base + r01));
    uint4 c = __ldg(reinterpret_cast<const uint4*>(base + dy + r00)), d = __ldg(reinterpret_cast<const uint4*>(base + dy + r01));
    const __half *ha = reinterpret_cast<const __half*>(&a), *hb = reinterpret_cast<const __half*>(&b);
    const __half *hc = reinterpret_cast<const __half*>(&c), *hd = reinterpret_cast<const __half*>(&d);
    uint4 o;
    __half* ho = reinterpret_cast<__half*>(&o);
#pragma unroll
    for (int k = 0; k < 8; ++k) {
      const float top = lx0 * __half2float(ha[k]) + lx1 * __half2float(hb[k]);
      const float bot = lx0 * __half2float(hc[k]) + lx1 * __half2float(hd[k]);
      ho[k] = __float2half_rn(ly0 * top + ly1 * bot);
    }
    *reinterpret_cast<uint4*>(y + pix * ldy + v * 8) = o;
  }
}

// out[n, s y + a, s x + b, c] = g[(n H + y) W + x, (a s + b) C + c]; one thread per output pixel and 8-channel vector.
__global__ void __launch_bounds__(256) depth_to_space_kernel(const __half* __restrict__ g, long long ldg, int NB, int H, int W,
                                                             int s, int CV, __half* __restrict__ y, long long ldy) {
  const int Ho = s * H, Wo = s * W;
  const long long total = static_cast<long long>(NB) * Ho * Wo * CV;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(i % CV);
    const long long pix = i / CV;
    const int X = static_cast<int>(pix % Wo);
    const int Y = static_cast<int>((pix / Wo) % Ho);
    const int n = static_cast<int>(pix / (static_cast<long long>(Wo) * Ho));
    const int yy = Y / s, a = Y - yy * s, xx = X / s, b = X - xx * s;
    const long long src = ((static_cast<long long>(n) * H + yy) * W + xx) * ldg + static_cast<long long>(a * s + b) * CV * 8;
    *reinterpret_cast<uint4*>(y + pix * ldy + v * 8) = __ldg(reinterpret_cast<const uint4*>(g + src + v * 8));
  }
}

// y[n (T - 1) + t - 1, :] = [h[n T + t, 0:H] | h[n T, 0:H]], t = 1 .. T - 1; one thread per output 8-channel vector.
__global__ void __launch_bounds__(256) readout_rows_kernel(const __half* __restrict__ h, long long ldh, int B, int T, int HV,
                                                           __half* __restrict__ y, long long ldy) {
  const long long total = static_cast<long long>(B) * (T - 1) * 2 * HV;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(i % (2 * HV));
    const long long r = i / (2 * HV);
    const long long n = r / (T - 1), t = r - n * (T - 1) + 1;
    const long long srow = v < HV ? n * T + t : n * T;
    const int col = (v < HV ? v : v - HV) * 8;
    *reinterpret_cast<uint4*>(y + r * ldy + v * 8) = __ldg(reinterpret_cast<const uint4*>(h + srow * ldh + col));
  }
}

}  // namespace
}  // namespace k2

using namespace k2;

extern "C" {

int k2_relu_f16(const void* x, int ldx, void* y, int ldy, int M, int N, k2_stream_t stream) {
  K2_REQUIRE(x && y && M > 0 && N > 0 && ldx >= N && ldy >= N, "relu_f16: bad arguments");
  K2_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 1) == 0, "relu_f16: 2-byte alignment");
  const auto xs = reinterpret_cast<const __half*>(x);
  const auto ys = reinterpret_cast<__half*>(y);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  if (N % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0 && aligned16(x) && aligned16(y))
    relu_f16_kernel<8><<<grid_for(static_cast<long long>(M) * (N / 8)), 256, 0, st>>>(xs, ldx, ys, ldy, M, N / 8);
  else
    relu_f16_kernel<1><<<grid_for(static_cast<long long>(M) * N), 256, 0, st>>>(xs, ldx, ys, ldy, M, N);
  K2_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int k2_relu_f32(const float* x, int ldx, float* y, int ldy, int M, int N, k2_stream_t stream) {
  K2_REQUIRE(x && y && M > 0 && N > 0 && ldx >= N && ldy >= N, "relu_f32: bad arguments");
  K2_REQUIRE(((reinterpret_cast<uintptr_t>(x) | reinterpret_cast<uintptr_t>(y)) & 3) == 0, "relu_f32: 4-byte alignment");
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  const int n = N;
  if (n % 4 == 0 && ldx % 4 == 0 && ldy % 4 == 0 && aligned16(x) && aligned16(y))
    relu_f32_kernel<4><<<grid_for(static_cast<long long>(M) * (n / 4)), 256, 0, st>>>(x, ldx, y, ldy, M, n / 4);
  else
    relu_f32_kernel<1><<<grid_for(static_cast<long long>(M) * n), 256, 0, st>>>(x, ldx, y, ldy, M, n);
  K2_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int k2_bilinear_f16(const void* x, int ldx, int NB, int Hi, int Wi, int C, void* y, int ldy, int Ho, int Wo, int align_corners,
                    k2_stream_t stream) {
  K2_REQUIRE(x && y && NB > 0 && Hi > 0 && Wi > 0 && Ho > 0 && Wo > 0 && C > 0, "bilinear_f16: bad arguments");
  K2_REQUIRE(align_corners == 0 || align_corners == 1, "bilinear_f16: align_corners must be 0 or 1");
  K2_REQUIRE(C % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0 && ldx >= C && ldy >= C,
             "bilinear_f16: C and the row strides must be multiples of 8, strides >= C");
  K2_REQUIRE(aligned16(x) && aligned16(y), "bilinear_f16: x and y must be 16-byte aligned");
  // area_pixel_compute_scale<float> of torch, without a scale factor (the sizes decide)
  const float rh = align_corners ? (Ho > 1 ? static_cast<float>(Hi - 1) / static_cast<float>(Ho - 1) : 0.f)
                                 : static_cast<float>(Hi) / static_cast<float>(Ho);
  const float rw = align_corners ? (Wo > 1 ? static_cast<float>(Wi - 1) / static_cast<float>(Wo - 1) : 0.f)
                                 : static_cast<float>(Wi) / static_cast<float>(Wo);
  const long long total = static_cast<long long>(NB) * Ho * Wo * (C / 8);
  bilinear_f16_kernel<<<grid_for(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __half*>(x), ldx, NB, Hi, Wi, C / 8, reinterpret_cast<__half*>(y), ldy, Ho, Wo, rh, rw,
      align_corners);
  K2_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int k2_depth_to_space_f16(const void* g, int ldg, int NB, int H, int W, int C, int s, void* y, int ldy, k2_stream_t stream) {
  K2_REQUIRE(g && y && NB > 0 && H > 0 && W > 0 && C > 0 && s >= 1, "depth_to_space_f16: bad arguments");
  K2_REQUIRE(C % 8 == 0 && ldg % 8 == 0 && ldy % 8 == 0 && static_cast<long long>(ldg) >= static_cast<long long>(s) * s * C &&
                 ldy >= C,
             "depth_to_space_f16: C and the row strides must be multiples of 8, ldg >= s^2 C, ldy >= C");
  K2_REQUIRE(aligned16(g) && aligned16(y), "depth_to_space_f16: g and y must be 16-byte aligned");
  const long long total = static_cast<long long>(NB) * s * H * s * W * (C / 8);
  depth_to_space_kernel<<<grid_for(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __half*>(g), ldg, NB, H, W, s, C / 8, reinterpret_cast<__half*>(y), ldy);
  K2_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int k2_readout_rows_f16(const void* h, int ldh, int B, int T, int H, void* y, int ldy, k2_stream_t stream) {
  K2_REQUIRE(h && y && B > 0 && T > 1 && H > 0, "readout_rows_f16: bad arguments");
  K2_REQUIRE(H % 8 == 0 && ldh % 8 == 0 && ldy % 8 == 0 && ldh >= H && ldy >= 2 * H,
             "readout_rows_f16: H and the row strides must be multiples of 8, ldh >= H, ldy >= 2 H");
  K2_REQUIRE(aligned16(h) && aligned16(y), "readout_rows_f16: h and y must be 16-byte aligned");
  const long long total = static_cast<long long>(B) * (T - 1) * 2 * (H / 8);
  readout_rows_kernel<<<grid_for(total), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      reinterpret_cast<const __half*>(h), ldh, B, T, H / 8, reinterpret_cast<__half*>(y), ldy);
  K2_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
