// k2_bit.cu -- the BiT ResNet-50 backbone of the hybrid DPT (MiDaS v3 DPT-Hybrid; kandinsky2/model/depth.py).  Its 1x1 and
// 3x3 convolutions are k2_conv_gemm launches with fused GroupNorm partials; these are the rest:
//   k2_im2col_f16     the 7x7 stride-2 stem's input rows: fp32 NCHW pixels -> fp16 GEMM rows in weight.reshape(Cout, -1)'s
//                     (c, ky, kx) column order, explicit top / left zero padding, zero columns up to Kp, one rounding each.
//   k2_maxpool_f16    3x3 stride-2 max pool of fp16 NHWC with explicit top / left padding whose value is 0 (BitMaxPool2d pads
//                     with DynamicPad2d(value=0), not -inf), compared as torch's max_pool2d does: (v > m) || isnan(v) in scan
//                     order, so the first of equal values (+0 / -0) wins.
//   k2_gn_act_f16     y = [relu]((x - mu) rstd gamma + beta + r): GroupNorm with the statistics of k2_gn_stats / k2_gn_finalize,
//                     r nothing, an fp16 source, or a second GroupNorm-normalised source with its own statistics and affine.
//                     fp32 arithmetic, one rounding.  k2_gn_apply is not used here: its act means SiLU.
// All three are bandwidth-bound grid-stride loops; the last two move fp16 as 16-byte vectors.  Parity:
// tests/test_gpu_dpt_hybrid_kernels.py.
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

// y[(n Ho + oy) Wo + ox, j] = fp16(x[n, c, oy s - pt + ky, ox s - pl + kx]) for j = (c k + ky) k + kx < k^2 C (0 outside the
// image), 0 for k^2 C <= j < Kp.  One thread per output element.
__global__ void __launch_bounds__(256) im2col_kernel(const float* __restrict__ x, int NB, int C, int H, int W, int k, int s,
                                                     int pt, int pl, int Ho, int Wo, __half* __restrict__ y, long long ldy,
                                                     int Kp) {
  pdl_wait();
  pdl_launch();
  const int K = k * k * C;
  const long long total = static_cast<long long>(NB) * Ho * Wo * Kp;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int j = static_cast<int>(i % Kp);
    const long long r = i / Kp;
    float v = 0.f;
    if (j < K) {
      const int ox = static_cast<int>(r % Wo);
      const int oy = static_cast<int>((r / Wo) % Ho);
      const int n = static_cast<int>(r / (static_cast<long long>(Wo) * Ho));
      const int c = j / (k * k), kk = j - c * k * k, ky = kk / k, kx = kk - ky * k;
      const int iy = oy * s - pt + ky, ix = ox * s - pl + kx;
      if (iy >= 0 && iy < H && ix >= 0 && ix < W) v = __ldg(x + ((static_cast<long long>(n) * C + c) * H + iy) * W + ix);
    }
    y[r * ldy + j] = __float2half_rn(v);
  }
}

// One thread per output pixel and 8-channel vector.
__global__ void __launch_bounds__(256) maxpool_kernel(const __half* __restrict__ x, long long ldx, int NB, int H, int W, int CV,
                                                      int pt, int pl, int Ho, int Wo, __half* __restrict__ y, long long ldy) {
  pdl_wait();
  pdl_launch();
  const long long total = static_cast<long long>(NB) * Ho * Wo * CV;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(i % CV);
    const long long pix = i / CV;
    const int ox = static_cast<int>(pix % Wo);
    const int oy = static_cast<int>((pix / Wo) % Ho);
    const int n = static_cast<int>(pix / (static_cast<long long>(Wo) * Ho));
    __half m[8];
    float mf[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      m[e] = __float2half_rn(-INFINITY);
      mf[e] = -INFINITY;
    }
    for (int ky = 0; ky < 3; ++ky) {
      const int iy = 2 * oy - pt + ky;
      for (int kx = 0; kx < 3; ++kx) {
        const int ix = 2 * ox - pl + kx;
        uint4 u = make_uint4(0u, 0u, 0u, 0u);   // the pad value: +0
        if (iy >= 0 && iy < H && ix >= 0 && ix < W)
          u = __ldg(reinterpret_cast<const uint4*>(x + ((static_cast<long long>(n) * H + iy) * W + ix) * ldx + v * 8));
        const __half* h = reinterpret_cast<const __half*>(&u);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float f = __half2float(h[e]);
          if (f > mf[e] || isnan(f)) {
            mf[e] = f;
            m[e] = h[e];
          }
        }
      }
    }
    *reinterpret_cast<uint4*>(y + pix * ldy + v * 8) = *reinterpret_cast<const uint4*>(m);
  }
}

// (a, b) of the 8 channels c0 .. c0 + 7 of image n: the GroupNorm as x a + b.
__device__ __forceinline__ void gn_affine(const float* __restrict__ stats, const float* __restrict__ gamma,
                                          const float* __restrict__ beta, int n, int c0, int groups, int cpg, float (&a)[8],
                                          float (&b)[8]) {
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    const int g = (c0 + e) / cpg;
    const float2 st = __ldg(reinterpret_cast<const float2*>(stats + (static_cast<long long>(n) * groups + g) * 2));
    const float ga = __ldg(gamma + c0 + e) * st.y;
    a[e] = ga;
    b[e] = __ldg(beta + c0 + e) - st.x * ga;
  }
}

// RES 0: no r; 1: r an fp16 source; 2: r a GroupNorm-normalised source.  One thread per pixel and 8-channel vector.
template <int RES>
__global__ void __launch_bounds__(256) gn_act_kernel(const __half* __restrict__ x, long long ldx, const float* __restrict__ st,
                                                     const float* __restrict__ ga, const float* __restrict__ be,
                                                     const __half* __restrict__ r, long long ldr, const float* __restrict__ rst,
                                                     const float* __restrict__ rga, const float* __restrict__ rbe, int NB,
                                                     int HW, int CV, int groups, int relu, __half* __restrict__ y,
                                                     long long ldy, long long ldy_img) {
  pdl_wait();
  pdl_launch();
  const int cpg = CV * 8 / groups;
  const long long total = static_cast<long long>(NB) * HW * CV;
  for (long long i = blockIdx.x * static_cast<long long>(blockDim.x) + threadIdx.x; i < total;
       i += static_cast<long long>(gridDim.x) * blockDim.x) {
    const int v = static_cast<int>(i % CV);
    const long long pix = i / CV;
    const int n = static_cast<int>(pix / HW);
    const int p = static_cast<int>(pix - static_cast<long long>(n) * HW);
    const int c0 = v * 8;
    float a[8], b[8], f[8], o[8];
    gn_affine(st, ga, be, n, c0, groups, cpg, a, b);
    const uint4 ux = __ldg(reinterpret_cast<const uint4*>(x + pix * ldx + c0));
    const __half* hx = reinterpret_cast<const __half*>(&ux);
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = fmaf(__half2float(hx[e]), a[e], b[e]);
    if constexpr (RES > 0) {
      const uint4 ur = __ldg(reinterpret_cast<const uint4*>(r + pix * ldr + c0));
      const __half* hr = reinterpret_cast<const __half*>(&ur);
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] = __half2float(hr[e]);
      if constexpr (RES == 2) {
        gn_affine(rst, rga, rbe, n, c0, groups, cpg, a, b);
#pragma unroll
        for (int e = 0; e < 8; ++e) f[e] = fmaf(f[e], a[e], b[e]);
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) o[e] += f[e];
    }
    uint4 uo;
    __half* ho = reinterpret_cast<__half*>(&uo);
#pragma unroll
    for (int e = 0; e < 8; ++e) ho[e] = __float2half_rn(relu ? fmaxf(o[e], 0.f) : o[e]);
    *reinterpret_cast<uint4*>(y + n * ldy_img + static_cast<long long>(p) * ldy + c0) = uo;
  }
}

}  // namespace
}  // namespace k2

using namespace k2;

extern "C" {

int k2_im2col_f16(const float* x, int NB, int C, int H, int W, int k, int s, int pad_top, int pad_left, int Ho, int Wo,
                  void* y, int ldy, int Kp, k2_stream_t stream) {
  K2_REQUIRE(x && y && NB > 0 && C > 0 && H > 0 && W > 0 && k > 0 && s > 0 && Ho > 0 && Wo > 0,
             "im2col_f16: bad arguments");
  K2_REQUIRE(pad_top >= 0 && pad_left >= 0 && pad_top < k && pad_left < k, "im2col_f16: pads must be in [0, k)");
  K2_REQUIRE(Kp >= k * k * C && ldy >= Kp, "im2col_f16: Kp >= k^2 C and ldy >= Kp");
  K2_REQUIRE((reinterpret_cast<uintptr_t>(x) & 3) == 0 && (reinterpret_cast<uintptr_t>(y) & 1) == 0,
             "im2col_f16: x 4-byte, y 2-byte aligned");
  const long long total = static_cast<long long>(NB) * Ho * Wo * Kp;
  K2_CHECK_CUDA(launch_k(im2col_kernel, dim3(grid_for(total)), dim3(256), 0, static_cast<cudaStream_t>(stream), x, NB, C, H, W,
                         k, s, pad_top, pad_left, Ho, Wo, reinterpret_cast<__half*>(y), static_cast<long long>(ldy), Kp));
  count_launch();
  return 0;
}

int k2_maxpool_f16(const void* x, int ldx, int NB, int H, int W, int C, int pad_top, int pad_left, int Ho, int Wo, void* y,
                   int ldy, k2_stream_t stream) {
  K2_REQUIRE(x && y && NB > 0 && H > 0 && W > 0 && C > 0 && Ho > 0 && Wo > 0, "maxpool_f16: bad arguments");
  K2_REQUIRE(pad_top >= 0 && pad_left >= 0 && pad_top < 3 && pad_left < 3, "maxpool_f16: pads must be in [0, 3)");
  K2_REQUIRE(C % 8 == 0 && ldx % 8 == 0 && ldy % 8 == 0 && ldx >= C && ldy >= C,
             "maxpool_f16: C and the row strides must be multiples of 8, strides >= C");
  K2_REQUIRE(aligned16(x) && aligned16(y), "maxpool_f16: x and y must be 16-byte aligned");
  const long long total = static_cast<long long>(NB) * Ho * Wo * (C / 8);
  K2_CHECK_CUDA(launch_k(maxpool_kernel, dim3(grid_for(total)), dim3(256), 0, static_cast<cudaStream_t>(stream),
                         reinterpret_cast<const __half*>(x), static_cast<long long>(ldx), NB, H, W, C / 8, pad_top, pad_left,
                         Ho, Wo, reinterpret_cast<__half*>(y), static_cast<long long>(ldy)));
  count_launch();
  return 0;
}

int k2_gn_act_f16(const void* x, int ldx, const float* stats, const float* gamma, const float* beta, const void* r, int ldr,
                  const float* r_stats, const float* r_gamma, const float* r_beta, int NB, int H, int W, int C, int groups,
                  int relu, void* y, int ldy, long long ldy_img, k2_stream_t stream) {
  K2_REQUIRE(x && y && stats && gamma && beta && NB > 0 && H > 0 && W > 0 && C > 0 && groups > 0,
             "gn_act_f16: bad arguments");
  K2_REQUIRE(relu == 0 || relu == 1, "gn_act_f16: relu must be 0 or 1");
  K2_REQUIRE(C % 8 == 0 && C % groups == 0, "gn_act_f16: C must be a multiple of 8 and of groups");
  K2_REQUIRE(ldx % 8 == 0 && ldy % 8 == 0 && ldx >= C && ldy >= C && (!r || (ldr % 8 == 0 && ldr >= C)),
             "gn_act_f16: row strides must be multiples of 8 and >= C");
  const long long HW = static_cast<long long>(H) * W;
  K2_REQUIRE(ldy_img % 8 == 0 && ldy_img >= (HW - 1) * ldy + C, "gn_act_f16: ldy_img must be a multiple of 8 covering an image");
  K2_REQUIRE(!r_stats || (r && r_gamma && r_beta), "gn_act_f16: a normalised residual needs r, r_gamma and r_beta");
  K2_REQUIRE(aligned16(x) && aligned16(y) && aligned16(r), "gn_act_f16: x, y and r must be 16-byte aligned");
  K2_REQUIRE(((reinterpret_cast<uintptr_t>(stats) | reinterpret_cast<uintptr_t>(r_stats)) & 7) == 0,
             "gn_act_f16: statistics must be 8-byte aligned");
  const long long total = static_cast<long long>(NB) * HW * (C / 8);
  const cudaStream_t st = static_cast<cudaStream_t>(stream);
  auto go = [&](auto kernel) {
    return launch_k(kernel, dim3(grid_for(total)), dim3(256), 0, st, reinterpret_cast<const __half*>(x),
                    static_cast<long long>(ldx), stats, gamma, beta, reinterpret_cast<const __half*>(r),
                    static_cast<long long>(ldr), r_stats, r_gamma, r_beta, NB, static_cast<int>(HW), C / 8, groups, relu,
                    reinterpret_cast<__half*>(y), static_cast<long long>(ldy), ldy_img);
  };
  if (!r) K2_CHECK_CUDA(go(gn_act_kernel<0>));
  else if (!r_stats) K2_CHECK_CUDA(go(gn_act_kernel<1>));
  else K2_CHECK_CUDA(go(gn_act_kernel<2>));
  count_launch();
  return 0;
}

}  // extern "C"
