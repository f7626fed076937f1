// k2_movq.cu -- MoVQ decoder elementwise kernels: SpatialNorm apply and the fp16 transpose of the attention values.
//
// Replaces (reference file:line):
//   SpatialNorm.forward   kandinsky2/vqgan/movq_modules.py:61-68
//       zq = interpolate(zq, size=f.shape[-2:], mode="nearest"); y = GroupNorm(f) * conv_y(zq) + conv_b(zq)   (+ swish, :21-23)
//   AttnBlock's  v.reshape / permute before torch.bmm   movq_modules.py:216-219
//
// SpatialNorm is HBM-bound: one read and one write of the feature map (up to 604 MB per tensor at 768x768).  The generic
// gn_apply kernel would re-derive the 2 x (4 -> C) modulation with 80 read-only loads per thread every time the latent pixel
// under a thread changes.  Here everything that does not depend on the pixel is folded ONCE per thread into 10 coefficients
// per channel that live in registers:
//       y = x * a(z) + b(z),   a(z) = A (wy.z + by),   b(z) = B (wy.z + by) + (wb.z + bb),   A = gamma rstd,  B = beta - mean A
//   ->  a = a5[0..3].z + a5[4],  b = b5[0..3].z + b5[4], evaluated once per (latent pixel, channel) and reused for the run of
//       pixels under it: ~2 FMA per element at the fine levels, the 4-float latent pixel z comes from L1.
#include "../../include/k2b200.h"
#include "k2_common.cuh"
#include "k2_internal.h"

namespace k2 {
namespace {

constexpr int VX = 16;   // channel vectors (8 fp16 = 16 B) per block: a half warp covers 256 contiguous bytes of a pixel
constexpr int PY = 16;   // pixel lanes per block
constexpr int UN = 8;    // vectors per thread per iteration, two iterations in flight (16 x 16 B loads per thread)

struct SnParams {
  const __half* x;
  int C, ldx;
  int NB, H, W, groups;
  const float* stats;   // [NB, groups, 2] (mean, rstd)
  const float* gamma;
  const float* beta;
  const float* zq;      // fp32 [NB, zh, zw, 4]
  int zh, zw;
  const float* sn_w;    // fp32 [C, 10] = (wy[4], by, wb[4], bb)
  int act;
  __half* y;
  int ldy;
  int chunk;            // pixels per block
  int zshift;           // log2(H / zh) when H / zh == W / zw is a power of two (nearest resize = a shift), else -1
};

__global__ void __launch_bounds__(256, 2) sn_apply_kernel(const SnParams p) {
  // the block's 128 channels x 10 folded coefficients live in shared memory as [k][vx][8 channels]: a thread re-reads its
  // 80 values (20 LDS.128, conflict-free: a half warp covers 512 contiguous bytes) only when the latent pixel under it changes,
  // which keeps the kernel at <= 128 registers = two resident blocks per SM with 16 x 16 B loads in flight per thread
  __shared__ __align__(16) float cs[10][VX][8];
  const int vx = threadIdx.x % VX;
  const int py = threadIdx.x / VX;
  const int v = blockIdx.y * VX + vx;
  const int n = blockIdx.z;
  const int CV = p.C / 8;
  pdl_wait();
  pdl_launch();
  {
    const int cpg = p.C / p.groups;
    for (int i = threadIdx.x; i < VX * 8; i += blockDim.x) {  // one thread per channel of the slab
      const int c = blockIdx.y * VX * 8 + i;
      if (c >= p.C) continue;
      const float2 st = __ldg(reinterpret_cast<const float2*>(p.stats + (static_cast<long long>(n) * p.groups + c / cpg) * 2));
      const float A = __ldg(p.gamma + c) * st.y;
      const float B = __ldg(p.beta + c) - st.x * A;
      const float* w = p.sn_w + static_cast<long long>(c) * 10;
#pragma unroll
      for (int k = 0; k < 5; ++k) {
        const float wy = __ldg(w + k), wb = __ldg(w + 5 + k);
        cs[k][i >> 3][i & 7] = A * wy;
        cs[5 + k][i >> 3][i & 7] = fmaf(B, wy, wb);
      }
    }
  }
  __syncthreads();
  if (v >= CV) return;
  const int c0 = v * 8;
  const int HW = p.H * p.W;
  const int p0 = blockIdx.x * p.chunk;
  const int p1 = min(HW, p0 + p.chunk);
  const __half* xb = p.x + c0;
  __half* yb = p.y + c0;
  const long long img = static_cast<long long>(n) * HW;
  const float4* zb = reinterpret_cast<const float4*>(p.zq) + static_cast<long long>(n) * p.zh * p.zw;

  uint4 raw[UN], nxt[UN];
  auto load_set = [&](int pp, uint4 (&dst)[UN]) {
#pragma unroll
    for (int u = 0; u < UN; ++u)
      if (pp + u < p1) dst[u] = __ldg(reinterpret_cast<const uint4*>(xb + (img + pp + u) * p.ldx));
  };
  // the per-channel (a, b) of the current latent pixel: a thread's UN consecutive pixels lie under the same latent pixel
  // wherever the feature map is >= UN times finer than the latent (the 384^2 and 768^2 levels, i.e. most of the bytes), so
  // the 2 x 8 x 4 modulation FMAs are paid once per run instead of once per pixel
  int last_z = -1;
  float a8[8], b8[8];
#pragma unroll
  for (int e = 0; e < 8; ++e) a8[e] = b8[e] = 0.f;
  int pp = p0 + py * UN;
  if (pp < p1) load_set(pp, raw);
  for (; pp < p1; pp += UN * PY) {
    const int npp = pp + UN * PY;
    if (npp < p1) load_set(npp, nxt);
    // one division per run of UN pixels: runs start at multiples of UN and W % UN == 0 on the fast path, so a run never
    // leaves its image row; the latent pixel is a shift where the scale is a power of two (all MoVQ decoder levels)
    const int y_run = pp / p.W, x_run = pp - y_run * p.W;
    const bool fast = (p.W % UN == 0) && (p.zshift >= 0);
#pragma unroll
    for (int u = 0; u < UN; ++u) {
      const int q = pp + u;
      if (q >= p1) break;
      int zi;
      if (fast) {
        zi = (y_run >> p.zshift) * p.zw + ((x_run + u) >> p.zshift);
      } else {
        const int yi = q / p.W, xi = q - yi * p.W;
        zi = ((yi * p.zh) / p.H) * p.zw + (xi * p.zw) / p.W;   // nearest: floor(dst * in / out)
      }
      if (zi != last_z) {
        last_z = zi;
        const float4 z = __ldg(zb + zi);
        const float zz[4] = {z.x, z.y, z.z, z.w};
#pragma unroll
        for (int hh = 0; hh < 2; ++hh) {  // channels 4*hh .. 4*hh+3
          float4 ta = *reinterpret_cast<const float4*>(&cs[4][vx][4 * hh]);
          float4 tb = *reinterpret_cast<const float4*>(&cs[9][vx][4 * hh]);
#pragma unroll
          for (int k = 0; k < 4; ++k) {
            const float4 wa = *reinterpret_cast<const float4*>(&cs[k][vx][4 * hh]);
            const float4 wb = *reinterpret_cast<const float4*>(&cs[5 + k][vx][4 * hh]);
            ta.x = fmaf(wa.x, zz[k], ta.x); ta.y = fmaf(wa.y, zz[k], ta.y); ta.z = fmaf(wa.z, zz[k], ta.z); ta.w = fmaf(wa.w, zz[k], ta.w);
            tb.x = fmaf(wb.x, zz[k], tb.x); tb.y = fmaf(wb.y, zz[k], tb.y); tb.z = fmaf(wb.z, zz[k], tb.z); tb.w = fmaf(wb.w, zz[k], tb.w);
          }
          a8[4 * hh] = ta.x; a8[4 * hh + 1] = ta.y; a8[4 * hh + 2] = ta.z; a8[4 * hh + 3] = ta.w;
          b8[4 * hh] = tb.x; b8[4 * hh + 1] = tb.y; b8[4 * hh + 2] = tb.z; b8[4 * hh + 3] = tb.w;
        }
      }
      const __half2* h2 = reinterpret_cast<const __half2*>(&raw[u]);
      uint4 ov;
      __half2* oh = reinterpret_cast<__half2*>(&ov);
#pragma unroll
      for (int e2 = 0; e2 < 4; ++e2) {
        const float2 f = __half22float2(h2[e2]);
        const float t0 = fmaf(f.x, a8[2 * e2], b8[2 * e2]);
        const float t1 = fmaf(f.y, a8[2 * e2 + 1], b8[2 * e2 + 1]);
        oh[e2] = __floats2half2_rn(p.act ? silu_f(t0) : t0, p.act ? silu_f(t1) : t1);
      }
      *reinterpret_cast<uint4*>(yb + (img + q) * p.ldy) = ov;
    }
#pragma unroll
    for (int u = 0; u < UN; ++u) raw[u] = nxt[u];
  }
}

// fp16 [B][T][ldx] (C columns) -> [B][C][T]: 64 x 64 tiles through shared memory, 16-byte accesses on both sides.
__global__ void __launch_bounds__(256) transpose_f16_kernel(const __half* __restrict__ x, int ldx, __half* __restrict__ y,
                                                            int T, int C) {
  __shared__ __half tile[64][64 + 8];
  const int b = blockIdx.z;
  const int t0 = blockIdx.x * 64, c0 = blockIdx.y * 64;
  pdl_wait();
  pdl_launch();
  const __half* xb = x + static_cast<long long>(b) * T * ldx;
  __half* yb = y + static_cast<long long>(b) * C * T;
  for (int i = threadIdx.x; i < 64 * 8; i += 256) {  // 64 rows (t) x 8 vectors of 8 channels
    const int r = i >> 3, vv = i & 7;
    uint4 val = make_uint4(0u, 0u, 0u, 0u);
    if (t0 + r < T && c0 + vv * 8 < C) val = __ldg(reinterpret_cast<const uint4*>(xb + static_cast<long long>(t0 + r) * ldx + c0 + vv * 8));
    *reinterpret_cast<uint4*>(&tile[r][vv * 8]) = val;
  }
  __syncthreads();
  for (int i = threadIdx.x; i < 64 * 8; i += 256) {  // 64 rows (c) x 8 vectors of 8 tokens
    const int r = i >> 3, vv = i & 7;
    if (c0 + r >= C || t0 + vv * 8 >= T) continue;
    __half o[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) o[e] = tile[vv * 8 + e][r];
    *reinterpret_cast<uint4*>(yb + static_cast<long long>(c0 + r) * T + t0 + vv * 8) = *reinterpret_cast<const uint4*>(o);
  }
}

}  // namespace
}  // namespace k2

using namespace k2;

extern "C" {

int k2_sn_apply(const void* x, int C, int ldx, int NB, int H, int W, int groups, const float* stats, const float* gamma,
                const float* beta, const float* zq, int zh, int zw, const float* sn_w, int act, void* y, int ldy,
                k2_stream_t stream) {
  K2_REQUIRE(x && y && stats && gamma && beta && zq && sn_w, "sn_apply: null pointer");
  K2_REQUIRE(C % 8 == 0 && C % groups == 0 && ldx % 8 == 0 && ldy % 8 == 0, "sn_apply: bad channel counts / strides");
  K2_REQUIRE(NB > 0 && H > 0 && W > 0 && zh > 0 && zw > 0 && NB <= 65535, "sn_apply: bad geometry");
  K2_REQUIRE(ldx >= C && ldy >= C, "sn_apply: row strides must be >= C");
  K2_REQUIRE(aligned16(x) && aligned16(y) && aligned16(zq), "sn_apply: x, y and zq must be 16-byte aligned");
  SnParams p;
  p.x = reinterpret_cast<const __half*>(x);
  p.C = C; p.ldx = ldx; p.NB = NB; p.H = H; p.W = W; p.groups = groups;
  p.stats = stats; p.gamma = gamma; p.beta = beta; p.zq = zq; p.zh = zh; p.zw = zw; p.sn_w = sn_w; p.act = act;
  p.y = reinterpret_cast<__half*>(y); p.ldy = ldy;
  p.zshift = -1;
  if (H % zh == 0 && W % zw == 0 && H / zh == W / zw) {
    const int sc = H / zh;
    if ((sc & (sc - 1)) == 0) {
      p.zshift = 0;
      while ((1 << p.zshift) < sc) ++p.zshift;
    }
  }
  const int ctiles = (C / 8 + VX - 1) / VX;
  const int HW = H * W;
  // 2 resident blocks per SM x 3 waves, each thread at least one full double-buffered iteration
  int chunks = (6 * num_sms()) / (ctiles * NB);
  const int max_chunks = (HW + UN * PY - 1) / (UN * PY);
  if (chunks > max_chunks) chunks = max_chunks;
  if (chunks < 1) chunks = 1;
  int chunk = (HW + chunks - 1) / chunks;
  chunk = (chunk + UN * PY - 1) / (UN * PY) * (UN * PY);
  p.chunk = chunk;
  dim3 grid((HW + chunk - 1) / chunk, ctiles, NB);
  K2_CHECK_CUDA(launch_k(sn_apply_kernel, grid, dim3(256), 0, static_cast<cudaStream_t>(stream), p));
  count_launch();
  return 0;
}

int k2_transpose_f16(const void* x, int ldx, void* y, int B, int T, int C, k2_stream_t stream) {
  K2_REQUIRE(x && y && B > 0 && T > 0 && C > 0, "transpose_f16: bad arguments");
  K2_REQUIRE(ldx % 8 == 0 && C % 8 == 0 && T % 8 == 0, "transpose_f16: T, C and the row stride must be multiples of 8");
  K2_REQUIRE((reinterpret_cast<uintptr_t>(x) & 15) == 0 && (reinterpret_cast<uintptr_t>(y) & 15) == 0, "transpose_f16: alignment");
  dim3 grid((T + 63) / 64, (C + 63) / 64, B);
  K2_CHECK_CUDA(launch_k(transpose_f16_kernel, grid, dim3(256), 0, static_cast<cudaStream_t>(stream),
                         reinterpret_cast<const __half*>(x), ldx, reinterpret_cast<__half*>(y), T, C));
  count_launch();
  return 0;
}

}  // extern "C"
