// k2_norm.cu -- GroupNorm statistics + fused normalise / FiLM / SiLU / resample / concat / SpatialNorm.
//
// Replaces (reference file:line):
//   GroupNorm32.forward                 kandinsky2/model/nn.py:31-37   (fp32 statistics, eps 1e-5, 32 groups)
//   ResBlock FiLM + SiLU                kandinsky2/model/unet.py:209-216
//   Upsample / Downsample (h_upd,x_upd) kandinsky2/model/unet.py:67-77,105-107,198-203
//   torch.cat([h, hs.pop()], 1)         kandinsky2/model/text2im_model2_1.py:99  (read as two sources)
//   SpatialNorm.forward                 kandinsky2/vqgan/movq_modules.py:61-68   (eps 1e-6)
//
// Both kernels are HBM-bound and organised the same way: a block is 16 channel-vectors (8 fp16 = 16 B each,
// so a half-warp covers 256 contiguous bytes of one pixel row) x 16 pixel lanes; it owns a 128-channel
// slab of a run of pixels of ONE image.  Everything per-channel (mean/rstd/gamma/beta/FiLM folded into one
// a*x+b) is computed once per thread and reused for every pixel of the run; the pixel loop keeps 4
// independent 16-byte loads in flight per thread.  stats reads the tensor once, apply reads it once and
// writes it once.  Statistics are reduced in a fixed order (no float atomics): results are bit-reproducible,
// which the multi-GPU == single-GPU test relies on.
#include "../../include/k2b200.h"
#include "k2_common.cuh"
#include "k2_internal.h"

namespace k2 {
namespace {

constexpr int VX = 16;   // channel vectors per block
constexpr int PY = 16;   // pixel lanes per block
constexpr int UNR = 4;   // loads in flight per thread (statistics)
constexpr int UNA = 4;   // vectors per thread per iteration (apply); two iterations are in flight

__device__ __forceinline__ const __half* src_ptr(const __half* s0, int C0, int ld0, const __half* s1, int ld1,
                                                 long long row, int c) {
  return (c < C0) ? (s0 + row * ld0 + c) : (s1 + row * ld1 + (c - C0));
}
__device__ __forceinline__ uint4 ldg16(const __half* p) { return __ldg(reinterpret_cast<const uint4*>(p)); }
__device__ __forceinline__ void unpack8(const uint4& raw, float (&f)[8]) {
  const __half2* h2 = reinterpret_cast<const __half2*>(&raw);
#pragma unroll
  for (int e = 0; e < 4; ++e) {
    float2 t = __half22float2(h2[e]);
    f[2 * e] = t.x;
    f[2 * e + 1] = t.y;
  }
}
__device__ __forceinline__ uint4 pack8(const float (&f)[8]) {
  uint4 ov;
  __half2* oh = reinterpret_cast<__half2*>(&ov);
#pragma unroll
  for (int e = 0; e < 4; ++e) oh[e] = __floats2half2_rn(f[2 * e], f[2 * e + 1]);
  return ov;
}

// ------------------------------------------------------------------------------------------------
// statistics: grid (chunks, channel tiles, images); per-channel partial sums -> last block of an image
// folds them into per-group mean / rstd in fp64, fixed order.
// ------------------------------------------------------------------------------------------------
// 4 resident blocks per SM: the wave pick_chunk sizes (the default register budget spills the fp64 fold)
__global__ void __launch_bounds__(256, 4) gn_stats_kernel(const __half* __restrict__ s0, int C0, int ld0,
                                                       const __half* __restrict__ s1, int C1, int ld1, int HW,
                                                       int groups, float eps, int chunk, float* __restrict__ stats,
                                                       float* __restrict__ partial, unsigned int* __restrict__ counters) {
  __shared__ float red[PY][VX][17];
  __shared__ bool is_last;
  const int C = C0 + C1;
  const int CV = C / 8;
  const int vx = threadIdx.x % VX;
  const int py = threadIdx.x / VX;
  const int v = blockIdx.y * VX + vx;
  const int n = blockIdx.z;
  const int chunks = gridDim.x;
  const int p0 = blockIdx.x * chunk;
  const int p1 = min(HW, p0 + chunk);
  pdl_wait();
  pdl_launch();
  // sums of d = x - pivot, pivot = the channel's value at the image's first pixel (every chunk reads the same one): d is of
  // the order of the channel's spread (exact in fp32 unless x and the pivot are more than ~12 binades apart), so the fp32 sums
  // of d and d^2 keep their precision whatever the mean
  float a[16];
#pragma unroll
  for (int e = 0; e < 16; ++e) a[e] = 0.f;
  if (v < CV) {
    const int c = v * 8;
    const __half* base = (c < C0) ? (s0 + c) : (s1 + (c - C0));
    const int ld = (c < C0) ? ld0 : ld1;
    const long long row0 = static_cast<long long>(n) * HW;
    float piv[8];
    unpack8(ldg16(base + row0 * ld), piv);
    int p = p0 + py;
    for (; p + (UNR - 1) * PY < p1; p += UNR * PY) {
      uint4 raw[UNR];
#pragma unroll
      for (int u = 0; u < UNR; ++u) raw[u] = ldg16(base + (row0 + p + u * PY) * ld);
#pragma unroll
      for (int u = 0; u < UNR; ++u) {
        float f[8];
        unpack8(raw[u], f);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float d = f[e] - piv[e];
          a[e] += d;
          a[8 + e] = fmaf(d, d, a[8 + e]);
        }
      }
    }
    for (; p < p1; p += PY) {
      float f[8];
      unpack8(ldg16(base + (row0 + p) * ld), f);
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        const float d = f[e] - piv[e];
        a[e] += d;
        a[8 + e] = fmaf(d, d, a[8 + e]);
      }
    }
  }
#pragma unroll
  for (int e = 0; e < 16; ++e) red[py][vx][e] = a[e];
  __syncthreads();
  // 256 threads = 16 vectors x 16 values: each sums its value over the 16 pixel lanes in lane order
  {
    const int e = threadIdx.x % 16, vv = threadIdx.x / 16;
    float s = 0.f;
#pragma unroll
    for (int q = 0; q < PY; ++q) s += red[q][vv][e];
    const int c = (blockIdx.y * VX + vv) * 8 + (e & 7);
    if (c < C)  // partial[n][chunk][c][0: sum, 1: sumsq]
      partial[((static_cast<long long>(n) * chunks + blockIdx.x) * C + c) * 2 + (e >> 3)] = s;
  }
  __threadfence();
  __syncthreads();
  if (threadIdx.x == 0) {
    const unsigned int total = gridDim.x * gridDim.y;
    unsigned int prev = atomicAdd(&counters[n], 1u);
    is_last = (prev == total - 1);
  }
  __syncthreads();
  if (!is_last) return;
  __threadfence();
  // fold: thread t -> group t/8, slice t%8 of that group's (chunk, channel) pairs; then a fixed-order shuffle sum.  In fp64,
  // every channel's sums are moved from its own pivot p_c to the group's K = p of its first channel:
  //   sum (x - K) = sum d + HW (p_c - K),   sum (x - K)^2 = sum d^2 + 2 (p_c - K) sum d + HW (p_c - K)^2
  const int cpg = C / groups;
  const double cnt = static_cast<double>(HW) * cpg;
  const float* pn = partial + static_cast<long long>(n) * chunks * C * 2;
  const long long row0 = static_cast<long long>(n) * HW;
  for (int g0 = 0; g0 < groups; g0 += 32) {
    const int g = g0 + threadIdx.x / 8;
    const int sub = threadIdx.x % 8;
    double s = 0.0, q = 0.0, K = 0.0;
    if (g < groups) {
      auto pivot = [&](int c) { return __half2float(*src_ptr(s0, C0, ld0, s1, ld1, row0, c)); };
      K = pivot(g * cpg);
      for (int j = sub; j < cpg; j += 8) {
        const double dk = static_cast<double>(pivot(g * cpg + j)) - K;
        s += HW * dk;
        q += HW * dk * dk;
      }
      const int items = chunks * cpg;
      int i = sub;
      for (; i + 56 < items; i += 64) {  // 8 independent loads in flight
        float2 t[8];
        float pc[8];
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          const int ii = i + 8 * u;
          const int ch = ii / cpg, c = g * cpg + (ii - ch * cpg);
          t[u] = __ldcg(reinterpret_cast<const float2*>(pn + (static_cast<long long>(ch) * C + c) * 2));
          pc[u] = pivot(c);
        }
#pragma unroll
        for (int u = 0; u < 8; ++u) {
          s += static_cast<double>(t[u].x);
          q += static_cast<double>(t[u].y) + 2.0 * (pc[u] - K) * t[u].x;
        }
      }
      for (; i < items; i += 8) {
        const int ch = i / cpg, c = g * cpg + (i - ch * cpg);
        const float2 t = __ldcg(reinterpret_cast<const float2*>(pn + (static_cast<long long>(ch) * C + c) * 2));
        s += static_cast<double>(t.x);
        q += static_cast<double>(t.y) + 2.0 * (static_cast<double>(pivot(c)) - K) * t.x;
      }
    }
#pragma unroll
    for (int o = 4; o > 0; o >>= 1) {
      s += __shfl_down_sync(0xffffffffu, s, o, 8);
      q += __shfl_down_sync(0xffffffffu, q, o, 8);
    }
    if (g < groups && sub == 0) {
      const double ms = s / cnt;
      const double mean = K + ms;
      double var = q / cnt - ms * ms;
      if (var < 0.0) var = 0.0;
      stats[(static_cast<long long>(n) * groups + g) * 2] = static_cast<float>(mean);
      stats[(static_cast<long long>(n) * groups + g) * 2 + 1] =
          static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
    }
  }
  if (threadIdx.x == 0) counters[n] = 0;  // ready for the next launch
}

// ------------------------------------------------------------------------------------------------
// finalize for statistics fused into the producing convolution's epilogue (k2_conv_gemm gn_partial):
// partial[(tile*4 + warp)][channel] = (sum, sumsq) over 32 output rows.  One block per (image, group): fixed-order
// fp64 fold over the image's row groups and the group's channels (which may span the two concatenated sources).
// ------------------------------------------------------------------------------------------------
constexpr int FIN_T = 512;  // the fold is latency-bound (short strided segments): many loads in flight per CTA
__global__ void __launch_bounds__(FIN_T) gn_finalize_kernel(const float2* __restrict__ part0, int C0, int rg0,
                                                          const float2* __restrict__ part1, int C1, int rg1, int HW,
                                                          int groups, float eps, float* __restrict__ stats) {
  __shared__ double red[2][FIN_T / 32];
  const int n = blockIdx.y, g = blockIdx.x;
  const int C = C0 + C1;
  const int cpg = C / groups;
  pdl_wait();
  pdl_launch();
  // 4 independent accumulator pairs per thread (loads in flight), fp64 from the first partial on: the partials are raw
  // (sum, sumsq) of x, so the variance q / cnt - mean^2 cancels, and fp32 accumulation error would be multiplied by (mean / std)^2
  double fs[4] = {0.0, 0.0, 0.0, 0.0}, fq[4] = {0.0, 0.0, 0.0, 0.0};
  // the group's channels [c_lo, c_hi) restricted to one source: part[(n*rgs + rg)][c - base]
  auto fold = [&](const float2* part, int Cs, int base, int rgs) {
    const int c_lo = max(g * cpg, base), c_hi = min((g + 1) * cpg, base + Cs);
    const int w = c_hi - c_lo;
    if (w <= 0) return;
    const int items = rgs * w;
    const float2* p0 = part + static_cast<long long>(n) * rgs * Cs + (c_lo - base);
    auto load = [&](int i) {
      const int rg = i / w;
      return __ldg(p0 + static_cast<long long>(rg) * Cs + (i - rg * w));
    };
    int i = threadIdx.x;
    for (; i + 3 * FIN_T < items; i += 4 * FIN_T) {
      float2 t[4];
#pragma unroll
      for (int u = 0; u < 4; ++u) t[u] = load(i + u * FIN_T);
#pragma unroll
      for (int u = 0; u < 4; ++u) {
        fs[u] += t[u].x;
        fq[u] += t[u].y;
      }
    }
    for (; i < items; i += FIN_T) {
      const float2 t = load(i);
      fs[0] += t.x;
      fq[0] += t.y;
    }
  };
  fold(part0, C0, 0, rg0);
  if (C1 > 0) fold(part1, C1, C0, rg1);
  double s = (fs[0] + fs[1]) + (fs[2] + fs[3]);
  double q = (fq[0] + fq[1]) + (fq[2] + fq[3]);
#pragma unroll
  for (int o = 16; o > 0; o >>= 1) {
    s += __shfl_down_sync(0xffffffffu, s, o);
    q += __shfl_down_sync(0xffffffffu, q, o);
  }
  if ((threadIdx.x & 31) == 0) {
    red[0][threadIdx.x >> 5] = s;
    red[1][threadIdx.x >> 5] = q;
  }
  __syncthreads();
  if (threadIdx.x == 0) {
    s = 0.0;
    q = 0.0;
#pragma unroll
    for (int w = 0; w < FIN_T / 32; ++w) {  // fixed order: deterministic
      s += red[0][w];
      q += red[1][w];
    }
    const double cnt = static_cast<double>(HW) * cpg;
    const double mean = s / cnt;
    double var = q / cnt - mean * mean;
    if (var < 0.0) var = 0.0;
    stats[(static_cast<long long>(n) * groups + g) * 2] = static_cast<float>(mean);
    stats[(static_cast<long long>(n) * groups + g) * 2 + 1] = static_cast<float>(1.0 / sqrt(var + static_cast<double>(eps)));
  }
}

// ------------------------------------------------------------------------------------------------
// apply
// ------------------------------------------------------------------------------------------------
struct ApplyParams {
  const __half* s0;
  const __half* s1;
  int C0, ld0, C1, ld1;
  int NB, H, W, groups;
  const float* stats;
  const float* gamma;
  const float* beta;
  const float* film;  // rows (scale | shift), stride film_ld, or null
  int film_ld;
  int act;
  __half* y;
  int ldy;
  __half* xres;
  int ldx;
  const float* zq;  // [NB, zh, zw, 4] or null
  int zh, zw;
  const float* sn_w;  // [C, 10]
  int chunk;          // work pixels per block
  // FOLD variant only (appended: the layout of everything above is what the validated kernels read)
  const float2* part0;  // producer partials [n][rg0][C0] (sum, sumsq), as for k2_gn_finalize
  const float2* part1;  // second source's partials [n][rg1][C1] or null
  int rg0, rg1;
  float eps;
};

// RESAMPLE 0: same size; 1: 2x2 average pool (work items = output pixels); 2: nearest 2x (work = input pixels)
// FOLD: the block derives mean / rstd of the groups it touches from the producers' partial sums itself (the work of
// k2_gn_finalize, redone per block: worthwhile where an image has few row groups -- levels 1-3 of the U with one partial per
// conv M tile -- because it removes a launch per GroupNorm).  Same fold as gn_finalize_kernel, warp-wide instead of block-wide.
constexpr int FOLD_MAXG = 66;  // groups one block of 128 channels can touch: 128 / 2 + 2 (at least 2 channels per group)
template <int RESAMPLE, bool SPATIAL, bool FOLD = false>
__global__ void __launch_bounds__(256) gn_apply_kernel(const ApplyParams p) {
  const int C = p.C0 + p.C1;
  const int CV = C / 8;
  const int vx = threadIdx.x % VX;
  const int py = threadIdx.x / VX;
  const int v = blockIdx.y * VX + vx;
  const int n = blockIdx.z;
  // Everything that the PREVIOUS kernel of the stream does not produce is fetched before griddepcontrol.wait, i.e. while that
  // kernel is still draining: gamma / beta are weights; launches <= N-2 of the stream are complete when launch N begins (every
  // kernel waits for its predecessor before it lets its successor start).  The FiLM rows come from a branch forked onto a side
  // stream (model/unet.py) and joined in by an event wait right before the first ResBlock's out-norm, which may be this kernel
  // (the folded variant).  That join acts as a full dependency, eagerly and as a captured graph, also when the launch after it
  // is a PDL launch: tests/test_gpu_pdl_plans.py holds the branch back and NaN-fills the FiLM rows before every run and
  // replay, and the output stays bit-identical to the serialised run (without the join, the same harness reads the NaN).
  // Reading the rows here relies on that.
  float ga8[8], be8[8], sc8[8], sh8[8];
  {
    const int cc = min(v, CV - 1) * 8;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      ga8[e] = __ldg(p.gamma + cc + e);
      be8[e] = __ldg(p.beta + cc + e);
      sc8[e] = p.film ? 1.f + __ldg(p.film + static_cast<long long>(n) * p.film_ld + cc + e) : 1.f;
      sh8[e] = p.film ? __ldg(p.film + static_cast<long long>(n) * p.film_ld + C + cc + e) : 0.f;
    }
  }
  pdl_wait();
  pdl_launch();
  __shared__ float2 s_fold[FOLD ? FOLD_MAXG : 1];
  int g_lo = 0;
  if constexpr (FOLD) {
    const int cpg = C / p.groups;
    const int c_lo = blockIdx.y * VX * 8;
    const int c_hi = min(C, c_lo + VX * 8);
    g_lo = c_lo / cpg;
    const int g_hi = (c_hi - 1) / cpg;
    const int warp = threadIdx.x >> 5, lane = threadIdx.x & 31;
    for (int g = g_lo + warp; g <= g_hi; g += 8) {
      double fs = 0.0, fq = 0.0;  // fp64 from the first partial on, as in gn_finalize_kernel
      auto fold = [&](const float2* part, int Cs, int base, int rgs) {
        const int lo = max(g * cpg, base), hi = min((g + 1) * cpg, base + Cs);
        const int w = hi - lo;
        if (w <= 0) return;
        const float2* p0 = part + static_cast<long long>(n) * rgs * Cs + (lo - base);
        auto load = [&](int i) {
          const int rg = i / w;
          return __ldg(p0 + static_cast<long long>(rg) * Cs + (i - rg * w));
        };
        const int items = rgs * w;
        int i = lane;
        for (; i + 7 * 32 < items; i += 8 * 32) {  // 8 loads in flight per lane: the fold is pure L2 latency
          float2 t[8];
#pragma unroll
          for (int u = 0; u < 8; ++u) t[u] = load(i + u * 32);
#pragma unroll
          for (int u = 0; u < 8; ++u) {
            fs += t[u].x;
            fq += t[u].y;
          }
        }
        for (; i < items; i += 32) {
          const float2 t = load(i);
          fs += t.x;
          fq += t.y;
        }
      };
      fold(p.part0, p.C0, 0, p.rg0);
      if (p.C1 > 0) fold(p.part1, p.C1, p.C0, p.rg1);
      double s = fs, q = fq;
#pragma unroll
      for (int o = 16; o > 0; o >>= 1) {
        s += __shfl_down_sync(0xffffffffu, s, o);
        q += __shfl_down_sync(0xffffffffu, q, o);
      }
      if (lane == 0) {
        const double cnt = static_cast<double>(p.H) * p.W * cpg;
        const double mean = s / cnt;
        double var = q / cnt - mean * mean;
        if (var < 0.0) var = 0.0;
        s_fold[g - g_lo] = make_float2(static_cast<float>(mean), static_cast<float>(1.0 / sqrt(var + static_cast<double>(p.eps))));
      }
    }
    __syncthreads();
  }
  if (v >= CV) return;
  const int c0 = v * 8;
  const int Hw = (RESAMPLE == 1) ? p.H / 2 : p.H;
  const int Ww = (RESAMPLE == 1) ? p.W / 2 : p.W;
  const int HWw = Hw * Ww;
  const int p0 = blockIdx.x * p.chunk;
  const int p1 = min(HWw, p0 + p.chunk);

  // per-thread affine: y = act(x * A + B), everything that does not depend on the pixel folded in
  float A[8], Bc[8];
  {
    const int cpg = C / p.groups;
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const int c = c0 + e;
      const int g = c / cpg;
      float2 st;
      if constexpr (FOLD) {
        st = s_fold[g - g_lo];
      } else {
        st = __ldg(reinterpret_cast<const float2*>(p.stats + (static_cast<long long>(n) * p.groups + g) * 2));
      }
      const float ga = ga8[e] * st.y;
      const float be = be8[e] - st.x * ga;
      A[e] = ga * sc8[e];
      Bc[e] = fmaf(be, sc8[e], sh8[e]);
    }
  }
  const __half* base = (c0 < p.C0) ? (p.s0 + c0) : (p.s1 + (c0 - p.C0));
  const int ld = (c0 < p.C0) ? p.ld0 : p.ld1;
  const long long img_in = static_cast<long long>(n) * p.H * p.W;

  // SpatialNorm: the modulation depends on the latent pixel under (yi, xi); a thread's consecutive pixels usually share
  // it (the feature map is up to 8x finer than the latent), so it is recomputed only when the latent pixel changes.
  float a8[8], b8[8];
  int last_z = -1;
#pragma unroll
  for (int e = 0; e < 8; ++e) {
    a8[e] = A[e];
    b8[e] = Bc[e];
  }
  auto transform = [&](const float (&f)[8], int yi, int xi, float (&o)[8]) {
    if (SPATIAL) {
      const int zy = (yi * p.zh) / p.H, zx = (xi * p.zw) / p.W;
      const int zi = zy * p.zw + zx;
      if (zi != last_z) {
        last_z = zi;
        const float4 z = __ldg(reinterpret_cast<const float4*>(p.zq + (static_cast<long long>(n) * p.zh * p.zw + zi) * 4));
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          const float* w = p.sn_w + static_cast<long long>(c0 + e) * 10;
          const float my = __ldg(w + 0) * z.x + __ldg(w + 1) * z.y + __ldg(w + 2) * z.z + __ldg(w + 3) * z.w + __ldg(w + 4);
          const float mb = __ldg(w + 5) * z.x + __ldg(w + 6) * z.y + __ldg(w + 7) * z.z + __ldg(w + 8) * z.w + __ldg(w + 9);
          a8[e] = A[e] * my;
          b8[e] = Bc[e] * my + mb;
        }
      }
    }
#pragma unroll
    for (int e = 0; e < 8; ++e) {
      const float t = fmaf(f[e], a8[e], b8[e]);
      o[e] = p.act ? silu_f(t) : t;
    }
  };

  if (RESAMPLE == 0 || RESAMPLE == 2) {
    // software-pipelined: the loads of iteration i+1 are in flight while iteration i is transformed and stored
    uint4 raw[UNA], nxt[UNA];
    auto load_set = [&](int pp, uint4 (&dst)[UNA]) {
#pragma unroll
      for (int u = 0; u < UNA; ++u) {
        const int q = pp + u;
        if (q < p1) dst[u] = ldg16(base + (img_in + q) * ld);
      }
    };
    int pp = p0 + py * UNA;
    if (pp < p1) load_set(pp, raw);
    for (; pp < p1; pp += UNA * PY) {
      const int npp = pp + UNA * PY;
      if (npp < p1) load_set(npp, nxt);
#pragma unroll
      for (int u = 0; u < UNA; ++u) {
        const int q = pp + u;
        if (q >= p1) break;
        float f[8], o[8];
        unpack8(raw[u], f);
        const int yi = q / p.W, xi = q - yi * p.W;
        transform(f, yi, xi, o);
        const uint4 ov = pack8(o);
        if (RESAMPLE == 0) {
          *reinterpret_cast<uint4*>(p.y + (img_in + q) * p.ldy + c0) = ov;
          if (p.xres) *reinterpret_cast<uint4*>(p.xres + (img_in + q) * p.ldx + c0) = raw[u];
        } else {
          const int Wo = p.W * 2;
#pragma unroll
          for (int dy = 0; dy < 2; ++dy)
#pragma unroll
            for (int dx = 0; dx < 2; ++dx) {
              const long long orow = (static_cast<long long>(n) * p.H * 2 + (2 * yi + dy)) * Wo + (2 * xi + dx);
              *reinterpret_cast<uint4*>(p.y + orow * p.ldy + c0) = ov;
              if (p.xres) *reinterpret_cast<uint4*>(p.xres + orow * p.ldx + c0) = raw[u];
            }
        }
      }
#pragma unroll
      for (int u = 0; u < UNA; ++u) raw[u] = nxt[u];
    }
  } else {
    // 2x2 average pool of act(norm(x)) and of raw x; work items are OUTPUT pixels
    for (int q = p0 + py; q < p1; q += PY) {
      const int yo = q / Ww, xo = q - yo * Ww;
      uint4 raw[4];
#pragma unroll
      for (int k = 0; k < 4; ++k)
        raw[k] = ldg16(base + (img_in + static_cast<long long>(2 * yo + (k >> 1)) * p.W + (2 * xo + (k & 1))) * ld);
      float acc[8], accx[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) acc[e] = accx[e] = 0.f;
#pragma unroll
      for (int k = 0; k < 4; ++k) {
        float f[8], o[8];
        unpack8(raw[k], f);
        transform(f, 2 * yo + (k >> 1), 2 * xo + (k & 1), o);
#pragma unroll
        for (int e = 0; e < 8; ++e) {
          // the reference rounds GN+SiLU to fp16 before AvgPool2d (nn.py:32, unet.py:199-200)
          acc[e] += __half2float(__float2half_rn(o[e]));
          accx[e] += f[e];
        }
      }
#pragma unroll
      for (int e = 0; e < 8; ++e) {
        acc[e] *= 0.25f;
        accx[e] *= 0.25f;
      }
      const long long orow = static_cast<long long>(n) * HWw + q;
      *reinterpret_cast<uint4*>(p.y + orow * p.ldy + c0) = pack8(acc);
      if (p.xres) *reinterpret_cast<uint4*>(p.xres + orow * p.ldx + c0) = pack8(accx);
    }
  }
}

// work pixels per block: `blocks_per_sm` blocks per SM in total, at least one pixel per lane.  For the apply kernels the
// caller passes the kernel's real occupancy (3 blocks of 256 threads at 80 registers): ONE full wave.  A fixed 4 per SM would
// ask for more blocks than there are resident slots, i.e. a second wave with one block per SM.
static int pick_chunk(int HW, int ctiles, int NB, int blocks_per_sm = 4) {
  const int target_blocks = blocks_per_sm * num_sms();
  // rounded DOWN: the grid must not exceed the resident slots by a few blocks (a short second wave leaves most SMs idle for
  // the whole of its duration)
  int chunks = target_blocks / (ctiles * NB);
  int max_chunks = (HW + PY - 1) / PY;
  if (chunks > max_chunks) chunks = max_chunks;
  if (chunks < 1) chunks = 1;
  int chunk = (HW + chunks - 1) / chunks;
  chunk = (chunk + PY - 1) / PY * PY;
  return chunk;
}

template <typename K>
static int apply_blocks_per_sm(K kernel) {
  const int forced = gn_apply_blocks_per_sm();  // tuning key 11 (0 = the kernel's occupancy)
  if (forced > 0) return forced;
  int occ = 0;
  if (cudaOccupancyMaxActiveBlocksPerMultiprocessor(&occ, kernel, 256, 0) != cudaSuccess || occ < 1) occ = 3;
  return occ;
}

}  // namespace
}  // namespace k2

using namespace k2;

extern "C" {

long long k2_gn_scratch_floats(int NB, int HW, int C) {
  // [0, 1024): one arrival counter per image (fixed location: they must stay zero between launches whatever
  // geometry the previous launch had); then per-(image, chunk, channel) partial (sum, sumsq) pairs.
  const int ctiles = (C / 8 + VX - 1) / VX;
  const int chunk = pick_chunk(HW, ctiles, NB);
  const int chunks = (HW + chunk - 1) / chunk;
  return 1024 + static_cast<long long>(NB) * chunks * C * 2;
}

int k2_gn_stats(const void* src0, int C0, int ld0, const void* src1, int C1, int ld1, int NB, int HW, int groups,
                float eps, float* stats, float* scratch, k2_stream_t stream) {
  const int C = C0 + C1;
  K2_REQUIRE(src0 && C0 > 0 && C0 % 8 == 0 && C1 % 8 == 0, "gn_stats: channels must be multiples of 8");
  K2_REQUIRE(C % groups == 0, "gn_stats: C % groups != 0");
  K2_REQUIRE(src1 || C1 == 0, "gn_stats: src1 null with C1 > 0");
  K2_REQUIRE(NB <= 1024, "gn_stats: at most 1024 images per launch");
  K2_REQUIRE(ld0 % 8 == 0 && ld0 >= C0 && (C1 == 0 || (ld1 % 8 == 0 && ld1 >= C1)),
             "gn_stats: row strides must be multiples of 8 elements and >= the channels");
  K2_REQUIRE(aligned16(src0) && aligned16(src1), "gn_stats: sources must be 16-byte aligned");
  K2_REQUIRE(stats && scratch, "gn_stats: null pointer");
  const int ctiles = (C / 8 + VX - 1) / VX;
  const int chunk = pick_chunk(HW, ctiles, NB);
  const int chunks = (HW + chunk - 1) / chunk;
  float* partial = scratch + 1024;
  unsigned int* counters = reinterpret_cast<unsigned int*>(scratch);  // zeroed once by the caller, self-resetting
  dim3 grid(chunks, ctiles, NB);
  K2_CHECK_CUDA(launch_k(gn_stats_kernel, grid, dim3(256), 0, static_cast<cudaStream_t>(stream),
                         reinterpret_cast<const __half*>(src0), C0, ld0, reinterpret_cast<const __half*>(src1), C1, ld1, HW,
                         groups, eps, chunk, stats, partial, counters));
  count_launch();
  return 0;
}

int k2_gn_finalize(const float* part0, int C0, int rg0, const float* part1, int C1, int rg1, int NB, int HW, int groups,
                   float eps, float* stats, k2_stream_t stream) {
  K2_REQUIRE(part0 && stats && C0 > 0 && (part1 || C1 == 0) && (C0 + C1) % groups == 0 && rg0 > 0 && (C1 == 0 || rg1 > 0),
             "gn_finalize: bad arguments");
  K2_REQUIRE(((reinterpret_cast<uintptr_t>(part0) | reinterpret_cast<uintptr_t>(part1)) & 7) == 0,
             "gn_finalize: partial buffers must be 8-byte aligned");
  dim3 grid(groups, NB);
  K2_CHECK_CUDA(launch_k(gn_finalize_kernel, grid, dim3(FIN_T), 0, static_cast<cudaStream_t>(stream),
                         reinterpret_cast<const float2*>(part0), C0, rg0, reinterpret_cast<const float2*>(part1), C1, rg1, HW,
                         groups, eps, stats));
  count_launch();
  return 0;
}

int k2_gn_apply(const void* src0, int C0, int ld0, const void* src1, int C1, int ld1, int NB, int H, int W,
                int groups, const float* stats, const float* gamma, const float* beta, const float* film, int film_ld,
                int act, int resample, void* y, int ldy, void* xres, int ldx, const float* zq, int zh, int zw,
                const float* sn_w, k2_stream_t stream) {
  const int C = C0 + C1;
  K2_REQUIRE(src0 && y && stats && gamma && beta, "gn_apply: null pointer");
  K2_REQUIRE(C0 % 8 == 0 && C1 % 8 == 0 && C % groups == 0, "gn_apply: bad channel counts");
  K2_REQUIRE(resample >= 0 && resample <= 2, "gn_apply: resample in {0,1,2}");
  K2_REQUIRE(resample != 1 || (H % 2 == 0 && W % 2 == 0), "gn_apply: avg-pool needs even H, W");
  K2_REQUIRE(!zq || sn_w, "gn_apply: zq without sn_w");
  K2_REQUIRE(src1 || C1 == 0, "gn_apply: src1 null with C1 > 0");
  K2_REQUIRE(ld0 % 8 == 0 && ld0 >= C0 && (C1 == 0 || (ld1 % 8 == 0 && ld1 >= C1)) && ldy % 8 == 0 && ldy >= C &&
                 (!xres || (ldx % 8 == 0 && ldx >= C)),
             "gn_apply: row strides must be multiples of 8 elements and >= the channels");
  K2_REQUIRE(aligned16(src0) && aligned16(src1) && aligned16(y) && aligned16(xres) && aligned16(zq),
             "gn_apply: x, y, xres and zq must be 16-byte aligned");
  ApplyParams p;
  p.s0 = reinterpret_cast<const __half*>(src0);
  p.s1 = reinterpret_cast<const __half*>(src1);
  p.C0 = C0; p.ld0 = ld0; p.C1 = C1; p.ld1 = ld1;
  p.NB = NB; p.H = H; p.W = W; p.groups = groups;
  p.stats = stats; p.gamma = gamma; p.beta = beta; p.film = film; p.film_ld = film_ld;
  p.act = act;
  p.y = reinterpret_cast<__half*>(y); p.ldy = ldy;
  p.xres = reinterpret_cast<__half*>(xres); p.ldx = ldx;
  p.zq = zq; p.zh = zh; p.zw = zw; p.sn_w = sn_w;
  p.part0 = nullptr; p.part1 = nullptr; p.rg0 = 0; p.rg1 = 0; p.eps = 0.f;  // FOLD variant only
  const int Hw = (resample == 1) ? H / 2 : H;
  const int Ww = (resample == 1) ? W / 2 : W;
  const int ctiles = (C / 8 + VX - 1) / VX;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  const bool sp = zq != nullptr;
  auto go = [&](auto kernel) -> cudaError_t {
    p.chunk = pick_chunk(Hw * Ww, ctiles, NB, apply_blocks_per_sm(kernel));
    dim3 grid((Hw * Ww + p.chunk - 1) / p.chunk, ctiles, NB);
    return launch_k(kernel, grid, dim3(256), 0, st, p);
  };
  if (resample == 0) {
    if (sp) K2_CHECK_CUDA(go(gn_apply_kernel<0, true>));
    else K2_CHECK_CUDA(go(gn_apply_kernel<0, false>));
  } else if (resample == 1) {
    if (sp) K2_CHECK_CUDA(go(gn_apply_kernel<1, true>));
    else K2_CHECK_CUDA(go(gn_apply_kernel<1, false>));
  } else {
    if (sp) K2_CHECK_CUDA(go(gn_apply_kernel<2, true>));
    else K2_CHECK_CUDA(go(gn_apply_kernel<2, false>));
  }
  K2_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

// Same launch as k2_gn_apply, statistics folded from the producers' partials inside the kernel (no k2_gn_finalize launch).
int k2_gn_apply_fold(const void* src0, int C0, int ld0, const void* src1, int C1, int ld1, int NB, int H, int W, int groups,
                     const float* part0, int rg0, const float* part1, int rg1, float eps, const float* gamma,
                     const float* beta, const float* film, int film_ld, int act, int resample, void* y, int ldy, void* xres,
                     int ldx, k2_stream_t stream) {
  const int C = C0 + C1;
  K2_REQUIRE(src0 && y && gamma && beta, "gn_apply_fold: null pointer");
  K2_REQUIRE(C0 % 8 == 0 && C1 % 8 == 0 && C % groups == 0 && C / groups >= 2, "gn_apply_fold: bad channel counts");
  K2_REQUIRE(resample >= 0 && resample <= 2, "gn_apply_fold: resample in {0,1,2}");
  K2_REQUIRE(resample != 1 || (H % 2 == 0 && W % 2 == 0), "gn_apply_fold: avg-pool needs even H, W");
  K2_REQUIRE(part0 && rg0 > 0 && (C1 == 0 || (src1 && part1 && rg1 > 0)), "gn_apply_fold: partial buffers");
  K2_REQUIRE(ld0 % 8 == 0 && ld0 >= C0 && (C1 == 0 || (ld1 % 8 == 0 && ld1 >= C1)) && ldy % 8 == 0 && ldy >= C &&
                 (!xres || (ldx % 8 == 0 && ldx >= C)),
             "gn_apply_fold: row strides must be multiples of 8 elements and >= the channels");
  K2_REQUIRE(aligned16(src0) && aligned16(src1) && aligned16(y) && aligned16(xres),
             "gn_apply_fold: x, y and xres must be 16-byte aligned");
  K2_REQUIRE(((reinterpret_cast<uintptr_t>(part0) | reinterpret_cast<uintptr_t>(part1)) & 7) == 0,
             "gn_apply_fold: partial buffers must be 8-byte aligned");
  ApplyParams p;
  p.s0 = reinterpret_cast<const __half*>(src0);
  p.s1 = reinterpret_cast<const __half*>(src1);
  p.C0 = C0; p.ld0 = ld0; p.C1 = C1; p.ld1 = ld1;
  p.NB = NB; p.H = H; p.W = W; p.groups = groups;
  p.stats = nullptr; p.gamma = gamma; p.beta = beta; p.film = film; p.film_ld = film_ld;
  p.act = act;
  p.y = reinterpret_cast<__half*>(y); p.ldy = ldy;
  p.xres = reinterpret_cast<__half*>(xres); p.ldx = ldx;
  p.zq = nullptr; p.zh = 0; p.zw = 0; p.sn_w = nullptr;
  p.part0 = reinterpret_cast<const float2*>(part0);
  p.part1 = reinterpret_cast<const float2*>(part1);
  p.rg0 = rg0; p.rg1 = rg1; p.eps = eps;
  const int Hw = (resample == 1) ? H / 2 : H;
  const int Ww = (resample == 1) ? W / 2 : W;
  const int ctiles = (C / 8 + VX - 1) / VX;
  cudaStream_t st = static_cast<cudaStream_t>(stream);
  auto go = [&](auto kernel) -> cudaError_t {
    p.chunk = pick_chunk(Hw * Ww, ctiles, NB, apply_blocks_per_sm(kernel));
    dim3 grid((Hw * Ww + p.chunk - 1) / p.chunk, ctiles, NB);
    return launch_k(kernel, grid, dim3(256), 0, st, p);
  };
  if (resample == 0) K2_CHECK_CUDA(go(gn_apply_kernel<0, false, true>));
  else if (resample == 1) K2_CHECK_CUDA(go(gn_apply_kernel<1, false, true>));
  else K2_CHECK_CUDA(go(gn_apply_kernel<2, false, true>));
  K2_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

}  // extern "C"
