// k2_conv_gemm.cu -- im2col-free 3x3 / 1x1 convolution and plain GEMM on sm_90a warpgroup MMA (wgmma) tensor cores.
//
// Replaces the cuDNN / cuBLAS call sites of the reference hot path:
//   nn.Conv2d 3x3   kandinsky2/model/unet.py:152,180,426,562 ; vqgan/movq_modules.py:139-148,268-270
//   nn.Conv2d 1x1   kandinsky2/model/unet.py:191 (skip_connection) ; movq_modules.py:150-157,188-199
//   nn.Conv1d k=1   kandinsky2/model/unet.py:251,257,258 (qkv / encoder_kv / proj_out)
//
// Formulation: D[M = pixels, N = Cout] = sum over (segment, tap, 64-channel chunk) A_tap[M, 64] * W[N, 64]^T.
//   * Activations are NHWC fp16. An M tile is a (TN x TH x TW) box of output pixels (<= 128 rows).
//     For tap (dy, dx) the A operand is the SAME box shifted by (dy, dx), fetched with ONE 4-D TMA
//     whose out-of-bounds elements are zero-filled by the hardware: conv padding costs nothing and no
//     im2col buffer exists in HBM or smem.
//   * Up to three A "segments" accumulate into the same accumulator tile: the 3x3 conv input plus 1x1 skip
//     inputs (raw x, optionally split in two for the un-materialised torch.cat of the up path). This is
//     how ResBlock's  skip_connection(x) + conv(h)  (unet.py:220) becomes a single kernel.
//   * Weights are pre-packed [Cout][K] fp16, K = concat over segments/taps/channels, loaded by 2-D TMA.
//   * Warp roles (384 threads): warpgroup 0 = TMA producer (one elected thread), warpgroups 1 and 2 = wgmma consumers, rows
//     [0, 64) and [64, 128) of the M tile: ONE m64nBNk16 per 16-element K step covers the whole N tile (BN = 16 ... 256), so
//     each warpgroup reads its A slice from shared memory once per K step, not once per 64 columns.  Both operands are K-major
//     in the 128 B-swizzled TMA tiles.  Persistent over tiles, smem ring of STAGES (A 16 KB + B BN*128 B).
//   * Epilogue: every consumer warp drains its own 16 accumulator rows from its registers (epilogue_warp), both warpgroups at
//     once: + bias (+ residual) -> fp16 rows, fp32 split-K partials or fp32 NCHW, plus the fused GroupNorm partial statistics,
//     through 2 KB of per-warp staging rather than a shared fp32 tile, so the shared memory goes to the operand ring.  The
//     producer keeps prefetching the next tile's operands meanwhile.
#include <stdio.h>

#include "k2_common.cuh"
#include "k2_internal.h"

namespace k2 {

namespace {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KB
constexpr int EPI_WARP_BYTES = 16 * 128;  // per consumer warp: its 16 accumulator rows x 128 B (64 fp16 / 32 fp32 columns)
constexpr int SMEM_LIMIT = 227 * 1024;    // sm_90 opt-in maximum per block

template <int BN>
struct Cfg {
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  static constexpr int EPI_BYTES = 8 * (EPI_WARP_BYTES + BN * 4);  // per consumer warp: staging rows + the N tile's bias
  static constexpr int BAR_BYTES = 256;
  static constexpr int FIXED = EPI_BYTES + BAR_BYTES + 1024;  // +1024 alignment slack
  static constexpr int STAGES = (SMEM_LIMIT - FIXED) / STAGE_BYTES > 6 ? 6 : (SMEM_LIMIT - FIXED) / STAGE_BYTES;
  static constexpr int SMEM_BYTES = STAGES * STAGE_BYTES + FIXED;
  static_assert(STAGES >= 2, "conv_gemm: shared memory does not hold two pipeline stages");
};

// up2 (3x3 conv over the nearest-2x upsampled source as four 2x2 phase convolutions): m_idx = phase * m_tiles_phase + box
// index; the box lives in SOURCE coordinates, `phase` = (a, b) = parity of the output pixel (2y + a, 2x + b).
__device__ __forceinline__ void decode_m_tile(const ConvGemmParams& p, int m_idx, int& n0, int& y0,
                                              int& x0, int& phase) {
  phase = 0;
  if (p.up2) {
    phase = m_idx / p.m_tiles_phase;
    m_idx -= phase * p.m_tiles_phase;
  }
  int tw_i = m_idx % p.tiles_w;
  int t = m_idx / p.tiles_w;
  int th_i = t % p.tiles_h;
  int tn_i = t / p.tiles_h;
  x0 = tw_i * p.TW;
  y0 = th_i * p.TH;
  n0 = tn_i * p.TN;
}

// ldmatrix.x4 kept in order with the shared-memory stores around it (the "memory" clobber)
__device__ __forceinline__ void ldsm_x4(uint32_t (&r)[4], uint32_t saddr) {
  asm volatile("ldmatrix.sync.aligned.m8n8.x4.shared.b16 {%0, %1, %2, %3}, [%4];"
               : "=r"(r[0]), "=r"(r[1]), "=r"(r[2]), "=r"(r[3])
               : "r"(saddr)
               : "memory");
}

// Epilogue of one consumer warp, rows [16 k, 16 k + 16) of the M tile (k = 4 g + w), straight from its m64nBN fragment
// (register 4 q + 2 h + e: row l / 4 + 8 h, column 8 q + 2 (l & 3) + e; `cbase` is the output column of column 0): + bias
// (+ residual) -> fp16 rows (out_mode 0), fp32 split-K partials (out_mode 2) or fp32 NCHW (out_mode 1), plus the fused
// GroupNorm partial statistics.  Both consumer warpgroups drain their own rows at the same time.
//
// In the fragment a warp store instruction covers 8 rows x 4 column pairs.  The fp16 and split-K paths therefore pass each
// 64-column (fp16) or 32-column (fp32) block through the warp's 16 x 128 B staging rows (16-byte pieces XOR-swizzled by the
// row): the residual comes in coalesced, 8 lanes per 128-byte row, and goes to the fragment layout with ldmatrix; the result
// goes back with stmatrix and out as 16-byte row pieces, 8 lanes per 128-byte line.  The bias is read from the warp's copy
// (`bsm`, columns cbase ..).  The GroupNorm statistics are column sums over the staged fp16 rows, summed in the order the
// partial formats have always used: 16 rows in row order per warp, then (gn_mode 1) warp pairs 2e, 2e + 1 folded for
// e = 0 .. 3 -- the only place where the two warpgroups meet.
template <int BN>
__device__ __forceinline__ void epilogue_warp(const ConvGemmParams& p, const float (&acc)[BN / 2], float* epi, uint32_t stg,
                                              const float* bsm, int k, int lane, int n0, int y0, int x0, int cbase, int split,
                                              int m_idx, int phase) {
  const int thw = p.TH * p.TW;
  // output row (pixel) of row `row` of the M tile, -1 outside the image; n, y, x: its image and source position
  auto out_row_of = [&](int row, int& n, int& y, int& x) -> long long {
    const int tn = row / thw;
    const int rem = row - tn * thw;
    const int th = rem / p.TW;
    const int tw = rem - th * p.TW;
    n = n0 + tn;
    y = y0 + th;
    x = x0 + tw;
    if (tn >= p.TN || n >= p.NB || y >= p.H || x >= p.W) return -1;
    return p.up2 ? (static_cast<long long>(n) * (2 * p.H) + (2 * y + (phase >> 1))) * (2 * p.W) + (2 * x + (phase & 1))
                 : (static_cast<long long>(n) * p.H + y) * p.W + x;
  };
  const int t4 = lane & 3, ra = lane >> 2;  // fragment rows ra, ra + 8; columns 8 q + 2 t4 + {0, 1}
  if constexpr (BN % 64 == 0) {
    if ((p.out_mode == 0 && p.Cout % 64 == 0) || (p.out_mode == 2 && p.Cout % 32 == 0)) {
      int n_, y_, x_;
      const int my_pix = static_cast<int>(out_row_of(16 * k + (lane & 15), n_, y_, x_));
      const int sub = lane >> 3, piece = lane & 7;
      int pix[4];  // pixel of the staged rows 4 i + sub this lane copies in and out
#pragma unroll
      for (int i = 0; i < 4; ++i) pix[i] = __shfl_sync(0xffffffffu, my_pix, 4 * i + sub);
      const bool va = __shfl_sync(0xffffffffu, my_pix, ra) >= 0, vb = __shfl_sync(0xffffffffu, my_pix, ra + 8) >= 0;
      auto row_addr = [&](int i) {
        const int rr = 4 * i + sub;
        return stg + rr * 128 + ((piece ^ (rr & 7)) << 4);
      };
      // ldmatrix / stmatrix: lanes 8 m .. 8 m + 7 address matrix m = (8-column group q + m / 2, row half m & 1)
      const int lrow = (lane & 7) + 8 * ((lane >> 3) & 1);
      auto frag_addr = [&](int q) { return stg + lrow * 128 + (((q + (lane >> 4)) ^ (lane & 7)) << 4); };
      if (p.out_mode == 2) {
        // split-K: raw fp32 partial sums [split][M][Cout] (bias / residual / statistics in the finalize pass)
        float* wsb = p.ws + static_cast<long long>(split) * p.M_total * p.Cout;
#pragma unroll
        for (int j = 0; j < BN / 32; ++j) {
          const int col0 = cbase + j * 32;
          if (col0 >= p.Cout) break;
#pragma unroll
          for (int q = 0; q < 4; ++q) {
#pragma unroll
            for (int h = 0; h < 2; ++h) {
              const int rr = ra + 8 * h;
              const int i = 16 * j + 4 * q + 2 * h;
              sts_v2(stg + rr * 128 + (((2 * q + (t4 >> 1)) ^ (rr & 7)) << 4) + ((t4 & 1) << 3), __float_as_uint(acc[i]),
                     __float_as_uint(acc[i + 1]));
            }
          }
          __syncwarp();
#pragma unroll
          for (int i = 0; i < 4; ++i) {
            const uint4 v4 = lds_v4(row_addr(i));
            if (pix[i] >= 0)
              *reinterpret_cast<uint4*>(wsb + static_cast<long long>(pix[i]) * p.Cout + col0 + piece * 4) = v4;
          }
          __syncwarp();
        }
        return;
      }
      constexpr int NP = BN / 64;
      // GroupNorm partial row groups stay image-major under up2: (box index) * 4 + phase
      const int m_in = p.up2 ? m_idx - phase * p.m_tiles_phase : m_idx;
      auto part_index = [&](long long base) { return p.up2 ? base * 4 + phase : base; };
      __half* outb = reinterpret_cast<__half*>(p.out);
      float4 st[NP];  // this warp's GroupNorm sums (sum, sumsq) of columns 2 l, 2 l + 1 of each 64-column block
      uint4 rpre[4];  // residual of the NEXT 64-column block, in flight while the current one is processed
      auto load_res = [&](int j) {
        const int c0 = cbase + j * 64;
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          rpre[i] = make_uint4(0u, 0u, 0u, 0u);
          if (pix[i] >= 0 && c0 < p.Cout)
            rpre[i] = *reinterpret_cast<const uint4*>(p.residual + static_cast<long long>(pix[i]) * p.ldr + c0 + piece * 8);
        }
      };
      if (p.residual) load_res(0);
#pragma unroll
      for (int j = 0; j < NP; ++j) {
        const int col0 = cbase + j * 64;
        st[j] = make_float4(0.f, 0.f, 0.f, 0.f);
        if (col0 >= p.Cout) continue;
        uint32_t res[16];  // residual pairs in fragment layout: [2 q + h]
        if (p.residual) {
#pragma unroll
          for (int i = 0; i < 4; ++i) sts_v4(row_addr(i), rpre[i].x, rpre[i].y, rpre[i].z, rpre[i].w);
          __syncwarp();
#pragma unroll
          for (int qq = 0; qq < 4; ++qq) {
            uint32_t r4[4];
            ldsm_x4(r4, frag_addr(2 * qq));
#pragma unroll
            for (int m = 0; m < 4; ++m) res[4 * qq + m] = r4[m];
          }
          if (j + 1 < NP) load_res(j + 1);
          __syncwarp();  // the staged residual is read before the result overwrites it
        }
        uint32_t o[16];
#pragma unroll
        for (int q = 0; q < 8; ++q) {
#pragma unroll
          for (int h = 0; h < 2; ++h) {
            float f0 = acc[32 * j + 4 * q + 2 * h], f1 = acc[32 * j + 4 * q + 2 * h + 1];
            if (p.bias) {
              const float2 b = *reinterpret_cast<const float2*>(bsm + j * 64 + 8 * q + 2 * t4);
              f0 += b.x;
              f1 += b.y;
            }
            if (p.residual) {
              const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&res[2 * q + h]));
              f0 += t.x;
              f1 += t.y;
            }
            const __half2 hh = __floats2half2_rn(f0, f1);
            o[2 * q + h] = (h ? vb : va) ? *reinterpret_cast<const uint32_t*>(&hh) : 0u;  // rows outside the image: zeros
          }
        }
#pragma unroll
        for (int qq = 0; qq < 4; ++qq) stmatrix_x4(frag_addr(2 * qq), o[4 * qq], o[4 * qq + 1], o[4 * qq + 2], o[4 * qq + 3]);
        __syncwarp();
#pragma unroll
        for (int i = 0; i < 4; ++i) {
          const uint4 v4 = lds_v4(row_addr(i));
          if (pix[i] >= 0) *reinterpret_cast<uint4*>(outb + static_cast<long long>(pix[i]) * p.ldo + col0 + piece * 8) = v4;
        }
        if (p.gn_part) {
          // statistics of the fp16-ROUNDED stored values: lane l sums columns 2 l, 2 l + 1 over the warp's 16 rows
          float4 hs = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int rr = 0; rr < 16; ++rr) {
            const uint32_t v = lds_u32(stg + rr * 128 + (((lane >> 2) ^ (rr & 7)) << 4) + ((lane & 3) << 2));
            const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&v));
            hs.x += t.x;
            hs.y = fmaf(t.x, t.x, hs.y);
            hs.z += t.y;
            hs.w = fmaf(t.y, t.y, hs.w);
          }
          if (p.gn_mode == 2) {
            // 16-pixel x 8-image tiles: warp k holds image n0 + k of spatial tile sp
            const int per = p.tiles_h * p.tiles_w;
            const int sp = m_in % per;
            const int img = n0 + k;
            if (k < p.TN && img < p.NB)
              *reinterpret_cast<float4*>(p.gn_part + part_index(static_cast<long long>(img) * per + sp) * p.Cout + col0 + 2 * lane) = hs;
          } else {
            st[j] = hs;
          }
        }
        __syncwarp();
      }
      if (p.gn_part && p.gn_mode == 1) {
        // one partial per (M tile, column): the eight warps' sums are folded in a fixed order through their (now idle)
        // staging rows, so k2_gn_finalize reads an eighth of what per-warp partials would cost
        float4* sums = reinterpret_cast<float4*>(epi);  // [warp][128]
#pragma unroll
        for (int j = 0; j < NP; ++j) sums[k * 128 + j * 32 + lane] = st[j];
        named_bar_sync(1, 256);
        if (k < NP && cbase + k * 64 < p.Cout) {
          float4 tot = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
          for (int e = 0; e < 4; ++e) {  // 32-row groups in row order: the sums of warps 2 e and 2 e + 1
            const float4 a = sums[(2 * e) * 128 + k * 32 + lane], b = sums[(2 * e + 1) * 128 + k * 32 + lane];
            tot.x += a.x + b.x;
            tot.y += a.y + b.y;
            tot.z += a.z + b.z;
            tot.w += a.w + b.w;
          }
          *reinterpret_cast<float4*>(p.gn_part + part_index(m_in) * p.Cout + cbase + k * 64 + 2 * lane) = tot;
        }
        named_bar_sync(1, 256);  // the sums are read before any warp stages the next tile
      }
      return;
    }
  }
  // element by element from the fragment: Cout not a multiple of 64 (fp16) / 32 (split-K), N tile 16, fp32 NCHW heads
  int n[2], y[2], x[2];
  long long orow[2];
#pragma unroll
  for (int h = 0; h < 2; ++h) orow[h] = out_row_of(16 * k + ra + 8 * h, n[h], y[h], x[h]);
#pragma unroll
  for (int q = 0; q < BN / 8; ++q) {
#pragma unroll
    for (int h = 0; h < 2; ++h) {
#pragma unroll
      for (int e = 0; e < 2; ++e) {
        const int col = cbase + 8 * q + 2 * t4 + e;
        if (orow[h] < 0 || col >= p.Cout) continue;
        float f = acc[4 * q + 2 * h + e];
        if (p.out_mode == 2) {
          p.ws[(static_cast<long long>(split) * p.M_total + orow[h]) * p.Cout + col] = f;
          continue;
        }
        if (p.bias) f += __ldg(p.bias + col);
        if (p.out_mode == 0) {
          if (p.residual) f += __half2float(p.residual[orow[h] * p.ldr + col]);
          reinterpret_cast<__half*>(p.out)[orow[h] * p.ldo + col] = __float2half_rn(f);
        } else {
          reinterpret_cast<float*>(p.out)[((static_cast<long long>(n[h]) * p.Cout + col) * p.H + y[h]) * p.W + x[h]] = f;
        }
      }
    }
  }
}


// WMAP: image n multiplies weight slab p.w_map[n] (k2_conv_gemm_wmap); otherwise slab n when p.w_batched, else the one
// weight matrix.  The flag only adds the map read, so the WMAP = false instances are the kernel as it was without it.
template <int BN, bool WMAP>
__global__ void __launch_bounds__(384, 1) conv_gemm_kernel(const __grid_constant__ ConvGemmParams p) {
  using C = Cfg<BN>;
  constexpr int NA = BN / 2;  // accumulator registers of the m64nBNk16 fragment
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  float* epi = reinterpret_cast<float*>(smem + C::STAGES * C::STAGE_BYTES);  // [8 warps][16 x 128 B], then [8 warps][BN] bias
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::STAGES * C::STAGE_BYTES + C::EPI_BYTES);
  uint64_t* empty_bar = full_bar + C::STAGES;

  const int warp_idx = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp_idx >> 2;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tmB);
    for (int s = 0; s < 3; ++s)
      if (p.seg_taps[s]) tma_prefetch_desc(&p.tmA[s]);
    for (int i = 0; i < C::STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);  // one arrival per consumer warp, after its wgmma.wait_group
    }
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_launch();

  // Tile order: N tile fastest.  The CTAs running at one time then cover SM count / n_tiles M tiles, all of whose N tiles, so
  // the source rows they re-read for every tap stay in L2.  With the M tile fastest they covered up to SM count M tiles:
  // for the 1536- and 1920-channel 48 x 48 convolutions that is 52-65 MB of source, more than the 50 MB L2, and every
  // tap's pass over the channel chunks came from HBM again.  In exchange the weights of all N tiles are live at once instead
  // of one N tile's (profiles/conv_layers.md lists the shapes that gain and lose).  Each tile computes exactly what it did,
  // so results are bit-identical.
  const int total_tiles = p.m_tiles * p.n_tiles * p.splits;

  if (wg == 0) {
    // ===================================== TMA producer =====================================
    setmaxnreg_dec<40>();
    if (warp_idx == 0 && elect_one()) {
      int stage = 0;
      uint32_t ring_phase = 0;
      const uint32_t tx_bytes = p.a_box_bytes + C::B_STAGE_BYTES;
      for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
        const int n_idx = tile % p.n_tiles;
        const int m_idx = (tile / p.n_tiles) % p.m_tiles;
        const int split = tile / (p.m_tiles * p.n_tiles);
        int n0, y0, x0, phase;
        decode_m_tile(p, m_idx, n0, y0, x0, phase);
        const int kb = phase * p.num_k_chunks;  // up2: each phase has its own 4-tap weight block
        const int k0 = split * p.k_per_split;
        const int k1 = min(p.num_k_chunks, k0 + p.k_per_split);
        // position (segment, tap, channel chunk) of flattened K chunk k0
        int s = 0, rem = k0;
        while (rem >= p.seg_taps[s] * p.seg_kchunks[s]) {
          rem -= p.seg_taps[s] * p.seg_kchunks[s];
          ++s;
        }
        int tap = rem / p.seg_kchunks[s];
        int c = rem - tap * p.seg_kchunks[s];
        // tiles never span images in batched mode (TN == 1); a slab index outside [0, n_slabs) loads TMA's zero fill
        int wslab = 0;
        if constexpr (WMAP) wslab = __ldg(p.w_map + n0);
        for (int kc = k0; kc < k1; ++kc) {
          const int taps = p.seg_taps[s];
          const int dy = (taps == 9) ? (tap / 3 - 1) : (taps == 4 ? (tap >> 1) + (phase >> 1) - 1 : 0);
          const int dx = (taps == 9) ? (tap % 3 - 1) : (taps == 4 ? (tap & 1) + (phase & 1) - 1 : 0);
          mbar_wait_lean(&empty_bar[stage], ring_phase ^ 1);
          uint8_t* sA = smem + stage * C::STAGE_BYTES;
          uint8_t* sB = sA + A_STAGE_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], tx_bytes);
          tma_load_4d(sA, &p.tmA[s], &full_bar[stage], c * BK, x0 + dx, y0 + dy, n0);
          tma_load_3d(sB, &p.tmB, &full_bar[stage], (kb + kc) * BK, n_idx * BN, WMAP ? wslab : (p.w_batched ? n0 : 0));
          if (++stage == C::STAGES) {
            stage = 0;
            ring_phase ^= 1;
          }
          if (++c == p.seg_kchunks[s]) {
            c = 0;
            if (++tap == taps) {
              tap = 0;
              ++s;
            }
          }
        }
      }
    }
  } else {
    // ============================ wgmma consumers + epilogue ================================
    setmaxnreg_inc<232>();
    const int g = wg - 1;          // accumulator rows [64 g, 64 g + 64)
    const int k = warp_idx - 4;    // consumer warp: rows 16 k .. 16 k + 15 of the M tile
    const uint32_t stg = smem_u32(epi) + k * EPI_WARP_BYTES;
    float* bsm = epi + 8 * EPI_WARP_BYTES / 4 + k * BN;
    int bias_cols = -1;  // output column of bsm[0]
    int stage = 0;
    uint32_t phase = 0;
    for (int tile = blockIdx.x; tile < total_tiles; tile += gridDim.x) {
      const int n_idx = tile % p.n_tiles;
      const int m_idx = (tile / p.n_tiles) % p.m_tiles;
      const int split = tile / (p.m_tiles * p.n_tiles);
      const int nk = min(p.num_k_chunks, (split + 1) * p.k_per_split) - split * p.k_per_split;
      float acc[NA];
#pragma unroll
      for (int i = 0; i < NA; ++i) acc[i] = 0.f;
      int prev_stage = -1;
      for (int kc = 0; kc < nk; ++kc) {
        mbar_wait_lean(&full_bar[stage], phase);  // no printf call: wgmma stays pipelined across the wait
        const uint32_t a_addr = smem_u32(smem + stage * C::STAGE_BYTES) + g * (64 * 128);
        const uint32_t b_addr = smem_u32(smem + stage * C::STAGE_BYTES + A_STAGE_BYTES);
        wgmma_fence();
#pragma unroll
        for (int ks = 0; ks < BK / 16; ++ks) {
          // +32 bytes (2 x 16 B units) per 16-element K step inside the 128 B swizzle row
          const uint64_t adesc = make_wgmma_desc(a_addr) + static_cast<uint64_t>(ks * 2);
          const uint64_t bdesc = make_wgmma_desc(b_addr) + static_cast<uint64_t>(ks * 2);
          if constexpr (BN == 256) {
            wgmma_m64n256k16(acc, adesc, bdesc, 1u);
          } else if constexpr (BN == 192) {
            wgmma_m64n192k16(acc, adesc, bdesc, 1u);
          } else if constexpr (BN == 128) {
            wgmma_m64n128k16(acc, adesc, bdesc, 1u);
          } else if constexpr (BN == 64) {
            wgmma_m64n64k16(acc, adesc, bdesc, 1u);
          } else {
            static_assert(BN == 16, "conv_gemm: N tile without a wgmma shape");
            wgmma_m64n16k16(acc, adesc, bdesc, 1u);
          }
        }
        wgmma_commit();
        // keep one K chunk in flight: the stage consumed by the previous chunk is free once only this one is pending
        wgmma_wait<1>();
        if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);
        prev_stage = stage;
        if (++stage == C::STAGES) {
          stage = 0;
          phase ^= 1;
        }
      }
      wgmma_wait<0>();
#pragma unroll
      for (int i = 0; i < NA; ++i) reg_fence(acc[i]);
      if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);  // an empty K range consumed no stage

      int n0, y0, x0, mphase;
      decode_m_tile(p, m_idx, n0, y0, x0, mphase);
      const int cbase = n_idx * BN;
      if (p.bias && cbase != bias_cols) {  // the warp's bias copy follows the N tile
        __syncwarp();
#pragma unroll
        for (int c = lane; c < BN; c += 32) bsm[c] = (cbase + c < p.Cout) ? __ldg(p.bias + cbase + c) : 0.f;
        __syncwarp();
        bias_cols = cbase;
      }
      epilogue_warp<BN>(p, acc, epi, stg, bsm, k, lane, n0, y0, x0, cbase, split, m_idx, mphase);
    }
  }
}

// split-K second pass: out[m, n] = fp16( sum_s ws[s][m][n] (fixed order) + bias[n] + residual[m, n] ).
// Block = 32 column vectors (256 channels) x 8 row lanes over 16 consecutive rows; optionally also emits the GroupNorm
// partial statistics of its 16 rows (same format as the conv epilogue's, 16-row groups) via a shared-memory fold.
__global__ void __launch_bounds__(256) splitk_finalize_kernel(const float* __restrict__ ws, int splits, long long M,
                                                              int Cout, const float* __restrict__ bias,
                                                              const __half* __restrict__ residual, int ldr,
                                                              __half* __restrict__ out, int ldo, float2* __restrict__ gn_part) {
  __shared__ float red[8][32][17];
  const int vx = threadIdx.x & 31, ry = threadIdx.x >> 5;
  const int c0 = (blockIdx.y * 32 + vx) * 8;
  const long long rg = blockIdx.x;
  pdl_wait();
  pdl_launch();
  float st[16];
#pragma unroll
  for (int e = 0; e < 16; ++e) st[e] = 0.f;
  if (c0 < Cout) {
    float bv[8];
#pragma unroll
    for (int e = 0; e < 8; ++e) bv[e] = bias ? __ldg(bias + c0 + e) : 0.f;
#pragma unroll
    for (int rr = 0; rr < 2; ++rr) {
      const long long m = rg * 16 + ry + rr * 8;
      if (m >= M) continue;
      float f[8];
#pragma unroll
      for (int e = 0; e < 8; ++e) f[e] = bv[e];
      for (int s = 0; s < splits; ++s) {
        const float4* w = reinterpret_cast<const float4*>(ws + (static_cast<long long>(s) * M + m) * Cout + c0);
        const float4 a = __ldcs(w), b = __ldcs(w + 1);
        f[0] += a.x; f[1] += a.y; f[2] += a.z; f[3] += a.w; f[4] += b.x; f[5] += b.y; f[6] += b.z; f[7] += b.w;
      }
      if (residual) {
        const uint4 rv = __ldg(reinterpret_cast<const uint4*>(residual + m * ldr + c0));
        const __half2* rh = reinterpret_cast<const __half2*>(&rv);
#pragma unroll
        for (int e = 0; e < 4; ++e) {
          const float2 t = __half22float2(rh[e]);
          f[2 * e] += t.x;
          f[2 * e + 1] += t.y;
        }
      }
      uint4 ov;
      __half2* oh = reinterpret_cast<__half2*>(&ov);
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        oh[e] = __floats2half2_rn(f[2 * e], f[2 * e + 1]);
        const float2 t = __half22float2(oh[e]);  // statistics of the ROUNDED values
        st[2 * e] += t.x;
        st[2 * e + 1] += t.y;
        st[8 + 2 * e] = fmaf(t.x, t.x, st[8 + 2 * e]);
        st[8 + 2 * e + 1] = fmaf(t.y, t.y, st[8 + 2 * e + 1]);
      }
      *reinterpret_cast<uint4*>(out + m * ldo + c0) = ov;
    }
  }
  if (gn_part == nullptr) return;
#pragma unroll
  for (int e = 0; e < 16; ++e) red[ry][vx][e] = st[e];
  __syncthreads();
  // thread -> (column vector vx2, channel e2 of it): sums the 8 row lanes in order
  const int vx2 = threadIdx.x >> 3, e2 = threadIdx.x & 7;
  const int c = (blockIdx.y * 32 + vx2) * 8 + e2;
  if (c < Cout) {
    float s1 = 0.f, s2 = 0.f;
#pragma unroll
    for (int q = 0; q < 8; ++q) {
      s1 += red[q][vx2][e2];
      s2 += red[q][vx2][8 + e2];
    }
    gn_part[rg * Cout + c] = make_float2(s1, s2);
  }
}


template <int BN, bool WMAP>
int launch_bn(const ConvGemmParams& p, cudaStream_t stream) {
  using C = Cfg<BN>;
  static bool attr_set = false;
  if (!attr_set) {
    K2_CHECK_CUDA(cudaFuncSetAttribute(conv_gemm_kernel<BN, WMAP>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       C::SMEM_BYTES));
    attr_set = true;
  }
  int total = p.m_tiles * p.n_tiles * p.splits;
  int grid = total < num_sms() ? total : num_sms();
  K2_CHECK_CUDA(launch_k(conv_gemm_kernel<BN, WMAP>, dim3(grid), dim3(384), C::SMEM_BYTES, stream, p));
  return 0;
}

template <bool WMAP>
int launch_wmap(const ConvGemmParams& p, int BN, cudaStream_t stream) {
  switch (BN) {
    case 16: return launch_bn<16, WMAP>(p, stream);
    case 64: return launch_bn<64, WMAP>(p, stream);
    case 128: return launch_bn<128, WMAP>(p, stream);
    case 192: return launch_bn<192, WMAP>(p, stream);
    case 256: return launch_bn<256, WMAP>(p, stream);
    default: return fail("conv_gemm: unsupported BN");
  }
}

}  // namespace

int launch_splitk_finalize(const float* ws, int splits, long long M, int Cout, const float* bias, const __half* residual,
                           int ldr, __half* out, int ldo, float2* gn_part, cudaStream_t stream) {
  dim3 grid(static_cast<unsigned int>((M + 15) / 16), (Cout / 8 + 31) / 32);
  K2_CHECK_CUDA(launch_k(splitk_finalize_kernel, grid, dim3(256), 0, stream, ws, splits, M, Cout, bias, residual, ldr, out, ldo,
                         gn_part));
  return 0;
}

int launch_conv_gemm(const ConvGemmParams& p, int BN, cudaStream_t stream) {
  return p.w_map ? launch_wmap<true>(p, BN, stream) : launch_wmap<false>(p, BN, stream);
}

}  // namespace k2
