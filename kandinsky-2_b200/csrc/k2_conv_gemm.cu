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
//   * Epilogue: the consumers park their register accumulators, BNC columns at a time, in a shared-memory tile with one fp32
//     row per output pixel; the epilogue warps then read it one ROW per thread (warp ew of a set owns rows [32 ew, 32 ew + 32))
//     -> + bias (+ residual) -> fp16 rows, fp32 split-K partials or fp32 NCHW, plus the fused GroupNorm partial statistics.
//     The producer keeps prefetching the next tile's operands meanwhile.
#include <stdio.h>

#include "k2_common.cuh"
#include "k2_internal.h"

namespace k2 {

namespace {

constexpr int BM = 128;
constexpr int BK = 64;
constexpr int A_STAGE_BYTES = BM * BK * 2;  // 16 KB
constexpr int ACC_PAD = 4;                  // fp32 row pitch BNC + 4: row-per-thread float4 reads hit distinct banks

constexpr int EPI_STAGE_FLOATS = 32 * 33;              // per-warp staging: 4224 B (4096 used)
constexpr int EPI_BYTES = 4 * EPI_STAGE_FLOATS * 4 + 4 * 256 * 4;  // + per-warp bias copy (<= 256 columns)
constexpr int SMEM_LIMIT = 227 * 1024;                 // sm_90 opt-in maximum per block

// ES = number of epilogue warp SETS (each set = 4 warps covering the 128 accumulator rows).  ES = 1: the warps of consumer
// warpgroup 0; ES = 2: both consumer warpgroups, set `es` handling the 64-column pairs jp with jp % 2 == es of a staged pass.
template <int BN, int ES>
struct Cfg {
  static constexpr int B_STAGE_BYTES = BN * BK * 2;
  static constexpr int STAGE_BYTES = A_STAGE_BYTES + B_STAGE_BYTES;
  // columns staged per epilogue pass: 64 (one pass per 64-column block); 128 with two epilogue sets so that both have work
  static constexpr int BNC = (BN < 64) ? BN : (ES == 2 ? 128 : 64);
  static_assert(ES == 1 || BN % 128 == 0, "two epilogue sets need N tiles of 128 or 256");
  static constexpr int ACC_BYTES = BM * (BNC + ACC_PAD) * 4;
  static constexpr int BAR_BYTES = 256;
  static constexpr int FIXED = ACC_BYTES + ES * EPI_BYTES + BAR_BYTES + 1024;  // +1024 alignment slack
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

// N consecutive fp32 of a staged accumulator row, as raw bits
template <int N>
__device__ __forceinline__ void acc_ld(const float* src, uint32_t (&r)[N]) {
#pragma unroll
  for (int v = 0; v < N / 4; ++v) {
    const float4 t = *reinterpret_cast<const float4*>(src + 4 * v);
    r[4 * v] = __float_as_uint(t.x);
    r[4 * v + 1] = __float_as_uint(t.y);
    r[4 * v + 2] = __float_as_uint(t.z);
    r[4 * v + 3] = __float_as_uint(t.w);
  }
}

// Epilogue of one (128-row x BN-column) pass of an accumulator tile staged in shared memory (`acc`, pitch BN + ACC_PAD):
// + bias (+ residual) -> fp16 rows (out_mode 0), fp32 split-K partials (out_mode 2) or fp32 NCHW (out_mode 1).  `cbase` is
// the output column of staged column 0.
//
// A thread owns one accumulator ROW, so storing straight from registers makes every warp store touch 32 different cache
// lines with 16 bytes each (and every residual load likewise): with short K loops (the attention qkv / proj GEMMs, 12..24
// chunks) that epilogue, not the tensor core, sets the pace.  The fp16 / split-K paths therefore go through a per-warp
// shared-memory transpose (32 rows x 128 B, 16-byte pieces XOR-swizzled by the row): registers -> smem by row, smem -> global
// with 8 lanes per row, i.e. 4 complete 128-byte lines per store instruction; the residual comes in the same way (coalesced
// load -> smem -> own row), the bias is read as broadcast LDS.128 from a per-warp copy, and the fused GroupNorm statistics
// are column sums over the staged fp16 tile.
template <int BN, int ES>
__device__ __forceinline__ void epilogue_tile(const ConvGemmParams& p, const float* acc, int ew, int lane, int n0, int y0,
                                              int x0, int cbase, int split, int m_idx, float* stat_smem, int es_arg,
                                              int phase) {
  const int es = (ES == 1) ? 0 : es_arg;
  const int row = ew * 32 + lane;
  const int thw = p.TH * p.TW;
  constexpr int CH = (BN >= 32) ? 32 : 16;  // columns per staged-accumulator read
  const float* arow = acc + row * (BN + ACC_PAD);  // this thread's accumulator row
      const int tn = row / thw;
      const int rem = row - tn * thw;
      const int th = rem / p.TW;
      const int tw = rem - th * p.TW;
      const int n = n0 + tn, y = y0 + th, x = x0 + tw;
      const bool valid = (tn < p.TN) && (n < p.NB) && (y < p.H) && (x < p.W);
      const long long out_row = p.up2 ? (static_cast<long long>(n) * (2 * p.H) + (2 * y + (phase >> 1))) * (2 * p.W) + (2 * x + (phase & 1))
                                      : (static_cast<long long>(n) * p.H + y) * p.W + x;
      // GroupNorm partial row groups stay image-major under up2: (box index) * 4 + phase
      const int m_in = p.up2 ? m_idx - phase * p.m_tiles_phase : m_idx;
      auto part_index = [&](long long base) { return p.up2 ? base * 4 + phase : base; };
      if constexpr (BN % 64 == 0) {
        if ((p.out_mode == 0 && p.Cout % 64 == 0) || (p.out_mode == 2 && p.Cout % 32 == 0)) {
          const uint32_t stage = smem_u32(stat_smem + (es * 4 + ew) * EPI_STAGE_FLOATS);  // [32 rows][8 x 16 B], piece ^= row & 7
          float* bsm = stat_smem + 4 * ES * EPI_STAGE_FLOATS + (es * 4 + ew) * 256;
          const int my_pix = valid ? static_cast<int>(out_row) : -1;
          const int sub = lane >> 3, piece = lane & 7;
          int pix[8];  // pixel (output row) of the 8 staged rows this lane copies out: rows i*4 + sub
#pragma unroll
          for (int i = 0; i < 8; ++i) pix[i] = __shfl_sync(0xffffffffu, my_pix, i * 4 + sub);
          const uint32_t own = stage + lane * 128;
          if (p.out_mode == 2) {
            // split-K: raw fp32 partial sums [split][M][Cout] (bias / residual / statistics in the finalize pass)
            float* wsb = p.ws + static_cast<long long>(split) * p.M_total * p.Cout;
#pragma unroll 1
            for (int j = 0; j < BN / 32; ++j) {
              const int col0 = cbase + j * 32;
              if (col0 >= p.Cout) break;
              if constexpr (ES > 1) {
                if ((j % ES) != es) continue;
              }
              uint32_t r[32];
              acc_ld(arow + j * 32, r);
#pragma unroll
              for (int v = 0; v < 8; ++v)
                sts_v4(own + ((v ^ (lane & 7)) << 4), r[v * 4], r[v * 4 + 1], r[v * 4 + 2], r[v * 4 + 3]);
              __syncwarp();
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const int rr = i * 4 + sub;
                const uint4 v4 = lds_v4(stage + rr * 128 + ((piece ^ (rr & 7)) << 4));
                if (pix[i] >= 0)
                  *reinterpret_cast<uint4*>(wsb + static_cast<long long>(pix[i]) * p.Cout + col0 + piece * 4) = v4;
              }
              __syncwarp();
            }
            return;
          }
          constexpr int NP = BN / 64;
          if (p.bias) {
#pragma unroll
            for (int c = lane; c < BN; c += 32) bsm[c] = (cbase + c < p.Cout) ? __ldg(p.bias + cbase + c) : 0.f;
            __syncwarp();
          }
          __half* outb = reinterpret_cast<__half*>(p.out);
          float4 st[NP];   // fused GroupNorm statistics of this warp's 32 rows: (sum, sumsq) of columns 2l, 2l+1 per pair
          uint4 rpre[8];   // residual of the NEXT 64-column pair, in flight while the current one is processed
          auto load_res = [&](int jp) {
            const int c0 = cbase + jp * 64;
#pragma unroll
            for (int i = 0; i < 8; ++i) {
              rpre[i] = make_uint4(0u, 0u, 0u, 0u);
              if (pix[i] >= 0 && c0 < p.Cout)
                rpre[i] = *reinterpret_cast<const uint4*>(p.residual + static_cast<long long>(pix[i]) * p.ldr + c0 + piece * 8);
            }
          };
          if constexpr (ES == 1) {
            if (p.residual) load_res(0);
          }
#pragma unroll
          for (int jp = 0; jp < NP; ++jp) {
            const int col0 = cbase + jp * 64;
            st[jp] = make_float4(0.f, 0.f, 0.f, 0.f);
            if (col0 < p.Cout && (ES == 1 || (jp % ES) == es)) {
              if constexpr (ES > 1) {
                if (p.residual) load_res(jp);  // no prefetch registers: the second warp set hides the latency instead
              }
              if (p.residual) {  // coalesced: 8 lanes x 16 B per row, 4 rows per instruction -> staged by row
#pragma unroll
                for (int i = 0; i < 8; ++i) {
                  const int rr = i * 4 + sub;
                  sts_v4(stage + rr * 128 + ((piece ^ (rr & 7)) << 4), rpre[i].x, rpre[i].y, rpre[i].z, rpre[i].w);
                }
                __syncwarp();
              }
              if constexpr (ES == 1) {
                if (p.residual && jp + 1 < NP) load_res(jp + 1);
              }
#pragma unroll
              for (int v = 0; v < 8; ++v) {  // 8 columns = one 16-byte piece of the staged row
                // read per piece: the unread part of the register accumulator is still live while the first passes of a
                // 256-column tile drain
                uint32_t r[8];
                acc_ld(arow + jp * 64 + v * 8, r);
                float f[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) f[e] = __uint_as_float(r[e]);
                if (p.bias) {
                  const float4 b0 = *reinterpret_cast<const float4*>(bsm + jp * 64 + v * 8);
                  const float4 b1 = *reinterpret_cast<const float4*>(bsm + jp * 64 + v * 8 + 4);
                  f[0] += b0.x; f[1] += b0.y; f[2] += b0.z; f[3] += b0.w;
                  f[4] += b1.x; f[5] += b1.y; f[6] += b1.z; f[7] += b1.w;
                }
                const uint32_t slot = own + ((v ^ (lane & 7)) << 4);
                if (p.residual) {
                  const uint4 rv = lds_v4(slot);
                  const __half2* rh = reinterpret_cast<const __half2*>(&rv);
#pragma unroll
                  for (int e = 0; e < 4; ++e) {
                    const float2 t = __half22float2(rh[e]);
                    f[2 * e] += t.x;
                    f[2 * e + 1] += t.y;
                  }
                }
                uint32_t o[4];
#pragma unroll
                for (int e = 0; e < 4; ++e) {
                  const __half2 hh = __floats2half2_rn(f[2 * e], f[2 * e + 1]);
                  o[e] = valid ? *reinterpret_cast<const uint32_t*>(&hh) : 0u;  // rows outside the image count as zeros
                }
                sts_v4(slot, o[0], o[1], o[2], o[3]);
              }
              __syncwarp();
#pragma unroll
              for (int i = 0; i < 8; ++i) {
                const int rr = i * 4 + sub;
                const uint4 v4 = lds_v4(stage + rr * 128 + ((piece ^ (rr & 7)) << 4));
                if (pix[i] >= 0)
                  *reinterpret_cast<uint4*>(outb + static_cast<long long>(pix[i]) * p.ldo + col0 + piece * 8) = v4;
              }
              if (p.gn_part) {
                // statistics of the fp16-ROUNDED stored values: lane l sums columns 2l, 2l+1 over the warp's rows
                float4 h0 = make_float4(0.f, 0.f, 0.f, 0.f), h1 = make_float4(0.f, 0.f, 0.f, 0.f);  // rows 0-15 / 16-31
#pragma unroll
                for (int rr = 0; rr < 32; ++rr) {
                  const uint32_t w = lds_u32(stage + rr * 128 + (((lane >> 2) ^ (rr & 7)) << 4) + ((lane & 3) << 2));
                  const float2 t = __half22float2(*reinterpret_cast<const __half2*>(&w));
                  float4& hacc = (rr < 16) ? h0 : h1;
                  hacc.x += t.x;
                  hacc.y = fmaf(t.x, t.x, hacc.y);
                  hacc.z += t.y;
                  hacc.w = fmaf(t.y, t.y, hacc.w);
                }
                if (p.gn_mode == 2) {
                  // 16-pixel x 8-image tiles: half warp h of warp ew holds image n0 + 2*ew + h of spatial tile sp
                  const int per = p.tiles_h * p.tiles_w;
                  const int sp = m_in % per;
                  const int img = n0 + 2 * ew;
                  if (2 * ew < p.TN && img < p.NB)
                    *reinterpret_cast<float4*>(p.gn_part + part_index(static_cast<long long>(img) * per + sp) * p.Cout + col0 + 2 * lane) = h0;
                  if (2 * ew + 1 < p.TN && img + 1 < p.NB)
                    *reinterpret_cast<float4*>(p.gn_part + part_index(static_cast<long long>(img + 1) * per + sp) * p.Cout + col0 + 2 * lane) = h1;
                } else {
                  st[jp] = make_float4(h0.x + h1.x, h0.y + h1.y, h0.z + h1.z, h0.w + h1.w);
                }
              }
              __syncwarp();
            }
          }
          if (p.gn_part && p.gn_mode == 1) {
            // one partial per (M tile, column): the four warps' sums are folded in a fixed order through the (now idle)
            // staging buffers, so k2_gn_finalize reads a quarter of what per-warp partials would cost
            if constexpr (ES == 1) {
              float4* mine = reinterpret_cast<float4*>(stat_smem + ew * EPI_STAGE_FLOATS);
#pragma unroll
              for (int jp = 0; jp < NP; ++jp) mine[jp * 32 + lane] = st[jp];
              named_bar_sync(1, 128);
              if (ew < NP) {
                const int col0 = cbase + ew * 64;
                if (col0 < p.Cout) {
                  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                  for (int w = 0; w < 4; ++w) {
                    const float4 t = reinterpret_cast<const float4*>(stat_smem + w * EPI_STAGE_FLOATS)[ew * 32 + lane];
                    acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w;
                  }
                  *reinterpret_cast<float4*>(p.gn_part + part_index(m_in) * p.Cout + col0 + 2 * lane) = acc;
                }
              }
              named_bar_sync(1, 128);
            } else {
              // each warp set folds the pairs it owns (jp % ES == es) among its own four warps: barrier 1 + es
              float4* mine = reinterpret_cast<float4*>(stat_smem + (es * 4 + ew) * EPI_STAGE_FLOATS);
#pragma unroll
              for (int jp = 0; jp < NP; ++jp) mine[jp * 32 + lane] = st[jp];
              named_bar_sync(1 + es, 128);
              const int jp_f = es + ew * ES;  // warp ew of the set folds the set's ew-th pair
              if (jp_f < NP) {
                const int col0 = cbase + jp_f * 64;
                if (col0 < p.Cout) {
                  float4 acc = make_float4(0.f, 0.f, 0.f, 0.f);
#pragma unroll
                  for (int w = 0; w < 4; ++w) {
                    const float4 t =
                        reinterpret_cast<const float4*>(stat_smem + (es * 4 + w) * EPI_STAGE_FLOATS)[jp_f * 32 + lane];
                    acc.x += t.x; acc.y += t.y; acc.z += t.z; acc.w += t.w;
                  }
                  *reinterpret_cast<float4*>(p.gn_part + part_index(m_in) * p.Cout + col0 + 2 * lane) = acc;
                }
              }
              named_bar_sync(1 + es, 128);
            }
          }
          return;
        }
      }
#pragma unroll 1
      for (int j = 0; j < BN / CH; ++j) {
        uint32_t r[CH];
        acc_ld(arow + j * CH, r);
        const int col0 = cbase + j * CH;
        if (valid && col0 < p.Cout) {
          if (p.out_mode == 2) {
            // split-K: raw fp32 partial sums [split][M][Cout] into the workspace (bias/residual in the finalize pass)
            float* w = p.ws + (static_cast<long long>(split) * p.M_total + out_row) * p.Cout + col0;
            if (col0 + CH <= p.Cout) {
#pragma unroll
              for (int v = 0; v < CH / 4; ++v)
                *reinterpret_cast<uint4*>(w + v * 4) = make_uint4(r[v * 4], r[v * 4 + 1], r[v * 4 + 2], r[v * 4 + 3]);
            } else {
#pragma unroll
              for (int e = 0; e < CH; ++e)
                if (col0 + e < p.Cout) w[e] = __uint_as_float(r[e]);
            }
          } else if (p.out_mode == 0) {
            __half* orow = reinterpret_cast<__half*>(p.out) + out_row * p.ldo + col0;
            const __half* rrow = p.residual ? p.residual + out_row * p.ldr + col0 : nullptr;
            if (col0 + CH <= p.Cout) {
#pragma unroll
              for (int v = 0; v < CH / 8; ++v) {
                float f[8];
#pragma unroll
                for (int e = 0; e < 8; ++e) {
                  f[e] = __uint_as_float(r[v * 8 + e]);
                  if (p.bias) f[e] += __ldg(p.bias + col0 + v * 8 + e);
                }
                if (rrow) {
                  uint4 rv = *reinterpret_cast<const uint4*>(rrow + v * 8);
                  const __half2* rh = reinterpret_cast<const __half2*>(&rv);
#pragma unroll
                  for (int e = 0; e < 4; ++e) {
                    float2 t = __half22float2(rh[e]);
                    f[2 * e] += t.x;
                    f[2 * e + 1] += t.y;
                  }
                }
                uint4 ov;
                __half2* oh = reinterpret_cast<__half2*>(&ov);
#pragma unroll
                for (int e = 0; e < 4; ++e) oh[e] = __floats2half2_rn(f[2 * e], f[2 * e + 1]);
                *reinterpret_cast<uint4*>(orow + v * 8) = ov;
              }
            } else {
#pragma unroll
              for (int e = 0; e < CH; ++e) {
                if (col0 + e < p.Cout) {
                  float f = __uint_as_float(r[e]);
                  if (p.bias) f += __ldg(p.bias + col0 + e);
                  if (rrow) f += __half2float(rrow[e]);
                  orow[e] = __float2half_rn(f);
                }
              }
            }
          } else {
            // fp32 NCHW (UNet / MoVQ output heads)
            float* o = reinterpret_cast<float*>(p.out);
#pragma unroll
            for (int e = 0; e < CH; ++e) {
              if (col0 + e < p.Cout) {
                float f = __uint_as_float(r[e]);
                if (p.bias) f += __ldg(p.bias + col0 + e);
                o[((static_cast<long long>(n) * p.Cout + (col0 + e)) * p.H + y) * p.W + x] = f;
              }
            }
          }
        }
      }
}


template <int BN, int ES>
__global__ void __launch_bounds__(384, 1) conv_gemm_kernel(const __grid_constant__ ConvGemmParams p) {
  using C = Cfg<BN, ES>;
  constexpr int BNC = C::BNC;
  constexpr int NA = BN / 2;  // accumulator registers of the m64nBNk16 fragment
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) &
                                             ~static_cast<uintptr_t>(1023));
  float* acc_smem = reinterpret_cast<float*>(smem + C::STAGES * C::STAGE_BYTES);
  float* stat_smem = reinterpret_cast<float*>(smem + C::STAGES * C::STAGE_BYTES + C::ACC_BYTES);
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(smem + C::STAGES * C::STAGE_BYTES + C::ACC_BYTES + ES * EPI_BYTES);
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
        for (int kc = k0; kc < k1; ++kc) {
          const int taps = p.seg_taps[s];
          const int dy = (taps == 9) ? (tap / 3 - 1) : (taps == 4 ? (tap >> 1) + (phase >> 1) - 1 : 0);
          const int dx = (taps == 9) ? (tap % 3 - 1) : (taps == 4 ? (tap & 1) + (phase & 1) - 1 : 0);
          mbar_wait_lean(&empty_bar[stage], ring_phase ^ 1);
          uint8_t* sA = smem + stage * C::STAGE_BYTES;
          uint8_t* sB = sA + A_STAGE_BYTES;
          mbar_arrive_expect_tx(&full_bar[stage], tx_bytes);
          tma_load_4d(sA, &p.tmA[s], &full_bar[stage], c * BK, x0 + dx, y0 + dy, n0);
          tma_load_3d(sB, &p.tmB, &full_bar[stage], (kb + kc) * BK, n_idx * BN, p.w_batched ? n0 : 0);
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
    const int w = warp_idx & 3;    // warp of the warpgroup: rows 16 w .. 16 w + 15 of the warpgroup's 64
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
        for (int k = 0; k < BK / 16; ++k) {
          // +32 bytes (2 x 16 B units) per 16-element K step inside the 128 B swizzle row
          const uint64_t adesc = make_wgmma_desc(a_addr) + static_cast<uint64_t>(k * 2);
          const uint64_t bdesc = make_wgmma_desc(b_addr) + static_cast<uint64_t>(k * 2);
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
      if (prev_stage >= 0 && lane == 0) mbar_arrive(&empty_bar[prev_stage]);  // an empty K range consumed no stage

      int n0, y0, x0, mphase;
      decode_m_tile(p, m_idx, n0, y0, x0, mphase);
      const int r0 = 64 * g + 16 * w + (lane >> 2);
      const int cq = 2 * (lane & 3);
#pragma unroll
      for (int pass = 0; pass < BN / BNC; ++pass) {
        named_bar_sync(3, 256);  // the staged tile of the previous pass / tile has been read
#pragma unroll
        for (int i = 0; i < NA; i += 2) {
          // register i: row 16 w + l / 4 + 8 ((i / 2) & 1), column 8 (i / 4) + 2 (l & 3) + (i & 1) of the tile
          if ((8 * (i >> 2)) / BNC != pass) continue;
          const int row = r0 + 8 * ((i >> 1) & 1);
          const int col = 8 * (i >> 2) - pass * BNC + cq;
          *reinterpret_cast<float2*>(acc_smem + row * (BNC + ACC_PAD) + col) = make_float2(acc[i], acc[i + 1]);
        }
        named_bar_sync(3, 256);  // staged tile complete
        if (ES == 2 || g == 0)
          epilogue_tile<BNC, ES>(p, acc_smem, w, lane, n0, y0, x0, n_idx * BN + pass * BNC, split, m_idx, stat_smem, g,
                                 mphase);
      }
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


template <int BN, int ES>
int launch_bn(const ConvGemmParams& p, cudaStream_t stream) {
  using C = Cfg<BN, ES>;
  static bool attr_set = false;
  if (!attr_set) {
    K2_CHECK_CUDA(cudaFuncSetAttribute(conv_gemm_kernel<BN, ES>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       C::SMEM_BYTES));
    attr_set = true;
  }
  int total = p.m_tiles * p.n_tiles * p.splits;
  int grid = total < num_sms() ? total : num_sms();
  K2_CHECK_CUDA(launch_k(conv_gemm_kernel<BN, ES>, dim3(grid), dim3(384), C::SMEM_BYTES, stream, p));
  return 0;
}

}  // namespace

int launch_splitk_finalize(const float* ws, int splits, long long M, int Cout, const float* bias, const __half* residual,
                           int ldr, __half* out, int ldo, float2* gn_part, cudaStream_t stream) {
  dim3 grid(static_cast<unsigned int>((M + 15) / 16), (Cout / 8 + 31) / 32);
  K2_CHECK_CUDA(launch_k(splitk_finalize_kernel, grid, dim3(256), 0, stream, ws, splits, M, Cout, bias, residual, ldr, out, ldo,
                         gn_part));
  return 0;
}

int launch_conv_gemm(const ConvGemmParams& p, int BN, int epilogue_sets, cudaStream_t stream) {
  if (epilogue_sets == 2) {  // both consumer warpgroups drain the accumulator: short-K GEMMs are epilogue-paced
    switch (BN) {
      case 128: return launch_bn<128, 2>(p, stream);
      case 256: return launch_bn<256, 2>(p, stream);
      default: break;  // N tile 192 stages 64 columns per pass: a second set would have nothing to drain
    }
  }
  switch (BN) {
    case 16: return launch_bn<16, 1>(p, stream);
    case 64: return launch_bn<64, 1>(p, stream);
    case 128: return launch_bn<128, 1>(p, stream);
    case 192: return launch_bn<192, 1>(p, stream);
    case 256: return launch_bn<256, 1>(p, stream);
    default: return fail("conv_gemm: unsupported BN");
  }
}

}  // namespace k2
