// k2_attention.cu -- fused softmax(Q K^T * scale) V on sm_90a tensor cores (fp16 in / fp32 accumulate), flash-style: no
// [T, Tkv] score matrix in HBM.  Two kernels serve the two attention shapes of the model:
//   head dim 64  (k2_attention_d64, attention_d64_kernel): QKVAttention.forward (kandinsky2/model/unet.py:286-340): the two
//                torch.einsum calls (:335,:339), the fp32 softmax (:338), the torch.cat that prepends the encoder K/V (:300-302)
//                and the optional flash-attn path (:303-332).  Keys / values are read from TWO tensor maps -- encoder tokens
//                first, then the spatial tokens -- so the concat never exists.  Warp-specialised TMA -> wgmma kernel with the
//                structure of FlashAttention-3 (Shah et al. 2024), described above the kernel.
//   head dim 512 (k2_attention_d512, flash_attention_kernel): the single-head MoVQ AttnBlock (kandinsky2/vqgan/movq_modules.py:
//                201-225; encoder twin vqgan_blocks.py:186-240) on mma.sync m16n8k16.  Its output channels are split over two
//                CTAs (DV = 256 each): an fp32 O row of 256 channels is 128 registers per thread, the full 512 would not fit
//                next to the scores.  8 warps = 128 queries per CTA, 16-key blocks.
//   head dim 104 (k2_attention_heads, flash_attention_kernel with DR = 104): the CLIP ViT-bigG/14 image tower's 16 heads
//                (kandinsky2/model/clip_vision.py).  The tiles are D = 112 wide (seven k16 steps); the 8 columns past the real
//                width arrive zero-filled and the matching output columns are not stored, so the arithmetic is the unpadded one.
// Both follow one numerical recipe: fp32 scores, scale * log2(e) folded into ex2, row sums from the unrounded fp32 P, P rounded
// to fp16 before PV (as in the reference's fp16 mode, unet.py:338), O / l rounded once to fp16.  Every key block they process
// holds at least one valid key, so the running maximum is finite from the first block on.
//
// flash_attention_kernel: CTA = NW warps, 16 query rows per warp; per key block of BKV keys:
//   (DR = the real head width, <= D, a multiple of 8: q / k / v columns [DR, D) of the tiles are zero-filled by cp.async with
//   src-size 0 -- zero q and k columns add exact zeros to the fp32 scores -- and output columns [DR, D) are never stored.
//   With DR = D every such test is a compile-time constant and the kernel is the unpadded one.)
//     S = Q K^T            Q fragments (ldmatrix) x K fragments (ldmatrix) from shared memory, fp32 in registers
//     m = max(m, rowmax S * c), P = exp2(S * c - m), l = l * alpha + rowsum P, O = O * alpha + fp16(P) V
//   P goes from the score accumulators straight into the A fragments of the PV product (same register layout), V is read
//   with ldmatrix.trans as it lies in memory ([key][channel] rows).  K / V blocks are double-buffered with cp.async.
//   P is rounded to fp16 before PV (as in the reference's fp16 mode, unet.py:338); the row sums use the unrounded fp32 P.
#include <string.h>

#include <algorithm>

#include "../../include/k2b200.h"
#include "k2_common.cuh"
#include "k2_internal.h"

namespace k2 {

namespace {

__device__ __forceinline__ float ex2(float x) {
  float y;
  asm("ex2.approx.ftz.f32 %0, %1;" : "=f"(y) : "f"(x));
  return y;
}
__device__ __forceinline__ uint32_t pack_h2(float lo, float hi) {
  __half2 h = __floats2half2_rn(lo, hi);
  return *reinterpret_cast<uint32_t*>(&h);
}

template <int D, int DV, int NW, int BKV>
struct FlashCfg {
  static constexpr int BQ = 16 * NW;
  static constexpr int QP = D + 8;    // row pitch (halves) of Q / K tiles: 16-byte ldmatrix rows on distinct bank groups
  static constexpr int VP = DV + 8;
  static constexpr int Q_BYTES = BQ * QP * 2;
  static constexpr int K_BYTES = BKV * QP * 2;
  static constexpr int V_BYTES = BKV * VP * 2;
  static constexpr int SMEM_BYTES = Q_BYTES + 2 * (K_BYTES + V_BYTES);
};

// grid: (query tiles, heads * D / DV, B); blockIdx.y = head * (D / DV) + output-channel split
template <int D, int DV, int NW, int BKV, int DR>
__global__ void __launch_bounds__(NW * 32, 1) flash_attention_kernel(const FlashParams p) {
  using C = FlashCfg<D, DV, NW, BKV>;
  constexpr int NSPLIT = D / DV;
  static_assert(DR % 8 == 0 && DR <= D && (DR == D || NSPLIT == 1), "a padded head keeps its output channels in one CTA");
  extern __shared__ __align__(16) uint8_t smem[];
  __half* sQ = reinterpret_cast<__half*>(smem);
  __half* sK = reinterpret_cast<__half*>(smem + C::Q_BYTES);                  // [2][BKV][QP]
  __half* sV = reinterpret_cast<__half*>(smem + C::Q_BYTES + 2 * C::K_BYTES);  // [2][BKV][VP]

  const int tid = threadIdx.x;
  const int warp = tid >> 5;
  const int lane = tid & 31;
  const int q0 = blockIdx.x * C::BQ;
  const int head = blockIdx.y / NSPLIT;
  const int dsplit = blockIdx.y - head * NSPLIT;
  const int b = blockIdx.z;
  const int Tkv = p.Tc + p.T;
  const int nblk = (Tkv + BKV - 1) / BKV;

  pdl_wait();
  pdl_launch();

  {  // Q tile (rows past T are zero-filled)
    constexpr int CPR = D / 8;  // 16-byte chunks per row
    for (int i = tid; i < C::BQ * CPR; i += NW * 32) {
      const int r = i / CPR, c = i - r * CPR;
      const int q = q0 + r;
      const bool real = DR == D || c < DR / 8;
      const __half* src = p.qkv + (static_cast<long long>(b) * p.T + (q < p.T ? q : 0)) * p.ldq + head * p.hs + p.q_off +
                          (real ? c * 8 : 0);
      cp_async_16(smem_u32(sQ + r * C::QP + c * 8), src, q < p.T && real ? 16 : 0);
    }
  }
  auto load_kv = [&](int jb, int st) {
    constexpr int KC = D / 8, VC = DV / 8;
    for (int i = tid; i < BKV * (KC + VC); i += NW * 32) {
      const int r = i / (KC + VC), c = i - r * (KC + VC);
      const int key = jb * BKV + r;
      const bool ok = key < Tkv && (DR == D || (c < KC ? c : c - KC) < DR / 8);
      const bool from_enc = key < p.Tc;
      const __half* row = from_enc ? p.enc + (static_cast<long long>(b) * p.Tc + key) * p.lde + head * p.ehs
                                   : p.qkv + (static_cast<long long>(b) * p.T + (ok ? key - p.Tc : 0)) * p.ldq + head * p.hs;
      if (c < KC) {
        const __half* src = row + (from_enc ? p.ek_off : p.k_off) + c * 8;
        cp_async_16(smem_u32(sK + (st * BKV + r) * C::QP + c * 8), ok ? src : p.qkv, ok ? 16 : 0);
      } else {
        const __half* src = row + (from_enc ? p.ev_off : p.v_off) + dsplit * DV + (c - KC) * 8;
        cp_async_16(smem_u32(sV + (st * BKV + r) * C::VP + (c - KC) * 8), ok ? src : p.qkv, ok ? 16 : 0);
      }
    }
  };
  load_kv(0, 0);
  cp_async_commit();

  const float c = p.scale_log2e;
  float m_r[2] = {-INFINITY, -INFINITY}, l_r[2] = {0.f, 0.f};
  float o[DV / 8][4];
#pragma unroll
  for (int n = 0; n < DV / 8; ++n) o[n][0] = o[n][1] = o[n][2] = o[n][3] = 0.f;

  const uint32_t q_lane = smem_u32(sQ + (warp * 16 + (lane & 15)) * C::QP + (lane >> 4) * 8);
  for (int jb = 0; jb < nblk; ++jb) {
    const int st = jb & 1;
    if (jb + 1 < nblk) {
      load_kv(jb + 1, st ^ 1);
      cp_async_commit();
      cp_async_wait<1>();
    } else {
      cp_async_wait<0>();
    }
    __syncthreads();

    // S = Q K^T for this warp's 16 rows x BKV keys
    float s[BKV / 8][4];
#pragma unroll
    for (int n = 0; n < BKV / 8; ++n) s[n][0] = s[n][1] = s[n][2] = s[n][3] = 0.f;
    const uint32_t k_lane = smem_u32(sK + (st * BKV + ((lane >> 4) << 3) + (lane & 7)) * C::QP + ((lane >> 3) & 1) * 8);
#pragma unroll 4
    for (int kk = 0; kk < D / 16; ++kk) {
      uint32_t a[4];
      ldmatrix_x4(a, q_lane + kk * 32);
#pragma unroll
      for (int n = 0; n < BKV / 8; n += 2) {
        uint32_t bk[4];
        ldmatrix_x4(bk, k_lane + n * 8 * C::QP * 2 + kk * 32);
        mma_16816(s[n], a, bk[0], bk[1]);
        mma_16816(s[n + 1], a, bk[2], bk[3]);
      }
    }

    // online softmax over the block (rows lane / 4 and lane / 4 + 8 of the warp's 16)
    const int kbase = jb * BKV + 2 * (lane & 3);
    float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
    for (int n = 0; n < BKV / 8; ++n) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        const int key = kbase + n * 8 + (e & 1);
        s[n][e] = key < Tkv ? s[n][e] * c : -INFINITY;
        mx[e >> 1] = fmaxf(mx[e >> 1], s[n][e]);
      }
    }
    float alpha[2];
#pragma unroll
    for (int h = 0; h < 2; ++h) {
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
      mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
      const float m_new = fmaxf(m_r[h], mx[h]);  // finite: every block holds at least one valid key
      alpha[h] = ex2(m_r[h] - m_new);            // 0 for the first block
      m_r[h] = m_new;
    }
    float ls[2] = {0.f, 0.f};
#pragma unroll
    for (int n = 0; n < BKV / 8; ++n) {
#pragma unroll
      for (int e = 0; e < 4; ++e) {
        s[n][e] = ex2(s[n][e] - m_r[e >> 1]);
        ls[e >> 1] += s[n][e];
      }
    }
#pragma unroll
    for (int h = 0; h < 2; ++h) l_r[h] = l_r[h] * alpha[h] + ls[h];
#pragma unroll
    for (int n = 0; n < DV / 8; ++n) {
      o[n][0] *= alpha[0];
      o[n][1] *= alpha[0];
      o[n][2] *= alpha[1];
      o[n][3] *= alpha[1];
    }

    // O += fp16(P) V
    const uint32_t v_lane = smem_u32(sV + (st * BKV + ((lane >> 3) & 1) * 8 + (lane & 7)) * C::VP + (lane >> 4) * 8);
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) {
      uint32_t a[4];
      a[0] = pack_h2(s[2 * kk][0], s[2 * kk][1]);
      a[1] = pack_h2(s[2 * kk][2], s[2 * kk][3]);
      a[2] = pack_h2(s[2 * kk + 1][0], s[2 * kk + 1][1]);
      a[3] = pack_h2(s[2 * kk + 1][2], s[2 * kk + 1][3]);
#pragma unroll
      for (int n = 0; n < DV / 8; n += 2) {
        uint32_t bv[4];
        ldmatrix_x4_trans(bv, v_lane + (kk * 16 * C::VP + n * 8) * 2);
        mma_16816(o[n], a, bv[0], bv[1]);
        mma_16816(o[n + 1], a, bv[2], bv[3]);
      }
    }
    __syncthreads();  // the next iteration's prefetch overwrites this stage
  }

  // out = O / l
  l_r[0] += __shfl_xor_sync(0xffffffffu, l_r[0], 1);
  l_r[0] += __shfl_xor_sync(0xffffffffu, l_r[0], 2);
  l_r[1] += __shfl_xor_sync(0xffffffffu, l_r[1], 1);
  l_r[1] += __shfl_xor_sync(0xffffffffu, l_r[1], 2);
  const float inv[2] = {1.f / l_r[0], 1.f / l_r[1]};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int q = q0 + warp * 16 + (lane >> 2) + 8 * h;
    if (q >= p.T) continue;
    __half* orow = p.out + (static_cast<long long>(b) * p.T + q) * p.ldo + head * p.ohs + dsplit * DV + 2 * (lane & 3);
#pragma unroll
    for (int n = 0; n < DV / 8; ++n)
      if (DR == D || n < DR / 8)
        *reinterpret_cast<uint32_t*>(orow + n * 8) = pack_h2(o[n][2 * h] * inv[h], o[n][2 * h + 1] * inv[h]);
  }
}

template <int D, int DV, int NW, int BKV, int DR = D>
int launch_flash(const FlashParams& p, cudaStream_t stream) {
  using C = FlashCfg<D, DV, NW, BKV>;
  static bool attr_set = false;
  if (!attr_set) {
    K2_CHECK_CUDA(cudaFuncSetAttribute(flash_attention_kernel<D, DV, NW, BKV, DR>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       C::SMEM_BYTES));
    attr_set = true;
  }
  dim3 grid((p.T + C::BQ - 1) / C::BQ, p.heads * (D / DV), p.B);
  K2_CHECK_CUDA(launch_k(flash_attention_kernel<D, DV, NW, BKV, DR>, grid, dim3(NW * 32), C::SMEM_BYTES, stream, p));
  return 0;
}

// ------------------------------------------------------------------------------------------------------------------------------
// Head width 64.  At this width a score costs 256 tensor FLOPs (QK^T + PV) and one ex2: an H100 SM does 16 scores' worth of MMA
// per clock and 16 ex2 per clock, so a warp that runs its MMAs and its softmax one after the other leaves the tensor cores idle
// half the time.  The kernel overlaps the two (FlashAttention-3, Shah et al. 2024, sections 3.1-3.2):
//   CTA = 3 warpgroups, 128 query rows.  Warpgroup 0 is the producer: one thread issues the TMA loads (Q once, then K / V blocks
//   of 128 keys into a STAGES-deep mbarrier ring); the warpgroup gives its registers to the two consumer warpgroups, each of which
//   owns 64 query rows.  Per key block j a consumer
//     issues  S_j = Q K_j^T         wgmma m64n128k16, both operands in shared memory (K stored [key][channel] is K-major)
//     issues  O += P_{j-1} V_{j-1}  wgmma m64n64k16, P in registers, V read MN-major ([key][channel]) with the transpose flag
//     waits for S_j, runs the online softmax of block j while PV_{j-1} is still on the tensor cores (intra-warpgroup overlap),
//     waits for PV_{j-1}, frees its stage, and rescales O by the new maximum before it issues PV_j.
//   Named barriers make the two consumers take turns at issuing (inter-warpgroup ping-pong), so one's softmax runs while the
//   other's products run.
// Keys: ceil(Tc / 128) blocks from the encoder tensor map, then ceil(T / 128) blocks from qkv.  The tensor maps are [B][T][width]
// with the width the heads span, so a box never reaches another image's rows or a strided view's gap columns; rows past Tc / T
// arrive zero-filled and only the last block of each source masks its tail.
// ------------------------------------------------------------------------------------------------------------------------------
namespace d64 {
constexpr int BQ = 128;                     // query rows per CTA (two consumer warpgroups of 64)
constexpr int BKV = 128;                    // keys per block
constexpr int STAGES = 4;                   // K / V ring depth: a stage stays busy until the PV of the next block is issued
constexpr int TILE = 128 * 128;             // one 128-row x 64-channel fp16 tile, 128-byte swizzled rows
constexpr int BAR_BYTES = 8 * (2 * STAGES + 1);
constexpr int SMEM_BYTES = 1024 + TILE * (1 + 2 * STAGES) + BAR_BYTES;  // + slack to align the tiles to 1024 B
constexpr int TURN_BAR = 1;                 // named barriers 1, 2: the issuing turn of consumer warpgroup 0, 1
}  // namespace d64

struct AttnD64Params {
  CUtensorMap tm_qkv;  // [B][T][width of the heads' q | k | v], box 64 x 128 x 1
  CUtensorMap tm_enc;  // [B][Tc][width of the heads' k | v] (unused when Tc = 0)
  __half* out;         // [B, T, ldo], head h at channels 64 h
  long long ldo;
  int hs, q_off, k_off, v_off;
  int ehs, ek_off, ev_off;
  int T, Tc;
  float scale_log2e;
};

// Online softmax of one 64 x 128 block held as an m64n128 accumulator: this thread's rows r0 = l / 4 and r0 + 8 of its warp's
// 16 (h = (i / 2) & 1), key 8 (i / 4) + 2 (l & 3) + (i & 1) of the block.  s becomes the unrounded fp32 P; m / l are the running
// maximum (scaled units) and this thread's partial row sums; alpha is the factor O must be rescaled by before P V is added.
template <bool MASK>
__device__ __forceinline__ void softmax_block(float (&s)[64], float (&m)[2], float (&l)[2], float (&alpha)[2], float c, int valid) {
  const int kq = 2 * (threadIdx.x & 3);
  if (MASK) {
#pragma unroll
    for (int i = 0; i < 64; ++i)
      if (8 * (i >> 2) + kq + (i & 1) >= valid) s[i] = -INFINITY;
  }
  float mx[2] = {-INFINITY, -INFINITY};
#pragma unroll
  for (int i = 0; i < 64; ++i) mx[(i >> 1) & 1] = fmaxf(mx[(i >> 1) & 1], s[i]);
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 1));
    mx[h] = fmaxf(mx[h], __shfl_xor_sync(0xffffffffu, mx[h], 2));
    const float m_new = fmaxf(m[h], mx[h] * c);  // finite: the block holds at least one valid key
    alpha[h] = ex2(m[h] - m_new);                // 0 for the first block
    m[h] = m_new;
  }
  float ls[2][2] = {{0.f, 0.f}, {0.f, 0.f}};  // two partial sums per row: shorter dependency chains
#pragma unroll
  for (int i = 0; i < 64; ++i) {
    const int h = (i >> 1) & 1;
    s[i] = ex2(fmaf(s[i], c, -m[h]));
    ls[h][(i >> 2) & 1] += s[i];
  }
#pragma unroll
  for (int h = 0; h < 2; ++h) l[h] = l[h] * alpha[h] + (ls[h][0] + ls[h][1]);
}

// grid: (query tiles, heads, B)
__global__ void __launch_bounds__(384, 1) attention_d64_kernel(const __grid_constant__ AttnD64Params p) {
  using namespace d64;
  extern __shared__ uint8_t smem_raw[];
  uint8_t* smem = reinterpret_cast<uint8_t*>((reinterpret_cast<uintptr_t>(smem_raw) + 1023) & ~static_cast<uintptr_t>(1023));
  uint8_t* sQ = smem;
  uint8_t* sK = smem + TILE;                   // [STAGES] tiles
  uint8_t* sV = sK + STAGES * TILE;            // [STAGES] tiles
  uint64_t* full_bar = reinterpret_cast<uint64_t*>(sV + STAGES * TILE);
  uint64_t* empty_bar = full_bar + STAGES;
  uint64_t* q_bar = empty_bar + STAGES;

  const int warp = threadIdx.x >> 5;
  const int lane = threadIdx.x & 31;
  const int wg = warp >> 2;
  const int q0 = blockIdx.x * BQ;
  const int head = blockIdx.y;
  const int b = blockIdx.z;
  const int nenc = (p.Tc + BKV - 1) / BKV;
  const int nblk = nenc + (p.T + BKV - 1) / BKV;

  if (threadIdx.x == 0) {
    tma_prefetch_desc(&p.tm_qkv);
    if (nenc) tma_prefetch_desc(&p.tm_enc);
    for (int i = 0; i < STAGES; ++i) {
      mbar_init(&full_bar[i], 1);
      mbar_init(&empty_bar[i], 8);  // one arrival per consumer warp, after its wgmma.wait_group
    }
    mbar_init(q_bar, 1);
    fence_barrier_init();
  }
  __syncthreads();
  pdl_wait();
  pdl_launch();

  if (wg == 0) {
    // ===================================== TMA producer =====================================
    setmaxnreg_dec<40>();
    if (warp == 0 && elect_one()) {
      mbar_arrive_expect_tx(q_bar, TILE);
      tma_load_3d(sQ, &p.tm_qkv, q_bar, head * p.hs + p.q_off, q0, b);
      for (int j = 0; j < nblk; ++j) {
        const int st = j % STAGES;
        if (j >= STAGES) mbar_wait_lean(&empty_bar[st], (j / STAGES - 1) & 1);
        mbar_arrive_expect_tx(&full_bar[st], 2 * TILE);  // zero-filled rows count: the box is always written whole
        if (j < nenc) {
          tma_load_3d(sK + st * TILE, &p.tm_enc, &full_bar[st], head * p.ehs + p.ek_off, j * BKV, b);
          tma_load_3d(sV + st * TILE, &p.tm_enc, &full_bar[st], head * p.ehs + p.ev_off, j * BKV, b);
        } else {
          tma_load_3d(sK + st * TILE, &p.tm_qkv, &full_bar[st], head * p.hs + p.k_off, (j - nenc) * BKV, b);
          tma_load_3d(sV + st * TILE, &p.tm_qkv, &full_bar[st], head * p.hs + p.v_off, (j - nenc) * BKV, b);
        }
      }
    }
    return;
  }

  // ====================================== consumers ======================================
  setmaxnreg_inc<232>();
  const int cw = wg - 1;  // query rows [64 cw, 64 cw + 64) of the tile
  const float c = p.scale_log2e;
  const uint64_t qdesc = make_wgmma_desc(smem_u32(sQ) + cw * 64 * 128);
  const uint32_t k_base = smem_u32(sK), v_base = smem_u32(sV);

  float o[32], s[64], m[2] = {-INFINITY, -INFINITY}, l[2] = {0.f, 0.f}, alpha[2] = {0.f, 0.f};
  uint32_t pa[32];  // fp16 P of the previous block: the A fragments of its 8 PV steps of 16 keys
#pragma unroll
  for (int i = 0; i < 32; ++i) o[i] = 0.f;

  auto issue_pv = [&](int st) {
#pragma unroll
    for (int kk = 0; kk < BKV / 16; ++kk) {
      const uint32_t a[4] = {pa[4 * kk], pa[4 * kk + 1], pa[4 * kk + 2], pa[4 * kk + 3]};
      wgmma_m64n64k16_rs_tb(o, a, make_wgmma_desc_mn(v_base + st * TILE) + static_cast<uint64_t>(kk * (2048 >> 4)));
    }
    wgmma_commit();
  };
  auto rescale_o = [&]() {
#pragma unroll
    for (int i = 0; i < 32; ++i) o[i] *= alpha[(i >> 1) & 1];
  };

  // S_j = Q K_j^T after this warpgroup's turn has come; hands the turn over once the block's products are issued
  auto issue_s = [&](int j) {
    const int st = j % STAGES;
    mbar_wait_lean(&full_bar[st], (j / STAGES) & 1);
    named_bar_sync(TURN_BAR + cw, 256);
    wgmma_fence();
#pragma unroll
    for (int kk = 0; kk < 4; ++kk)  // +32 B per 16 channels inside the 128 B swizzle row
      wgmma_m64n128k16(s, qdesc + static_cast<uint64_t>(kk * 2), make_wgmma_desc(k_base + st * TILE) + static_cast<uint64_t>(kk * 2),
                       kk > 0);
    wgmma_commit();
  };
  // warpgroup 1 skips its last hand-over, so that every arrival at a turn barrier meets a wait
  auto pass_turn = [&](int j) {
    if (cw == 0 || j + 1 < nblk) named_bar_arrive(TURN_BAR + 1 - cw, 256);
  };
  auto softmax = [&](int j) {
#pragma unroll
    for (int i = 0; i < 64; ++i) reg_fence(s[i]);
    const int valid = j < nenc ? p.Tc - j * BKV : p.T - (j - nenc) * BKV;
    if (valid < BKV) softmax_block<true>(s, m, l, alpha, c, valid);
    else softmax_block<false>(s, m, l, alpha, c, valid);
  };
  auto to_p = [&]() {
#pragma unroll
    for (int i = 0; i < 32; ++i) pa[i] = pack_h2(s[2 * i], s[2 * i + 1]);
  };

  if (cw == 1) named_bar_arrive(TURN_BAR, 256);  // warpgroup 0 takes the first turn
  mbar_wait_lean(q_bar, 0);
  issue_s(0);
  pass_turn(0);
  wgmma_wait<0>();
  softmax(0);
  to_p();
  for (int j = 1; j < nblk; ++j) {
    const int pst = (j - 1) % STAGES;
    rescale_o();  // by the maximum of block j - 1, before P_{j-1} V_{j-1} is added
    issue_s(j);
    issue_pv(pst);
    pass_turn(j);
    wgmma_wait<1>();  // S_j; P_{j-1} V_{j-1} stays on the tensor cores during the softmax
    softmax(j);
    wgmma_wait<0>();
#pragma unroll
    for (int i = 0; i < 32; ++i) reg_fence(o[i]);
    if (lane == 0) mbar_arrive(&empty_bar[pst]);
    to_p();
  }
  rescale_o();
  wgmma_fence();
  issue_pv((nblk - 1) % STAGES);
  wgmma_wait<0>();
#pragma unroll
  for (int i = 0; i < 32; ++i) reg_fence(o[i]);

  // out = O / l
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 1);
    l[h] += __shfl_xor_sync(0xffffffffu, l[h], 2);
  }
  const float inv[2] = {1.f / l[0], 1.f / l[1]};
#pragma unroll
  for (int h = 0; h < 2; ++h) {
    const int q = q0 + 64 * cw + 16 * (warp & 3) + (lane >> 2) + 8 * h;
    if (q >= p.T) continue;
    __half* orow = p.out + (static_cast<long long>(b) * p.T + q) * p.ldo + head * 64 + 2 * (lane & 3);
#pragma unroll
    for (int n = 0; n < 8; ++n)
      *reinterpret_cast<uint32_t*>(orow + n * 8) = pack_h2(o[4 * n + 2 * h] * inv[h], o[4 * n + 2 * h + 1] * inv[h]);
  }
}

int launch_attention_d64(const FlashParams& f, cudaStream_t stream) {
  using namespace d64;
  AttnD64Params p;
  memset(&p, 0, sizeof p);
  const uint32_t box[3] = {64, BKV, 1};  // BQ = BKV: Q, K and V tiles share the box
  {
    const uint64_t width = static_cast<uint64_t>(f.heads - 1) * f.hs + std::max(std::max(f.q_off, f.k_off), f.v_off) + 64;
    const uint64_t dims[3] = {width, static_cast<uint64_t>(f.T), static_cast<uint64_t>(f.B)};
    const uint64_t strides[2] = {static_cast<uint64_t>(f.ldq) * 2, static_cast<uint64_t>(f.ldq) * 2 * f.T};
    if (encode_tmap_f16(&p.tm_qkv, f.qkv, 3, dims, strides, box)) return -1;
  }
  if (f.Tc > 0) {
    const uint64_t width = static_cast<uint64_t>(f.heads - 1) * f.ehs + std::max(f.ek_off, f.ev_off) + 64;
    const uint64_t dims[3] = {width, static_cast<uint64_t>(f.Tc), static_cast<uint64_t>(f.B)};
    const uint64_t strides[2] = {static_cast<uint64_t>(f.lde) * 2, static_cast<uint64_t>(f.lde) * 2 * f.Tc};
    if (encode_tmap_f16(&p.tm_enc, f.enc, 3, dims, strides, box)) return -1;
  }
  p.out = f.out;
  p.ldo = f.ldo;
  p.hs = f.hs; p.q_off = f.q_off; p.k_off = f.k_off; p.v_off = f.v_off;
  p.ehs = f.ehs; p.ek_off = f.ek_off; p.ev_off = f.ev_off;
  p.T = f.T; p.Tc = f.Tc;
  p.scale_log2e = f.scale_log2e;
  static bool attr_set = false;
  if (!attr_set) {
    K2_CHECK_CUDA(cudaFuncSetAttribute(attention_d64_kernel, cudaFuncAttributeMaxDynamicSharedMemorySize, SMEM_BYTES));
    attr_set = true;
  }
  dim3 grid((f.T + BQ - 1) / BQ, f.heads, f.B);
  K2_CHECK_CUDA(launch_k(attention_d64_kernel, grid, dim3(384), SMEM_BYTES, stream, p));
  return 0;
}

}  // namespace

int launch_attention(const FlashParams& p, int head_dim, cudaStream_t stream) {
  // head width 512: 8 warps x 16-key blocks (Q 130 KB + two K / V stages 49 KB of shared memory) -- 7.5 ms at the MoVQ 768 x 768
  // geometry on an H100 SXM at 700 W, against 12.0 ms with 4 warps x 32-key blocks (one CTA of 4 warps per SM)
  if (head_dim == 512) return launch_flash<512, 256, 8, 16>(p, stream);
  // head width 104 (CLIP ViT-bigG/14: T = 257, 16 heads): 4 warps = 64 queries per CTA and 64-key blocks.  An image is then
  // 5 query tiles x 16 heads = 80 CTAs, and a B >= 2 batch fills the 132 SMs; each CTA keeps O (14 x 4 fp32), the scores
  // (8 x 4) and a 64-key block's K / V stages (Q 15 KB + 2 x 30 KB of shared memory) resident, so two CTAs fit per SM.
  // Smaller query tiles would cut the padding of the last tile (257 = 4 x 64 + 1) but re-read every key from L2 for half as
  // many queries.  Not tuned: the attention is 2.2 % of the tower's FLOPs.
  if (head_dim == 104) return launch_flash<112, 112, 4, 64, 104>(p, stream);
  return launch_attention_d64(p, stream);
}

}  // namespace k2

using namespace k2;

extern "C" int k2_attention_d64(const void* qkv, int ldq, int hs, int q_off, int k_off, int v_off, const void* enc,
                                int lde, int ehs, int ek_off, int ev_off, int B, int heads, int T, int Tc, float scale,
                                void* out, int ldo, k2_stream_t stream) {
  K2_REQUIRE(qkv && out && B > 0 && heads > 0 && T > 0, "attention_d64: bad arguments");
  K2_REQUIRE(ldq % 8 == 0 && ldo % 8 == 0 && hs % 8 == 0 && q_off % 8 == 0 && k_off % 8 == 0 && v_off % 8 == 0,
             "attention_d64: strides/offsets must be multiples of 8 elements");
  K2_REQUIRE((enc != nullptr) == (Tc > 0), "attention_d64: enc and Tc go together");
  K2_REQUIRE((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
             "attention_d64: 16-byte alignment");
  K2_REQUIRE((heads - 1) * hs + std::max(std::max(q_off, k_off), v_off) + 64 <= ldq,
             "attention_d64: qkv row narrower than heads*hs");
  if (Tc > 0) {
    K2_REQUIRE(lde % 8 == 0 && ehs % 8 == 0 && ek_off % 8 == 0 && ev_off % 8 == 0 &&
                   (reinterpret_cast<uintptr_t>(enc) & 15) == 0,
               "attention_d64: encoder strides/alignment");
    K2_REQUIRE((heads - 1) * ehs + std::max(ek_off, ev_off) + 64 <= lde, "attention_d64: encoder row narrower than heads*ehs");
  }
  FlashParams p;
  memset(&p, 0, sizeof p);
  p.qkv = reinterpret_cast<const __half*>(qkv);
  p.ldq = ldq; p.hs = hs; p.q_off = q_off; p.k_off = k_off; p.v_off = v_off;
  p.enc = reinterpret_cast<const __half*>(enc);
  p.lde = lde; p.ehs = ehs; p.ek_off = ek_off; p.ev_off = ev_off;
  p.B = B; p.heads = heads; p.T = T; p.Tc = Tc;
  p.out = reinterpret_cast<__half*>(out);
  p.ldo = ldo;
  p.ohs = 64;
  p.scale_log2e = scale * 1.4426950408889634f;
  int rc = launch_attention(p, 64, static_cast<cudaStream_t>(stream));
  if (rc == 0) count_launch();
  return rc;
}
