// k2_attention.cu -- fused softmax(Q K^T * scale) V on sm_90 tensor cores (mma.sync m16n8k16, fp16 in / fp32 accumulate),
// flash-style: no [T, Tkv] score matrix in HBM.  One kernel template serves both attention shapes of the model:
//   head dim 64  (k2_attention_d64): QKVAttention.forward (kandinsky2/model/unet.py:286-340): the two torch.einsum calls
//                (:335,:339), the fp32 softmax (:338), the torch.cat that prepends the encoder K/V (:300-302) and the optional
//                flash-attn path (:303-332).  Keys / values are read from TWO buffers -- encoder tokens first, then the
//                spatial tokens -- so the concat never exists.
//   head dim 512 (k2_attention_d512): the single-head MoVQ AttnBlock (kandinsky2/vqgan/movq_modules.py:201-225; encoder twin
//                vqgan_blocks.py:186-240).  Its output channels are split over two CTAs (DV = 256 each): an fp32 O row of 256
//                channels is 128 registers per thread, the full 512 would not fit next to the scores.  8 warps = 128 queries
//                per CTA, 16-key blocks.
//
// CTA = NW warps, 16 query rows per warp; per key block of BKV keys:
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
template <int D, int DV, int NW, int BKV>
__global__ void __launch_bounds__(NW * 32, 1) flash_attention_kernel(const FlashParams p) {
  using C = FlashCfg<D, DV, NW, BKV>;
  constexpr int NSPLIT = D / DV;
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
      const __half* src = p.qkv + (static_cast<long long>(b) * p.T + (q < p.T ? q : 0)) * p.ldq + head * p.hs + p.q_off + c * 8;
      cp_async_16(smem_u32(sQ + r * C::QP + c * 8), src, q < p.T ? 16 : 0);
    }
  }
  auto load_kv = [&](int jb, int st) {
    constexpr int KC = D / 8, VC = DV / 8;
    for (int i = tid; i < BKV * (KC + VC); i += NW * 32) {
      const int r = i / (KC + VC), c = i - r * (KC + VC);
      const int key = jb * BKV + r;
      const bool ok = key < Tkv;
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
      *reinterpret_cast<uint32_t*>(orow + n * 8) = pack_h2(o[n][2 * h] * inv[h], o[n][2 * h + 1] * inv[h]);
  }
}

template <int D, int DV, int NW, int BKV>
int launch_flash(const FlashParams& p, cudaStream_t stream) {
  using C = FlashCfg<D, DV, NW, BKV>;
  static bool attr_set = false;
  if (!attr_set) {
    K2_CHECK_CUDA(cudaFuncSetAttribute(flash_attention_kernel<D, DV, NW, BKV>, cudaFuncAttributeMaxDynamicSharedMemorySize,
                                       C::SMEM_BYTES));
    attr_set = true;
  }
  dim3 grid((p.T + C::BQ - 1) / C::BQ, p.heads * (D / DV), p.B);
  K2_CHECK_CUDA(launch_k(flash_attention_kernel<D, DV, NW, BKV>, grid, dim3(NW * 32), C::SMEM_BYTES, stream, p));
  return 0;
}

}  // namespace

int launch_attention(const FlashParams& p, int head_dim, cudaStream_t stream) {
  // head width 512: 8 warps x 16-key blocks (Q 130 KB + two K / V stages 49 KB of shared memory) -- 7.5 ms at the MoVQ 768 x 768
  // geometry on an H100 SXM at 700 W, against 12.0 ms with 4 warps x 32-key blocks (one CTA of 4 warps per SM)
  if (head_dim == 512) return launch_flash<512, 256, 8, 16>(p, stream);
  // tuning key 9: query rows per CTA, 128 (8 warps, default) or 64 (4 warps); every warp computes its rows the same way
  return attention_half_rows() ? launch_flash<64, 64, 8, 64>(p, stream) : launch_flash<64, 64, 4, 64>(p, stream);
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
