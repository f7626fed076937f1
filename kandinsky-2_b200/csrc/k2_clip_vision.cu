// k2_clip_vision.cu -- the two entry points the CLIP ViT-bigG/14 image tower (kandinsky2/model/clip_vision.py) needs on top of
// the flat-row GEMM, LayerNorm, GELU and fp16 -> fp32 widening the diffusion prior already uses:
//   k2_clip_patchify    fp32 NCHW pixels -> fp16 GEMM rows: the CLS slot and the P x P patches, so that the patch convolution,
//                       the class embedding and the position embedding are ONE k2_conv_gemm launch (weight [hidden, Kp] =
//                       the conv weight flattened (c, ky, kx), then class_embedding as column 3 P^2; the position embedding is
//                       the epilogue's residual).
//   k2_attention_heads  multi-head attention at head width 104 (16 heads over 257 tokens in the tower), the flash template of
//                       k2_attention.cu with the head padded to 112 in shared memory only.
// Parity: tests/test_gpu_clip_vision_kernels.py (patchify bit-exact against torch, attention against float64).
#include <string.h>

#include <algorithm>

#include "../../include/k2b200.h"
#include "k2_common.cuh"
#include "k2_internal.h"

namespace k2 {
namespace {

// One block per output row m = b * (G^2 + 1) + t.  Row t = 0 is the one-hot CLS row (1 in column 3 P^2); row t = 1 + py G + px
// holds patch (py, px) in column c P^2 + ky P + kx, rounded to fp16 (the fp16 model's pixel_values.to(fp16)).  Columns past
// 3 P^2 (+ 1 for the CLS row) up to Kp are zero.
__global__ void __launch_bounds__(256) clip_patchify_kernel(const float* __restrict__ x, int S, int P, int G,
                                                            __half* __restrict__ y, long long ldy, int Kp) {
  const int T = G * G + 1;
  const int b = blockIdx.x / T, t = blockIdx.x - b * T;
  const int PP = P * P, K = 3 * PP;
  __half* yr = y + static_cast<long long>(blockIdx.x) * ldy;
  if (t == 0) {
    for (int k = threadIdx.x; k < Kp; k += blockDim.x) yr[k] = __float2half_rn(k == K ? 1.f : 0.f);
    return;
  }
  const int py = (t - 1) / G, px = (t - 1) - py * G;
  const float* xb = x + static_cast<long long>(b) * 3 * S * S + static_cast<long long>(py * P) * S + px * P;
  for (int k = threadIdx.x; k < Kp; k += blockDim.x) {
    float v = 0.f;
    if (k < K) {
      const int c = k / PP, r = k - c * PP;
      const int ky = r / P, kx = r - ky * P;
      v = xb[static_cast<long long>(c) * S * S + ky * S + kx];
    }
    yr[k] = __float2half_rn(v);
  }
}

}  // namespace
}  // namespace k2

using namespace k2;

extern "C" {

int k2_clip_patchify(const float* x, int B, int S, int P, void* out, int ldo, int Kp, k2_stream_t stream) {
  K2_REQUIRE(x && out && B > 0 && S > 0 && P > 0, "clip_patchify: bad arguments");
  K2_REQUIRE(S % P == 0, "clip_patchify: image size must be a multiple of the patch size");
  K2_REQUIRE(Kp >= 3 * P * P + 1 && ldo >= Kp, "clip_patchify: Kp must hold 3 P^2 + 1 columns and ldo >= Kp");
  K2_REQUIRE((reinterpret_cast<uintptr_t>(x) & 3) == 0 && (reinterpret_cast<uintptr_t>(out) & 1) == 0,
             "clip_patchify: alignment");
  const int G = S / P;
  const long long rows = static_cast<long long>(B) * (G * G + 1);
  K2_REQUIRE(rows <= 0x7fffffffLL, "clip_patchify: too many rows");
  clip_patchify_kernel<<<static_cast<unsigned int>(rows), 256, 0, static_cast<cudaStream_t>(stream)>>>(
      x, S, P, G, reinterpret_cast<__half*>(out), ldo, Kp);
  K2_CHECK_CUDA(cudaGetLastError());
  count_launch();
  return 0;
}

int k2_attention_heads(const void* qkv, int ldq, int hs, int q_off, int k_off, int v_off, int B, int heads, int T, int head_dim,
                       float scale, void* out, int ldo, int ohs, k2_stream_t stream) {
  K2_REQUIRE(head_dim == 104, "attention_heads: only head width 104 is implemented");
  K2_REQUIRE(qkv && out && B > 0 && heads > 0 && T > 0 && B <= 65535 && heads <= 65535, "attention_heads: bad arguments");
  K2_REQUIRE(ldq % 8 == 0 && ldo % 8 == 0 && hs % 8 == 0 && ohs % 8 == 0 && q_off % 8 == 0 && k_off % 8 == 0 &&
                 v_off % 8 == 0 && q_off >= 0 && k_off >= 0 && v_off >= 0,
             "attention_heads: strides / offsets must be non-negative multiples of 8 elements");
  K2_REQUIRE(static_cast<long long>(heads - 1) * hs + std::max(std::max(q_off, k_off), v_off) + head_dim <= ldq,
             "attention_heads: qkv row narrower than the heads");
  K2_REQUIRE(ohs >= head_dim && static_cast<long long>(heads - 1) * ohs + head_dim <= ldo,
             "attention_heads: output row narrower than the heads");
  K2_REQUIRE(aligned16(qkv) && aligned16(out), "attention_heads: 16-byte alignment");
  FlashParams p;
  memset(&p, 0, sizeof p);
  p.qkv = reinterpret_cast<const __half*>(qkv);
  p.ldq = ldq; p.hs = hs; p.q_off = q_off; p.k_off = k_off; p.v_off = v_off;
  p.B = B; p.heads = heads; p.T = T;
  p.out = reinterpret_cast<__half*>(out);
  p.ldo = ldo;
  p.ohs = ohs;
  p.scale_log2e = scale * 1.4426950408889634f;
  int rc = launch_attention(p, head_dim, static_cast<cudaStream_t>(stream));
  if (rc == 0) count_launch();
  return rc;
}

}  // extern "C"
