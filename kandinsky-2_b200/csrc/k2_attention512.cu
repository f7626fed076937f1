// k2_attention512.cu -- fused softmax(q k^T / sqrt(C)) v for ONE head of width C = 512: the MoVQ AttnBlock
// (kandinsky2/vqgan/movq_modules.py:201-225; encoder twin vqgan_blocks.py:186-240) without the [T, T] score matrix in HBM
// (680 MB for four 768 x 768 images, written once and read twice by the unfused path).  The kernel is the flash-attention
// template of k2_attention.cu with head width 512, its output channels split over two CTAs per query tile.
#include <string.h>

#include <algorithm>

#include "../../include/k2b200.h"
#include "k2_internal.h"

using namespace k2;

extern "C" int k2_attention_d512(const void* qkv, int ldq, int q_off, int k_off, int v_off, int B, int T, float scale, void* out,
                                 int ldo, k2_stream_t stream) {
  constexpr int CH = 512;
  K2_REQUIRE(qkv && out && B > 0 && T > 0, "attention_d512: bad arguments");
  K2_REQUIRE(ldq % 8 == 0 && ldo % 8 == 0 && q_off % 8 == 0 && k_off % 8 == 0 && v_off % 8 == 0 && ldo >= CH,
             "attention_d512: strides / offsets must be multiples of 8 elements");
  K2_REQUIRE(std::max(std::max(q_off, k_off), v_off) + CH <= ldq, "attention_d512: qkv row narrower than the offsets + 512");
  K2_REQUIRE((reinterpret_cast<uintptr_t>(qkv) & 15) == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0,
             "attention_d512: 16-byte alignment");
  FlashParams p;
  memset(&p, 0, sizeof p);
  p.qkv = reinterpret_cast<const __half*>(qkv);
  p.ldq = ldq; p.q_off = q_off; p.k_off = k_off; p.v_off = v_off;
  p.B = B; p.heads = 1; p.T = T;
  p.out = reinterpret_cast<__half*>(out);
  p.ldo = ldo;
  p.scale_log2e = scale * 1.4426950408889634f;
  int rc = launch_attention(p, CH, static_cast<cudaStream_t>(stream));
  if (rc == 0) count_launch();
  return rc;
}
