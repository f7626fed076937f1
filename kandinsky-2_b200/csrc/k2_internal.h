// k2_internal.h -- declarations shared between the kernel translation units and the C-ABI layer.
#pragma once
#include <cuda.h>
#include <cuda_fp16.h>
#include <cuda_runtime.h>
#include <stdint.h>

#include <string>

namespace k2 {

// ---- error plumbing (no exceptions cross the C ABI) ---------------------------------------------
void set_error(const std::string& msg);
int fail(const std::string& msg);  // records msg, returns -1
#define K2_CHECK_CUDA(expr)                                                                 \
  do {                                                                                      \
    cudaError_t _e = (expr);                                                                \
    if (_e != cudaSuccess)                                                                  \
      return ::k2::fail(std::string(#expr) + ": " + cudaGetErrorString(_e));                \
  } while (0)
#define K2_REQUIRE(cond, msg)                                  \
  do {                                                         \
    if (!(cond)) return ::k2::fail(std::string("k2b200: ") + (msg)); \
  } while (0)

// True when p may be accessed with 16-byte (uint4 / float4) vector loads and stores; null counts as aligned (optional
// arguments are checked for presence separately).
inline bool aligned16(const void* p) { return (reinterpret_cast<uintptr_t>(p) & 15) == 0; }

int num_sms();
bool pdl_enabled();

// Launch with (optionally) the programmatic-stream-serialization attribute. ONLY for kernels that call pdl_wait().
template <typename... KArgs, typename... Args>
inline cudaError_t launch_k(void (*kernel)(KArgs...), dim3 grid, dim3 block, size_t smem, cudaStream_t stream,
                            Args&&... args) {
  cudaLaunchConfig_t cfg = {};
  cfg.gridDim = grid;
  cfg.blockDim = block;
  cfg.dynamicSmemBytes = smem;
  cfg.stream = stream;
  cudaLaunchAttribute attr[1];
  attr[0].id = cudaLaunchAttributeProgrammaticStreamSerialization;
  attr[0].val.programmaticStreamSerializationAllowed = 1;
  cfg.attrs = attr;
  cfg.numAttrs = pdl_enabled() ? 1 : 0;
  return cudaLaunchKernelEx(&cfg, kernel, static_cast<KArgs>(args)...);
}
void count_launch(int n = 1);  // bump the library-wide kernel launch counter

// ---- TMA tensor-map encoding (driver entry point fetched at run time; no libcuda link) ----------
// fp16 tensor, rank<=4, 128B swizzle, inner box dim must be 64 elements (=128 bytes).
int encode_tmap_f16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes /* rank-1 */, const uint32_t* box);

// ---- implicit-GEMM convolution / GEMM (k2_conv_gemm.cu) -----------------------------------------
struct ConvGemmParams {
  CUtensorMap tmA[3];  // activation sources, 4-D (C, W, H, N)
  CUtensorMap tmB;     // packed weights, 3-D (Ktot, Cout_rows, batch), K contiguous; batch = 1 unless w_batched
  int w_batched;       // 1: image n of the NB images multiplies its own weight matrix (batched GEMM; tiles never span images)
  int seg_taps[3];     // 9 (3x3, pad 1), 1 (1x1) or 0 (unused)
  int seg_kchunks[3];  // 64-channel chunks per tap
  int num_k_chunks;
  int NB, H, W;        // output geometry
  int TN, TH, TW;      // rows of one M tile = TN*TH*TW <= 128 (a TMA box)
  int tiles_n, tiles_h, tiles_w;
  int m_tiles, n_tiles;
  int Cout;            // logical output channels
  const float* bias;   // [Cout] or nullptr
  const __half* residual;  // [M, ldr] or nullptr (added after bias)
  int ldr;
  void* out;
  int ldo;
  int out_mode;        // 0: fp16 [M, ldo] rows (NHWC); 1: fp32 NCHW [NB, Cout, H, W]; 2: split-K fp32 partials -> ws
  uint32_t a_box_bytes;
  int splits;          // split-K factor (1 = off)
  int k_per_split;     // K chunks per split
  float* ws;           // [splits][M_total][Cout] fp32 partial sums (out_mode 2)
  long long M_total;
  float2* gn_part;     // fused GroupNorm partials (sum, sumsq) of the fp16-rounded output, or null:
  int gn_mode;         //   1: [m_tiles][Cout], one per M tile (TN == 1); 2: [image][spatial tile][Cout] for 16-pixel x 8-image tiles
  int up2;             // 1: source 0 has taps == 4: 3x3 conv over the nearest-2x upsampled source as four 2x2 phase convs;
                       //    NB/H/W and the tile box are SOURCE geometry, outputs go to pixel (2y + a, 2x + b) of a 2H x 2W image
  int m_tiles_phase;   // up2: tile slots per phase (m_tiles = 4 * m_tiles_phase)
  const int* w_map;    // w_batched only, or null: image n multiplies weight slab w_map[n] of tmB's n_slabs instead of slab n
};
int launch_conv_gemm(const ConvGemmParams& p, int BN, cudaStream_t stream);
int launch_splitk_finalize(const float* ws, int splits, long long M, int Cout, const float* bias, const __half* residual,
                           int ldr, __half* out, int ldo, float2* gn_part, cudaStream_t stream);

// ---- fused attention, head dim 64 / 104 / 512 (k2_attention.cu) ----------------------------------
struct FlashParams {
  const __half* qkv;   // [B, T, ldq] rows; head h reads q / k / v at channels h*hs + {q,k,v}_off
  long long ldq;
  int hs, q_off, k_off, v_off;
  const __half* enc;   // [B, Tc, lde] encoder rows (keys 0 .. Tc-1 come first), or null with Tc = 0
  long long lde;
  int ehs, ek_off, ev_off;
  int B, heads, T, Tc;
  __half* out;         // [B, T, ldo], head h at channels h*ohs
  int ldo, ohs;
  float scale_log2e;   // softmax scale * log2(e)
};
int gn_apply_blocks_per_sm();  // tuning key 11: blocks per SM the GroupNorm apply kernels are sized for (0 = their occupancy)
int launch_attention(const FlashParams& p, int head_dim, cudaStream_t stream);

}  // namespace k2
