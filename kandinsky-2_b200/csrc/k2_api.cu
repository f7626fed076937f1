// k2_api.cu -- C-ABI plumbing: error state, launch counter, TMA descriptor encoding, and the
// k2_conv_gemm entry point (geometry selection + tensor maps) declared in include/k2b200.h.
#include <stdio.h>
#include <stdlib.h>
#include <string.h>

#include <algorithm>
#include <atomic>
#include <mutex>

#include "../../include/k2b200.h"
#include "k2_internal.h"

namespace k2 {

static thread_local std::string g_err;
static std::atomic<long long> g_launches{0};
static int g_force_bn = 0;
static int g_force_split = 0;  // 0 auto, 1 off, n>1 forced
static int g_pdl = 0;          // programmatic dependent launch of the step's kernels


void set_error(const std::string& msg) { g_err = msg; }
int fail(const std::string& msg) {
  g_err = msg;
  return -1;
}
void count_launch(int n) { g_launches.fetch_add(n, std::memory_order_relaxed); }

bool pdl_enabled() { return g_pdl != 0; }
static int g_gn_bps = 0;
int gn_apply_blocks_per_sm() { return g_gn_bps; }

int num_sms() {
  static int n = 0;
  if (n == 0) {
    int dev = 0;
    cudaGetDevice(&dev);
    cudaDeviceGetAttribute(&n, cudaDevAttrMultiProcessorCount, dev);
    if (n <= 0) n = 132;  // H100 SXM
  }
  return n;
}

typedef CUresult (*EncodeTiledFn)(CUtensorMap*, CUtensorMapDataType, cuuint32_t, void*, const cuuint64_t*,
                                  const cuuint64_t*, const cuuint32_t*, const cuuint32_t*,
                                  CUtensorMapInterleave, CUtensorMapSwizzle, CUtensorMapL2promotion,
                                  CUtensorMapFloatOOBfill);

static EncodeTiledFn get_encode_fn() {
  static EncodeTiledFn fn = nullptr;
  static std::once_flag once;
  std::call_once(once, [] {
    void* p = nullptr;
    cudaDriverEntryPointQueryResult qres;
    cudaError_t e = cudaGetDriverEntryPoint("cuTensorMapEncodeTiled", &p, cudaEnableDefault, &qres);
    if (e == cudaSuccess && qres == cudaDriverEntryPointSuccess) fn = reinterpret_cast<EncodeTiledFn>(p);
  });
  return fn;
}

int encode_tmap_f16(CUtensorMap* out, const void* base, int rank, const uint64_t* dims,
                    const uint64_t* strides_bytes, const uint32_t* box) {
  EncodeTiledFn fn = get_encode_fn();
  if (!fn) return fail("cuTensorMapEncodeTiled unavailable (no CUDA driver)");
  cuuint64_t gdim[5];
  cuuint64_t gstr[4];
  cuuint32_t bx[5];
  cuuint32_t es[5];
  for (int i = 0; i < rank; ++i) {
    gdim[i] = dims[i];
    bx[i] = box[i];
    es[i] = 1;
  }
  for (int i = 0; i + 1 < rank; ++i) gstr[i] = strides_bytes[i];
  CUresult r = fn(out, CU_TENSOR_MAP_DATA_TYPE_FLOAT16, static_cast<cuuint32_t>(rank), const_cast<void*>(base),
                  gdim, gstr, bx, es, CU_TENSOR_MAP_INTERLEAVE_NONE, CU_TENSOR_MAP_SWIZZLE_128B,
                  CU_TENSOR_MAP_L2_PROMOTION_L2_256B, CU_TENSOR_MAP_FLOAT_OOB_FILL_NONE);
  if (r != CUDA_SUCCESS) {
    char buf[256];
    snprintf(buf, sizeof buf,
             "cuTensorMapEncodeTiled failed (%d): rank %d dims %llu %llu %llu %llu box %u %u %u %u base %p",
             static_cast<int>(r), rank, (unsigned long long)dims[0], (unsigned long long)(rank > 1 ? dims[1] : 0),
             (unsigned long long)(rank > 2 ? dims[2] : 0), (unsigned long long)(rank > 3 ? dims[3] : 0), box[0],
             rank > 1 ? box[1] : 0, rank > 2 ? box[2] : 0, rank > 3 ? box[3] : 0, base);
    return fail(buf);
  }
  return 0;
}

// Pick the (TN, TH, TW) output box of one M tile (<= 128 pixels = the rows of one MMA tile): minimise the number of
// tiles.  Boxes may span several images (TN > 1) when that packs at least 15 % fewer tiles than the best single-image
// box -- e.g. 12x12 latents, 8 images: 8 images x 4 x 4 pixels = 128 rows per tile, 9 tiles with every MMA row used,
// instead of 1 image x 6 rows x 12 (16 tiles, 56 % used).  Single-image boxes are preferred otherwise because the fused
// GroupNorm statistics of the epilogue need them.
static void choose_tile(int NB, int H, int W, int& TN, int& TH, int& TW, bool single_image_only = false) {
  long long best_tiles[2] = {-1, -1};  // [0]: TN == 1 only, [1]: any TN
  int bn[2] = {1, 1}, bw[2] = {1, 1}, bh[2] = {1, 1};
  const int wmax = W < 128 ? W : 128;
  for (int tw = 1; tw <= wmax; ++tw) {
    const long long tiles_w = (W + tw - 1) / tw;
    for (int tn = 1; tn <= NB && tn * tw <= 128; ++tn) {
      int thmax = 128 / (tw * tn);
      if (thmax > H) thmax = H;
      if (thmax < 1) continue;
      const long long tiles_h = (H + thmax - 1) / thmax;
      const int th = static_cast<int>((H + tiles_h - 1) / tiles_h);  // balanced
      const long long tiles = tiles_h * tiles_w * ((NB + tn - 1) / tn);
      for (int k = (tn == 1 ? 0 : 1); k < 2; ++k) {
        bool better = best_tiles[k] < 0 || tiles < best_tiles[k];
        if (!better && tiles == best_tiles[k]) {
          // ties: fewer images per box, then the squarer box, then the wider
          if (tn != bn[k]) {
            better = tn < bn[k];
          } else {
            const int d_new = tw > th ? tw - th : th - tw;
            const int d_old = bw[k] > bh[k] ? bw[k] - bh[k] : bh[k] - bw[k];
            better = (d_new < d_old) || (d_new == d_old && tw > bw[k]);
          }
        }
        if (better) {
          best_tiles[k] = tiles;
          bn[k] = tn;
          bw[k] = tw;
          bh[k] = th;
        }
      }
    }
  }
  const int k = (!single_image_only && best_tiles[1] * 100 <= best_tiles[0] * 85) ? 1 : 0;
  TN = bn[k];
  TW = bw[k];
  TH = bh[k];
}


// Everything k2_conv_gemm decides before it touches a pointer: the M tile box, N tile, split-K factor and how the fused
// GroupNorm partials come out.  Pure host arithmetic (k2_conv_plan exposes it for tests and tooling).
struct ConvPlan {
  int TN, TH, TW, tiles_w, tiles_h, tiles_n, m_tiles;
  int m_tiles_phase;  // up2: tile slots per output phase
  int BN, splits;
  int fuse_stats, row_groups;
};

// cfg (may be null): per-call overrides {N tile, CTA-pair mode (0 / 1 = single CTA, the only kernel on sm_90), split-K factor,
// epilogue warp sets (ignored: every consumer warp drains its own rows)}; 0 = the process-wide tuning knob, else automatic.  The caller's launch plan bakes its choice per launch (kandinsky2/model/unet.py).
static void plan_conv(int NB, int H, int W, bool any9, int kchunks, int Cout, int out_mode, bool has_workspace,
                      long long workspace_bytes, bool want_gn, ConvPlan& pl, const int* cfg = nullptr, bool up2 = false,
                      bool w_batched = false) {
  // up2: NB/H/W are the SOURCE geometry; every box is visited once per output phase (4x the tiles, same K loop)
  const int g_force_bn = (cfg && cfg[0]) ? cfg[0] : k2::g_force_bn;
  const int g_force_split = (cfg && cfg[2]) ? cfg[2] : k2::g_force_split;
  choose_tile(NB, H, W, pl.TN, pl.TH, pl.TW, w_batched);
  pl.tiles_w = (W + pl.TW - 1) / pl.TW;
  pl.tiles_h = (H + pl.TH - 1) / pl.TH;
  pl.tiles_n = (NB + pl.TN - 1) / pl.TN;
  pl.m_tiles = pl.tiles_w * pl.tiles_h * pl.tiles_n;
  pl.m_tiles_phase = pl.m_tiles;

  // Tile width N and split-K factor from a cycle model of the sm_90 kernel (its MMA and operand rates, not a fit to
  // measurements): one K chunk of a 128 x BN x 64 work unit costs 4*BN + 60 cycles (2048 fp16 FMA/clk/SM, the operand
  // stream of 16 KB + BN*128 B per chunk stays below that at BN >= 128), a unit adds ~2000 cycles of exposed prologue /
  // epilogue, the launch takes ceil(units / SMs) waves of those, and a split-K launch pays the second pass (fixed ~4000
  // cycles + its traffic at ~1800 B/cycle of HBM).  Among the N tiles the model picks 192 / 128 where they divide Cout better
  // or give a fuller last wave, and splits K only where the tile count would leave most SMs idle.
  int BN = g_force_bn;
  int splits = 1;
  const long long M_total = static_cast<long long>(NB) * H * W;
  const bool can_split = !up2 && !w_batched && has_workspace && out_mode == 0 && Cout % 8 == 0;
  auto split_ok = [&](int sp) {
    if (sp == 1) return true;
    const int kps = (kchunks + sp - 1) / sp;
    return can_split && kps >= 8 && (sp - 1) * kps < kchunks &&
           static_cast<long long>(sp) * M_total * Cout * 4 <= workspace_bytes;
  };
  auto model = [&](int bn, int sp) {
    const long long nt = (Cout + bn - 1) / bn;
    const long long units = static_cast<long long>(pl.m_tiles) * nt * sp * (up2 ? 4 : 1);
    const long long slots = num_sms();
    const long long waves = (units + slots - 1) / slots;
    const long long kps = (kchunks + sp - 1) / sp;
    long long cost = waves * (kps * (4LL * bn + 60) + 2000);
    if (sp > 1) cost += 4000 + (static_cast<long long>(sp) + 1) * M_total * Cout * 4 / 1800;
    return cost;
  };
  if (BN == 0) {
    if (Cout <= 16) BN = 16;
    else if (Cout <= 64) BN = 64;
    else if (Cout <= 128) BN = 128;
    else BN = 0;  // chosen below together with the split factor
  }
  {
    const int cand[3] = {256, 192, 128};
    long long best = -1;
    int best_bn = BN ? BN : 256, best_sp = 1;
    for (int ci = 0; ci < 3; ++ci) {
      const int bn = BN ? BN : cand[ci];
      if (BN && ci > 0) break;
      for (int sp = 1; sp <= 8; ++sp) {
        if (g_force_split > 0 && sp != g_force_split) continue;
        if (!split_ok(sp)) continue;
        const long long c = model(bn, sp);
        if (best < 0 || c < best) {  // ties keep the wider tile / the smaller split (visited first)
          best = c;
          best_bn = bn;
          best_sp = sp;
        }
      }
    }
    BN = best_bn;
    splits = best_sp;
  }
  pl.BN = BN;
  pl.splits = splits;

  // fused GroupNorm partial statistics: from the epilogue when a tile never straddles two images (one partial per M
  // tile: the epilogue folds its four warps) or when it holds 16 pixels of each of 8 images (one partial per (image,
  // spatial tile): every half warp of the epilogue holds exactly one image's pixels); split-K launches produce them in
  // the second pass instead, as 16-row groups of the flat pixel order
  pl.fuse_stats = 0;
  pl.row_groups = 0;
  if (want_gn && out_mode == 0 && Cout % 8 == 0) {
    if (splits == 1 && BN >= 64 && Cout % 64 == 0 && (pl.TN == 1 || pl.TH * pl.TW == 16)) {
      pl.fuse_stats = 1;
      pl.row_groups = ((pl.TN == 1) ? pl.m_tiles : NB * pl.tiles_h * pl.tiles_w) * (up2 ? 4 : 1);
    } else if (splits > 1 && (static_cast<long long>(H) * W) % 16 == 0) {
      pl.fuse_stats = 2;
      pl.row_groups = static_cast<int>(M_total / 16);
    }
  }
}

static void plan_to_info(const ConvPlan& pl, int* info) {
  if (!info) return;
  info[0] = pl.BN; info[1] = 0;  // CTA-pair mode: there is no CTA-pair kernel on sm_90
  info[2] = pl.splits; info[3] = pl.m_tiles; info[4] = pl.TN;
  info[5] = pl.fuse_stats; info[6] = pl.row_groups;
}

}  // namespace k2

using namespace k2;

extern "C" {

const char* k2_last_error(void) { return g_err.c_str(); }
int k2_version(void) { return 100; }
long long k2_launch_count(void) { return g_launches.load(); }
void k2_reset_launch_count(void) { g_launches.store(0); }
int k2_set_tuning(int key, int value) {
  if (key == 0) {
    g_force_bn = value;
    return 0;
  }
  if (key == 1) {
    g_force_split = value;
    return 0;
  }
  if (key == 2) {  // CTA-pair mode: 0 auto / 1 off are the same single-CTA kernel; sm_90 has no CTA-pair MMA
    if (value == 2) return fail("k2_set_tuning: no CTA-pair conv kernel on sm_90");
    return 0;
  }
  if (key == 4) {
    g_pdl = value;
    return 0;
  }
  if (key == 10) {  // accepted and ignored: both consumer warpgroups of the conv kernel always drain their own rows
    return 0;
  }
  if (key == 11) {  // GroupNorm apply: blocks per SM the grid is sized for (0 = the kernel's occupancy; round 1 used 4)
    g_gn_bps = value;
    return 0;
  }
  if (key == 9) {  // accepted and ignored: the head-width-64 attention kernel has a single CTA layout (128 query rows)
    return 0;
  }

  return fail("k2_set_tuning: unknown key");
}

int k2_conv_gemm(const K2ConvSrc* srcs, int nsrc, int NB, int H, int W, const void* w_packed, int w_rows,
                 int Ktot, int ldw, int Cout, const float* bias, const void* residual, int ldr, void* out, int ldo,
                 int out_mode, void* workspace, long long workspace_bytes, float* gn_partial, int* info,
                 k2_stream_t stream) {
  return k2_conv_gemm_cfg(srcs, nsrc, NB, H, W, w_packed, w_rows, Ktot, ldw, Cout, bias, residual, ldr, out, ldo, out_mode,
                          workspace, workspace_bytes, gn_partial, info, nullptr, 0, stream);
}

}  // extern "C"

// k2_conv_gemm_cfg, and k2_conv_gemm_wmap when w_map is not null (n_slabs >= 1, checked by the caller)
static int conv_gemm_impl(const K2ConvSrc* srcs, int nsrc, int NB, int H, int W, const void* w_packed, int w_rows, int Ktot,
                          int ldw, int Cout, const float* bias, const void* residual, int ldr, void* out, int ldo, int out_mode,
                          void* workspace, long long workspace_bytes, float* gn_partial, int* info, const int* cfg,
                          long long w_batch_stride, int n_slabs, const int* w_map, k2_stream_t stream) {
  K2_REQUIRE(w_batch_stride >= 0 && w_batch_stride % 8 == 0, "conv_gemm_cfg: w_batch_stride must be a multiple of 8 elements");
  // out_mode 2 (raw fp32 split-K partials into the workspace) is internal: the split-K plan sets it and adds the finalize pass
  K2_REQUIRE(out_mode == 0 || out_mode == 1, "conv_gemm: out_mode must be 0 (fp16 rows) or 1 (fp32 NCHW)");
  K2_REQUIRE(out_mode == 0 || residual == nullptr, "conv_gemm: out_mode 1 (fp32 NCHW) takes no residual");
  const bool w_batched = w_batch_stride > 0;
  if (cfg) {
    K2_REQUIRE(cfg[0] == 0 || cfg[0] == 16 || cfg[0] == 64 || cfg[0] == 128 || cfg[0] == 192 || cfg[0] == 256,
               "conv_gemm_cfg: N tile must be 0, 16, 64, 128, 192 or 256");
    K2_REQUIRE(cfg[1] >= 0 && cfg[1] <= 2 && cfg[2] >= 0 && cfg[2] <= 8 && cfg[3] >= 0 && cfg[3] <= 2,
               "conv_gemm_cfg: pair mode in 0..2, splits in 0..8, epilogue sets in 0..2");
    K2_REQUIRE(cfg[1] != 2, "conv_gemm_cfg: no CTA-pair conv kernel on sm_90");
  }
  K2_REQUIRE(nsrc >= 1 && nsrc <= 3, "conv_gemm: 1..3 sources");
  K2_REQUIRE((reinterpret_cast<uintptr_t>(gn_partial) & 7) == 0, "conv_gemm: gn_partial must be 8-byte aligned");
  K2_REQUIRE(NB > 0 && H > 0 && W > 0 && Cout > 0, "conv_gemm: bad geometry");
  K2_REQUIRE(w_rows >= Cout, "conv_gemm: w_rows < Cout");
  K2_REQUIRE(Ktot % 64 == 0, "conv_gemm: Ktot must be a multiple of 64");
  if (ldw == 0) ldw = Ktot;
  K2_REQUIRE(ldw >= Ktot && ldw % 8 == 0 && (reinterpret_cast<uintptr_t>(w_packed) & 15) == 0,
             "conv_gemm: weight row stride / alignment");
  if (out_mode == 0) {
    K2_REQUIRE(ldo % 8 == 0 && (reinterpret_cast<uintptr_t>(out) & 15) == 0, "conv_gemm: out alignment");
    if (residual)
      K2_REQUIRE(ldr % 8 == 0 && (reinterpret_cast<uintptr_t>(residual) & 15) == 0, "conv_gemm: residual alignment");
  }
  ConvGemmParams p;
  memset(&p, 0, sizeof p);
  p.NB = NB;
  p.H = H;
  p.W = W;
  bool any9 = false;
  int kchunks = 0;
  const bool up2 = srcs[0].taps == 4;
  if (up2) {
    K2_REQUIRE(nsrc == 1 && out_mode == 0 && residual == nullptr && H % 2 == 0 && W % 2 == 0,
               "conv_gemm: a taps == 4 source (3x3 conv over its nearest-2x upsampling) must be the only source, with fp16 "
               "output, no residual and even output H, W");
    H /= 2;  // from here on: SOURCE geometry (the tile boxes live there)
    W /= 2;
    p.H = H;
    p.W = W;
  }
  for (int s = 0; s < nsrc; ++s) {
    const K2ConvSrc& src = srcs[s];
    K2_REQUIRE(src.taps == 9 || src.taps == 1 || (s == 0 && src.taps == 4), "conv_gemm: taps must be 9 or 1 (or 4: up2)");
    K2_REQUIRE(src.C > 0 && src.C % 8 == 0 && src.ld % 8 == 0 && src.ld >= src.C, "conv_gemm: bad source C/ld");
    K2_REQUIRE((reinterpret_cast<uintptr_t>(src.ptr) & 15) == 0, "conv_gemm: source not 16B aligned");
    any9 = any9 || src.taps == 9;
    p.seg_taps[s] = src.taps;
    p.seg_kchunks[s] = (src.C + 63) / 64;
    kchunks += src.taps * p.seg_kchunks[s];
  }
  K2_REQUIRE(kchunks * 64 * (up2 ? 4 : 1) == Ktot,
             "conv_gemm: Ktot does not match the sources (taps * ceil(C/64)*64 summed; x4 phases for a taps == 4 source)");
  p.num_k_chunks = kchunks;

  ConvPlan pl;
  plan_conv(NB, H, W, any9 || up2, kchunks, Cout, out_mode, workspace != nullptr, workspace_bytes, gn_partial != nullptr, pl,
            cfg, up2, w_batched);
  K2_REQUIRE(!w_batched || (!up2 && pl.TN == 1), "conv_gemm_cfg: batched weights need single-image tiles");
  p.w_batched = w_batched ? 1 : 0;
  p.w_map = w_map;
  plan_to_info(pl, info);
  p.TN = pl.TN;
  p.TH = pl.TH;
  p.TW = pl.TW;
  p.tiles_w = pl.tiles_w;
  p.tiles_h = pl.tiles_h;
  p.tiles_n = pl.tiles_n;
  p.m_tiles = up2 ? 4 * pl.m_tiles_phase : pl.m_tiles;
  p.m_tiles_phase = pl.m_tiles_phase;
  p.up2 = up2 ? 1 : 0;
  p.a_box_bytes = static_cast<uint32_t>(p.TN * p.TH * p.TW * 128);
  for (int s = 0; s < nsrc; ++s) {
    const K2ConvSrc& src = srcs[s];
    uint64_t dims[4] = {static_cast<uint64_t>(src.C), static_cast<uint64_t>(W), static_cast<uint64_t>(H),
                        static_cast<uint64_t>(NB)};
    uint64_t str[3] = {static_cast<uint64_t>(src.ld) * 2, static_cast<uint64_t>(src.ld) * 2 * W,
                       static_cast<uint64_t>(src.ld) * 2 * W * H};
    uint32_t box[4] = {64, static_cast<uint32_t>(p.TW), static_cast<uint32_t>(p.TH), static_cast<uint32_t>(p.TN)};
    if (encode_tmap_f16(&p.tmA[s], src.ptr, 4, dims, str, box)) return -1;
  }
  const int BN = pl.BN, splits = pl.splits, fuse_stats = pl.fuse_stats;
  p.splits = splits;
  p.k_per_split = (kchunks + splits - 1) / splits;
  p.M_total = static_cast<long long>(NB) * H * W * (up2 ? 4 : 1);
  p.ws = reinterpret_cast<float*>(workspace);
  p.n_tiles = (Cout + BN - 1) / BN;
  p.Cout = Cout;
  {
    const int slabs = w_map ? n_slabs : (w_batched ? NB : 1);
    uint64_t dims[3] = {static_cast<uint64_t>(Ktot), static_cast<uint64_t>(w_rows), static_cast<uint64_t>(slabs)};
    uint64_t str[2] = {static_cast<uint64_t>(ldw) * 2,
                       (w_batched ? static_cast<uint64_t>(w_batch_stride) : static_cast<uint64_t>(ldw) * w_rows) * 2};
    uint32_t box[3] = {64, static_cast<uint32_t>(BN), 1};
    if (encode_tmap_f16(&p.tmB, w_packed, 3, dims, str, box)) return -1;
  }
  p.bias = bias;
  p.residual = reinterpret_cast<const __half*>(residual);
  p.ldr = ldr;
  p.out = out;
  p.ldo = ldo;
  p.out_mode = (splits > 1) ? 2 : out_mode;
  p.gn_part = (fuse_stats == 1) ? reinterpret_cast<float2*>(gn_partial) : nullptr;
  p.gn_mode = (fuse_stats == 1) ? (p.TN == 1 ? 1 : 2) : 0;
  int rc = launch_conv_gemm(p, BN, static_cast<cudaStream_t>(stream));
  if (rc == 0) g_launches.fetch_add(1, std::memory_order_relaxed);
  if (rc == 0 && splits > 1) {
    rc = launch_splitk_finalize(p.ws, splits, p.M_total, Cout, bias, p.residual, ldr, reinterpret_cast<__half*>(out), ldo,
                                fuse_stats == 2 ? reinterpret_cast<float2*>(gn_partial) : nullptr,
                                static_cast<cudaStream_t>(stream));
    if (rc == 0) g_launches.fetch_add(1, std::memory_order_relaxed);
  }
  return rc;
}

extern "C" {

int k2_conv_gemm_cfg(const K2ConvSrc* srcs, int nsrc, int NB, int H, int W, const void* w_packed, int w_rows,
                     int Ktot, int ldw, int Cout, const float* bias, const void* residual, int ldr, void* out, int ldo,
                     int out_mode, void* workspace, long long workspace_bytes, float* gn_partial, int* info,
                     const int* cfg, long long w_batch_stride, k2_stream_t stream) {
  return conv_gemm_impl(srcs, nsrc, NB, H, W, w_packed, w_rows, Ktot, ldw, Cout, bias, residual, ldr, out, ldo, out_mode,
                        workspace, workspace_bytes, gn_partial, info, cfg, w_batch_stride, 0, nullptr, stream);
}

int k2_conv_gemm_wmap(const K2ConvSrc* srcs, int nsrc, int NB, int H, int W, const void* w_packed, int w_rows,
                      int Ktot, int ldw, int Cout, const float* bias, const void* residual, int ldr, void* out, int ldo,
                      int out_mode, void* workspace, long long workspace_bytes, float* gn_partial, int* info,
                      const int* cfg, long long w_batch_stride, int n_slabs, const int* w_map, k2_stream_t stream) {
  K2_REQUIRE(w_map != nullptr, "conv_gemm_wmap: null w_map");
  K2_REQUIRE((reinterpret_cast<uintptr_t>(w_map) & 3) == 0, "conv_gemm_wmap: w_map must be 4-byte aligned");
  K2_REQUIRE(n_slabs >= 1, "conv_gemm_wmap: n_slabs must be >= 1");
  K2_REQUIRE(w_batch_stride > 0, "conv_gemm_wmap: w_batch_stride must be > 0 (the elements between two slabs)");
  K2_REQUIRE(srcs != nullptr && w_packed != nullptr && out != nullptr, "conv_gemm_wmap: null source, weight or output");
  return conv_gemm_impl(srcs, nsrc, NB, H, W, w_packed, w_rows, Ktot, ldw, Cout, bias, residual, ldr, out, ldo, out_mode,
                        workspace, workspace_bytes, gn_partial, info, cfg, w_batch_stride, n_slabs, w_map, stream);
}

int k2_conv_plan(int NB, int H, int W, int taps, int Ktot, int Cout, int out_mode, long long workspace_bytes,
                 int want_gn_partial, int* info) {
  K2_REQUIRE(NB > 0 && H > 0 && W > 0 && Cout > 0 && info, "conv_plan: bad arguments");
  K2_REQUIRE(Ktot > 0 && Ktot % 64 == 0, "conv_plan: Ktot must be a positive multiple of 64");
  ConvPlan pl;
  plan_conv(NB, H, W, taps == 9, Ktot / 64, Cout, out_mode, workspace_bytes > 0, workspace_bytes, want_gn_partial != 0, pl);
  plan_to_info(pl, info);
  return 0;
}

}  // extern "C"
