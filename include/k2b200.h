/* k2b200.h -- C ABI of libk2b200.so, the H100 (sm_90a) kernel library behind the Kandinsky-2
 * denoising hot path.
 *
 * The reference (ai-forever/Kandinsky-2) has no FFI: its "operator API" for this path is the set of
 * PyTorch library calls issued by kandinsky2/model/unet.py, kandinsky2/model/nn.py,
 * kandinsky2/model/gaussian_diffusion.py and kandinsky2/vqgan/movq_modules.py.  Each entry point
 * below replaces one such call-site family (cited per function) and is what the Python boundary
 * modules in kandinsky-2_b200/kandinsky2/ bind through ctypes (see INTEGRATION.md).
 *
 * Conventions
 *   - every function returns 0 on success and <0 on error; k2_last_error() gives the thread-local
 *     message; no C++ exception crosses the boundary;
 *   - all pointers are DEVICE pointers unless a parameter is documented as host memory; the library
 *     never allocates user-visible memory and never synchronises the device;
 *   - every launch is enqueued on the caller's stream (pass torch.cuda.current_stream().cuda_stream);
 *   - activations are NHWC fp16 ("rows" = pixels, row stride `ld*` in ELEMENTS so that a tensor may
 *     be a channel slice of a wider buffer); weights are pre-packed by the host (layout per function);
 *   - kernels that move fp16 rows as 16-byte vectors need 16-byte aligned pointers, row strides that are multiples of 8
 *     elements and >= the row width; such calls are refused (< 0) before anything is launched;
 *   - there is no CPU fallback: without an sm_90 device every call fails.
 */
#ifndef K2B200_H_
#define K2B200_H_

#include <stdint.h>

#ifdef __cplusplus
extern "C" {
#endif

typedef void* k2_stream_t; /* cudaStream_t */

const char* k2_last_error(void);
int k2_version(void);
/* Number of kernels launched by this library in this process since the last reset (bench evidence). */
long long k2_launch_count(void);
void k2_reset_launch_count(void);
/* Tuning knobs: key 0 = force conv/GEMM N tile (0 = auto); key 1 = split-K (0 auto, 1 off, n>1 forced);
 * key 2 = CTA-pair conv kernel (0 auto, 1 off; 2 = on is refused: sm_90 has no CTA-pair MMA);
 * key 4 = programmatic dependent launch (0/1); key 9 = accepted for compatibility and ignored (it chose between two CTA
 * layouts of an earlier head-width-64 attention kernel; the current one has one); key 10 = accepted for compatibility and
 * ignored (it chose how many consumer warpgroups drained the conv kernel's accumulators; every consumer warp now drains its
 * own rows).  Keys 0, 1 and 2 are process-wide defaults; k2_conv_gemm_cfg overrides them per call.
 * key 11 = blocks per SM the GroupNorm apply grids are sized for (0 = each kernel's real occupancy, i.e. one full wave). */
int k2_set_tuning(int key, int value);

/* ---------------------------------------------------------------------------------------------
 * Convolution / GEMM on wgmma tensor cores.
 * Replaces nn.Conv2d 3x3 (unet.py:152,180,426,562; movq_modules.py:139-148), nn.Conv2d 1x1
 * (unet.py:191; movq_modules.py:150-157,188-199) and nn.Conv1d k=1 (unet.py:251,257,258).
 *
 *   out[m, n] = bias[n] + residual[m, n] + sum_s sum_tap sum_c A_s[shift_tap(m), c] * Wp[n, k(s,tap,c)]
 *
 * m runs over the NB*H*W output pixels (NHWC order).  Up to 3 activation sources accumulate into the
 * same output; source s has `taps` = 9 (3x3, zero padding 1) or 1 (1x1).  Packed weights Wp are fp16
 * [w_rows >= Cout][Ktot], K contiguous, k ordered source-major, then tap (ky*3+kx), then channel, each
 * source's channel count padded to a multiple of 64 (zero weights for the padding).
 * out_mode 0: fp16 rows [M, ldo]; out_mode 1: fp32 NCHW [NB, Cout, H, W] (output heads), which takes no residual
 * (residual must be NULL); any other out_mode is refused.  Both checks happen before any CUDA call.
 * ldw is the row stride of Wp in elements (0 = Ktot); a strided Wp lets an ACTIVATION matrix be the B operand
 * (MoVQ attention: scores = q k^T with k rows as "weights").
 * workspace (may be NULL): caller-owned scratch for split-K.  Where a cycle model of the launch (waves of work units x
 * K chunks per unit, plus the second pass) says so -- small M with a huge K -- K is split over several CTAs that write
 * fp32 partial tiles [split][M][Cout] there, and a second launch sums them in a fixed order (+bias, +residual) --
 * deterministic, no atomics.  Launches sharing a workspace must be stream-ordered.
 * gn_partial (may be NULL): fp32 [row groups][Cout][2]; when given and the launch qualifies (fp16 output, Cout % 64 == 0,
 * N tile >= 64) the launch also emits (sum, sum of squares) partials of the ROUNDED output, image-major, which
 * k2_gn_finalize turns into GroupNorm statistics -- the consumer's statistics pass disappears.  Row groups: one per M tile
 * when a tile lies inside one image; one per (image, spatial tile) for the (16 pixel x 8 image) tiles of tiny images; 16-row
 * groups from the second pass of a split-K launch.  gn_partial must hold max(M tiles*4, M/16)*Cout*2 floats
 * (k2_gn_scratch_floats); info[5] / info[6] tell what was written.
 * info (HOST pointer, may be NULL): int[7] = {N tile, CTA-pair mode (always 0 on sm_90), split-K factor, M tiles, images per tile,
 * gn_partial written (0 no / 1 epilogue / 2 split-K pass), row groups written in total}.
 * taps = 4 (allowed for a single source, fp16 output, no residual, H and W even): the source is [NB, H/2, W/2, C] and the call
 * computes the 3x3 convolution over its NEAREST-2x UPSAMPLING (unet.py:67-77 + :199-203; movq_modules.py:93-97) without
 * materialising it: output pixel (2y+a, 2x+b) = a 2x2 convolution of the source around (y, x) with the kernel rows / columns
 * that fall on the same source pixel pre-summed by the host (2.25x fewer MACs).  Wp = fp16 [Cout][16 * pad64(C)],
 * k = ((a*2+b)*4 + ty*2+tx) * pad64(C) + c, source offset (ty+a-1, tx+b-1); Ktot = 16 * pad64(C).
 * A plain GEMM [M,K]x[K,N] is the call with NB=1, H=1, W=M, one source with taps=1.
 * ------------------------------------------------------------------------------------------- */
typedef struct {
  const void* ptr; /* fp16, NHWC; may point at a channel offset inside a wider buffer */
  int C;           /* channels of this source (multiple of 8) */
  int ld;          /* row stride in elements */
  int taps;        /* 9, 1, or 4 (3x3 over the nearest-2x upsampled source, see above) */
} K2ConvSrc;

int k2_conv_gemm(const K2ConvSrc* srcs, int nsrc, int NB, int H, int W, const void* w_packed, int w_rows,
                 int Ktot, int ldw, int Cout, const float* bias, const void* residual, int ldr, void* out, int ldo,
                 int out_mode, void* workspace, long long workspace_bytes, float* gn_partial, int* info,
                 k2_stream_t stream);

/* k2_conv_gemm with the launch configuration chosen by the caller instead of the library's cycle model:
 * cfg (HOST pointer, may be NULL = k2_conv_gemm) = int[4] {N tile (16/64/128/192/256), CTA-pair kernel (1 off; 2 is refused
 * on sm_90), split-K factor (1 = off), epilogue warp sets}; a 0 entry keeps the automatic choice.  The epilogue-sets
 * entry is checked (0, 1 or 2) and otherwise ignored: both consumer warpgroups always drain their own accumulator rows, so
 * 1 and 2 run the same kernel.  The N tile never changes a result bit (same K order per output element); the split factor does.
 * The UNet / MoVQ launch plans time the candidates once per distinct layer shape and bake the winner into their CUDA graph.
 * w_batch_stride (elements, multiple of 8; 0 = one weight matrix): > 0 makes the call a BATCHED GEMM -- image n of the NB
 * images multiplies Wp + n * w_batch_stride.  This is how the MoVQ AttnBlock (movq_modules.py:201-225) runs without a loop
 * over images: scores[n] = q[n] k[n]^T with the k rows of image n as "weights" (w_rows = T, ldw = row stride of the qkv
 * buffer), out[n] = P[n] v[n] with v[n]^T as "weights".  Tiles then never span two images; no split-K. */
int k2_conv_gemm_cfg(const K2ConvSrc* srcs, int nsrc, int NB, int H, int W, const void* w_packed, int w_rows,
                     int Ktot, int ldw, int Cout, const float* bias, const void* residual, int ldr, void* out, int ldo,
                     int out_mode, void* workspace, long long workspace_bytes, float* gn_partial, int* info,
                     const int* cfg, long long w_batch_stride, k2_stream_t stream);

/* k2_conv_gemm_cfg in batched mode with the weight matrix of each image CHOSEN: image n of the NB images multiplies slab
 * w_map[n] of n_slabs slabs, Wp + w_map[n] * w_batch_stride (w_batch_stride > 0).  w_map: DEVICE int32 [NB], read by the
 * kernel when it runs, so a captured CUDA graph follows the map's current contents.  Slabs may repeat and need not all be
 * used.  Bias, residual, fp16 / fp32 output and the fused GroupNorm partials are those of batched mode; tiles never span
 * images and K is never split.  A map entry outside [0, n_slabs) multiplies zeros (TMA's out-of-bounds fill); callers write
 * only valid entries.  The Kandinsky 2.2 batcher runs its attention projections this way, one adapter slab per request. */
int k2_conv_gemm_wmap(const K2ConvSrc* srcs, int nsrc, int NB, int H, int W, const void* w_packed, int w_rows,
                      int Ktot, int ldw, int Cout, const float* bias, const void* residual, int ldr, void* out, int ldo,
                      int out_mode, void* workspace, long long workspace_bytes, float* gn_partial, int* info,
                      const int* cfg, long long w_batch_stride, int n_slabs, const int* w_map, k2_stream_t stream);

/* The decisions k2_conv_gemm takes for a geometry -- M tile box, N tile, split-K factor, how the GroupNorm
 * partials come out -- without touching a pointer or the GPU (host arithmetic only; for tests, tooling and the caller's
 * scratch sizing).  taps: 9 if any source is a 3x3, else 1; Ktot as for k2_conv_gemm; workspace_bytes 0 = no workspace;
 * info = int[7] with the meaning given above. */
int k2_conv_plan(int NB, int H, int W, int taps, int Ktot, int Cout, int out_mode, long long workspace_bytes,
                 int want_gn_partial, int* info);

/* ---------------------------------------------------------------------------------------------
 * GroupNorm (32 groups in the UNet) statistics + fused apply.
 * Replaces GroupNorm32.forward (nn.py:31-37), the FiLM  norm(h)*(1+scale)+shift  and SiLU of
 * ResBlock.forward (unet.py:209-216), Upsample/Downsample on h and x (unet.py:67-77,105-107), the
 * torch.cat of the up path (text2im_model2_1.py:99) and MoVQ SpatialNorm (movq_modules.py:61-68).
 *
 * k2_gn_stats: per (image, group) mean and rstd of the channel-concatenation [src0 | src1]
 *   (src1 may be NULL); stats is fp32 [NB, groups, 2]; scratch is fp32 workspace of
 *   k2_gn_scratch_floats(NB, HW, C0+C1) floats that the caller ZEROES once at allocation (its first
 *   1024 words are self-resetting arrival counters); deterministic.
 * k2_gn_apply: y = act( ((x-mean)*rstd*gamma+beta) * (1+scale[n,c]) + shift[n,c] ), written as fp16
 *   rows of the concatenated tensor, optionally resampled:
 *     resample 0: same size; 1: 2x2 average pool of y (and of raw x into xres); 2: nearest 2x upsample.
 *   film is fp32 rows (scale[0..C) | shift[C..2C)) with row stride film_ld, or NULL.  act: 0 none, 1 SiLU.
 *   spatial (MoVQ): if zq != NULL, y = GN(x) * (Wy.zq + by) + (Wb.zq + bb) with zq fp32 NHWC
 *   [NB, zh, zw, 4] nearest-resized to (H, W); sn_w is fp32 [C, 10] = (Wy[4], by, Wb[4], bb).
 * ------------------------------------------------------------------------------------------- */
long long k2_gn_scratch_floats(int NB, int HW, int C);
int k2_gn_stats(const void* src0, int C0, int ld0, const void* src1, int C1, int ld1, int NB, int HW,
                int groups, float eps, float* stats, float* scratch, k2_stream_t stream);
/* statistics from the partials k2_conv_gemm wrote (one or two channel-concatenated sources of the same image size);
 * rg0 / rg1 = row groups per image of each source (info[6] / NB of the producing call). */
int k2_gn_finalize(const float* part0, int C0, int rg0, const float* part1, int C1, int rg1, int NB, int HW, int groups,
                   float eps, float* stats, k2_stream_t stream);
int k2_gn_apply(const void* src0, int C0, int ld0, const void* src1, int C1, int ld1, int NB, int H, int W,
                int groups, const float* stats, const float* gamma, const float* beta, const float* film,
                int film_ld, int act, int resample, void* y, int ldy, void* xres, int ldx, const float* zq, int zh,
                int zw, const float* sn_w, k2_stream_t stream);
/* k2_gn_apply with the statistics pass folded in: instead of `stats` the producers' partial sums (the part0 / rg0 / part1 / rg1
 * / eps arguments of k2_gn_finalize) are given and every block derives mean / rstd of the groups it touches itself -- one
 * launch less per GroupNorm.  No SpatialNorm inputs.  Statistics equal k2_gn_finalize's up to fp32 summation order
 * (tests/test_gpu_ops.py::test_gn_apply_fold_matches_finalize_plus_apply). */
int k2_gn_apply_fold(const void* src0, int C0, int ld0, const void* src1, int C1, int ld1, int NB, int H, int W, int groups,
                     const float* part0, int rg0, const float* part1, int rg1, float eps, const float* gamma,
                     const float* beta, const float* film, int film_ld, int act, int resample, void* y, int ldy, void* xres,
                     int ldx, k2_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Attention, head dim 64, online softmax, on wgmma tensor cores (QK^T and PV) with encoder K/V prepended.
 * Replaces QKVAttention.forward (unet.py:286-340) incl. the optional flash-attn path (:303-332).
 *   qkv   fp16 [B, T, ldq] rows; head h owns channels [h*hs, (h+1)*hs) with q at +q_off, k at +k_off,
 *         v at +v_off (reference layout: hs=192, 0/64/128 -- unet.py:296).
 *   enc   fp16 [B, Tc, lde] rows or NULL (Tc=0); head h: k at h*ehs+ek_off, v at h*ehs+ev_off.
 *   out   fp16 [B, T, ldo], channel h*64+d.
 *   scale multiplies q.k (reference: 1/sqrt(64), applied as d^-1/4 on each operand, unet.py:334-337).
 * ------------------------------------------------------------------------------------------- */
int k2_attention_d64(const void* qkv, int ldq, int hs, int q_off, int k_off, int v_off, const void* enc,
                     int lde, int ehs, int ek_off, int ev_off, int B, int heads, int T, int Tc, float scale,
                     void* out, int ldo, k2_stream_t stream);

/* One head of width 512 over T tokens, no [T, T] score matrix: the MoVQ AttnBlock (movq_modules.py:201-225; the encoder's
 * twin vqgan_blocks.py:186-240).  qkv fp16 rows [B, T, ldq] with q / k / v at element offsets q_off / k_off / v_off (512 channels
 * each); out fp16 [B, T, ldo] (512 channels); scale multiplies q.k (the reference: C ** -0.5).  A CTA owns 128 queries and half
 * of the output channels (an fp32 O row of 256 channels fills 128 registers per thread), so the score tile is computed twice
 * per query tile. */
int k2_attention_d512(const void* qkv, int ldq, int q_off, int k_off, int v_off, int B, int T, float scale, void* out, int ldo,
                      k2_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Small dense layers (fp32 math): nn.Linear (+ optional SiLU on the input and/or the output),
 * nn.LayerNorm, and the sinusoidal timestep embedding.
 * Replaces time_embed (unet.py:414-419), emb_layers (unet.py:166-172), the conditioning head
 * (text2im_model2_1.py:57-80) and timestep_embedding (nn.py:101-121).
 *   y[m, n] = (silu_out ? silu : id)( b[n] + sum_k (silu_in ? silu(x[m,k]) : x[m,k]) * W[n,k] ) (+ add[m,n])
 * x fp32 [M, K] (ldx), W fp16 or fp32 [N, K] (w_is_half), y fp32 [M, N] (ldy).
 * ------------------------------------------------------------------------------------------- */
int k2_linear(const float* x, int ldx, const void* W, int w_is_half, const float* b, const float* add,
              int ldadd, float* y, int ldy, int M, int N, int K, int silu_in, int silu_out,
              k2_stream_t stream);
int k2_layernorm(const float* x, const float* gamma, const float* beta, float* y, int M, int N, float eps,
                 k2_stream_t stream);
int k2_timestep_embedding(const float* t, float* out, int B, int dim, float max_period, k2_stream_t stream);
/* fp32 rows -> fp16 rows (context tokens), and generic strided copy helpers */
int k2_f32_to_f16(const float* x, void* y, long long n, k2_stream_t stream);
/* y = silu(x) on n fp16 elements, may run in place: the activations of the Kandinsky 2.2 ControlNet hint stem (diffusers
 * ImageHintTimeEmbedding.input_hint_block, once per generation; BASELINE configs[4]) */
int k2_silu_f16(const void* x, void* y, long long n, k2_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Stem im2col: fp32 NCHW latent (+ optional inpaint image*mask and mask, text2im_model2_1.py:146-155)
 * -> fp16 rows [NB*H*W, Kpad] holding the 3x3xCin patch (k = tap*Cin + c), zero padded, so that
 * input_blocks.0 (unet.py:426) runs through k2_conv_gemm as a GEMM.
 * ------------------------------------------------------------------------------------------- */
int k2_stem_im2col(const float* x, int Cx, const float* x2, int C2, const float* x3, int C3, int mul23,
                   int NB, int H, int W, void* out, int Kpad, k2_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Sampler step (classifier-free guidance + DDPM learned-range posterior), fused.
 * Replaces model_fn (kandinsky2_1_model.py:222-233), p_mean_variance / process_xstart / p_sample
 * (gaussian_diffusion.py:223-322,352-382) and denoised_fun (kandinsky2_1_model.py:237-243).
 *   model_out fp32 NCHW [2B, 8, H, W]; x fp32 [B, 4, H, W] (in place -> x_{t-1}); noise fp32 [B,4,H,W].
 *   coef (device, fp32[8]): sqrt_recip_ac, sqrt_recipm1_ac, post_coef1, post_coef2, min_log, max_log,
 *   nonzero, sqrt(alphas_cumprod[next timestep]) (2.2 inpainting only).  cond_first: 1 = rows [0,B) conditional (2.1), 0 = unconditional first (2.2).
 *   noise is not read when nonzero == 0 (the last step), so its contents (even NaN) cannot reach the result.
 *   The Kandinsky 2.2 prior's UnCLIP step runs here too (kandinsky2/model/prior.py: UnCLIPSchedule): H = 1, W = 320, the
 *   prediction in channels 0-3 and zeros in 4-7, rows {0, -1, c_x0, c_x, log var, log var, t > 0, 0}, clip 10.
 *   threshold_mode 0: x0 = clamp(x0, -clip, clip); 1: additionally the reference's dynamic threshold
 *   s = max(percentile_99.5(|x0[sample 0]|), 1); x0 = clip(x0, -s, s)/s   (gaussian_diffusion.py:284-294).
 *   Split step for sharded runs (the reference's "sample 0" is GLOBAL sample 0): 2 = x0 + percentile of local sample 0 -> s in
 *   work[B*4*H*W], no update; 4 = x0 only; 3 = the update, with s read from work[B*4*H*W] (the caller broadcasts that float
 *   from the rank that owns global sample 0 between the two calls).
 *   Inpainting (mask fp32 [B,1,H,W], 1 = keep; init fp32 [B,4,H,W] = the clean latent):
 *     inpaint_noise == NULL (Kandinsky 2.1, kandinsky2_1_model.py:237-243): x0 = x0*(1-mask) + init*mask after the clamp;
 *     inpaint_noise != NULL (Kandinsky 2.2 = diffusers KandinskyV22InpaintPipeline, restated: not in /root/reference): x0 is
 *     left alone and  x_{t-1} = mask * (c*init + sqrt(1-c^2)*inpaint_noise) + (1-mask) * x_{t-1}  with c = coef[7] =
 *     sqrt(alphas_cumprod[next timestep]) (1 at the last step = the final blend with the clean latent); inpaint_noise fp32
 *     [B,4,H,W] is the run's initial latent noise.
 *   work: fp32 scratch of at least B*4*H*W + 4096 floats.
 * ------------------------------------------------------------------------------------------- */
int k2_sampler_step(const float* model_out, float* x, const float* noise, const float* coef, int B, int H,
                    int W, float guidance, int cond_first, float clip, int threshold_mode,
                    const float* inpaint_init, const float* inpaint_mask, const float* inpaint_noise, float* work,
                    k2_stream_t stream);

/* Device-side schedule of the sampling loop, so that a whole denoising step (latent duplication for CFG + UNet + guidance +
 * scheduler update) is one CUDA graph replayed once per step with nothing copied from the host (gaussian_diffusion.py:
 * 426-475 p_sample_loop_progressive runs the loop on the host).  `counter` is a device int[2] = (step, number of steps in the
 * schedule), written by the caller before step 0; with k = counter[0] % counter[1]:
 *   k2_step_begin: x_in[0:n) = x_in[n:2n) = x[0:n) (n = B*4*H*W);  t_in[0:nt) = ts_seq[k];  coef_out[0:8) = coef_seq[k][0:8);
 *                  noise[0:n) = noise_seq[k][0:n) if noise_seq != NULL (per-step noise drawn up front, one stream per image).
 *   k2_step_end:   counter[0] += 1. */
int k2_step_begin(const float* x, float* x_in, long long n, float* t_in, int nt, float* coef_out, const float* ts_seq,
                  const float* coef_seq, const float* noise_seq, float* noise, const int* counter, k2_stream_t stream);
int k2_step_end(int* counter, k2_stream_t stream);

/* The same step for a continuously refilled batch of S slots, each slot a request at its own step of its own schedule
 * (kandinsky2/batching.py; row order, unless cond_first says otherwise: unconditional row s, conditional row S + s of the
 * CFG-doubled UNet batch, as Kandinsky 2.2 orders them).
 * state is a device int32 [2][S] = (k_s, steps_s); slot s is ACTIVE while 0 <= k_s < steps_s (and, for the tables,
 * k_s < kmax); k_s = -1 marks a free slot.  n = 4 H W floats per slot.
 *   k2_slot_step_begin: for an active slot, x_in rows s and S + s = x[s]; t_in[s] = t_in[S + s] = ts_tab[s][k_s];
 *     coef_out[s][0:8) = coef_tab[s][k_s][0:8); noise[s] = noise_tab[s][k_s] if noise_tab != NULL.  For any other slot the same
 *     places get zeros, so the UNet only sees finite input whatever the slot's buffers hold.  x fp32 [S][n], x_in [2S][n],
 *     t_in [2S], coef_out [S][8], ts_tab [S][kmax], coef_tab [S][kmax][8], noise_tab [S][kmax][n], noise [S][n].
 *   k2_slot_step_end: k_s += 1 for every active slot (a slot past its last step becomes inactive by itself).
 *   k2_slot_sampler_step / k2_slot_dpm_solver_step: k2_sampler_step (+-clip, no inpainting) / k2_dpm_solver_step (no
 *     inpainting) per slot, with the slot's coefficient row coef[s] (the coef_out above) and guidance scale guidance[s]
 *     (device fp32 [S]); work and hist fp32 [S][n] per slot.  cond_first is the row order (1: conditional row s,
 *     unconditional row S + s, the Kandinsky 2.1 order).  threshold_mode 1 is k2_sampler_step's dynamic threshold with each
 *     slot's own percentile: sval[s] = max(99.5th percentile of |x0| over slot s's n elements, 1), written to sval (device
 *     fp32 [S], required; unused at threshold_mode 0) and applied to that slot alone, which is what k2_sampler_step computes
 *     at B = 1.
 * The step entries run the same kernels as their batch forms, so an active slot's result is bit-identical to the batch form
 * applied to that slot alone; they neither read nor write an inactive slot's elements (its rows of model_out may hold NaN).
 * Arguments are checked before any CUDA call. */
int k2_slot_step_begin(const float* x, float* x_in, int S, long long n, float* t_in, float* coef_out, const float* ts_tab,
                       const float* coef_tab, int kmax, const float* noise_tab, float* noise, const int* state,
                       k2_stream_t stream);
int k2_slot_step_end(int* state, int S, k2_stream_t stream);
int k2_slot_sampler_step(const float* model_out, float* x, const float* noise, const float* coef, const float* guidance,
                         const int* state, int S, int H, int W, float clip, int cond_first, int threshold_mode, float* sval,
                         float* work, k2_stream_t stream);
int k2_slot_dpm_solver_step(const float* model_out, int C2, float* x, float* hist, const float* coef, const float* guidance,
                            const int* state, int S, int H, int W, int cond_first, k2_stream_t stream);

/* PLMS / DDIM update with an explicit epsilon history (replaces PLMSSampler.p_sample_plms, samplers.py:571-637, and the
 * CFG closure): e_t = uncond + g (cond - uncond) from model_out's first 4 channels (C2 channels per sample);
 * e' = coef[4] e_t + coef[5] hist0 + coef[6] hist1 + coef[7] hist2 (NULL history entries are skipped);
 * out = coef[2] (coef[0] x - coef[1] e') + coef[3] e'; e_t is also written to `store` if not NULL.  coef is device fp32[8]
 * = {1/sqrt(a_t), sqrt(1-a_t)/sqrt(a_t), sqrt(a_prev), sqrt(1-a_prev), w0, w1, w2, w3}. */
int k2_plms_step(const float* model_out, int C2, const float* x, float* out, const float* hist0, const float* hist1,
                 const float* hist2, float* store, const float* coef, int B, int H, int W, float guidance, int cond_first,
                 k2_stream_t stream);

/* DPM-Solver++(2M) step (Lu et al. 2022, "DPM-Solver++", Algorithm 2; multistep, one UNet evaluation per step), with the CFG
 * closure fused.  Per element of x fp32 [B, 4, H, W] (in place):
 *   eps  = uncond + g (cond - uncond) from model_out's first 4 channels (fp32 NCHW [2B, C2, H, W]; cond_first as in
 *          k2_sampler_step; the variance channels are ignored);
 *   x0   = coef[0] x - coef[1] eps   (no clamp, no threshold);
 *   x0   = x0 (1 - mask) + init mask                         if inpaint_mask != NULL and inpaint_noise == NULL (2.1);
 *   x'   = coef[2] x + coef[3] x0 + coef[4] hist   -- hist is NOT read when coef[4] == 0 (first-order steps), so its
 *          contents (even NaN) cannot reach the result;
 *   x'  += coef[7] noise   -- k2_dpm_solver_sde_step only; noise is NOT read when coef[7] == 0 (the SDE's last step);
 *   hist = x0   (hist fp32 [B, 4, H, W]: the previous step's x0 in, this step's out);
 *   x'   = mask (coef[5] init + coef[6] inpaint_noise) + (1 - mask) x'   if inpaint_noise != NULL (2.2: the known region is
 *          the clean latent noised to the next timestep with the run's initial noise; (1, 0) at the last step).
 * coef is device fp32[8] = {1/alpha_k, sigma_k/alpha_k, c_x, c_D, c_P, alpha_{k+1}, sigma_{k+1}, c_N}, one row of the host's
 * schedule (kandinsky2/model/gaussian_diffusion.py: DPMSolverSchedule), so k2_step_begin can pick it by the step counter.
 * k2_dpm_solver_step (the ODE solver) ignores c_N.  Arguments are checked before any CUDA call. */
int k2_dpm_solver_step(const float* model_out, int C2, float* x, float* hist, const float* coef, int B, int H, int W,
                       float guidance, int cond_first, const float* inpaint_init, const float* inpaint_mask,
                       const float* inpaint_noise, k2_stream_t stream);
/* DPM-Solver++(2M) SDE step (Lu et al. 2022, the data-prediction SDE solver in its 2M form): the update above with this
 * step's Gaussian noise z, noise fp32 [B, 4, H, W] (not NULL), added as coef[7] z.  Same kernel, same checks. */
int k2_dpm_solver_sde_step(const float* model_out, int C2, float* x, float* hist, const float* noise, const float* coef,
                           int B, int H, int W, float guidance, int cond_first, const float* inpaint_init,
                           const float* inpaint_mask, const float* inpaint_noise, k2_stream_t stream);

/* UniPC step (Zhao et al. 2023, "UniPC"; data prediction, B(h) = bh2, order 2): the corrector UniC of the previous interval
 * and the predictor UniP of the next one in one pass, one UNet evaluation per step, CFG closure fused.  Per element of x fp32
 * [B, 4, H, W] (in place), with r = the step's row of 16 floats:
 *   eps  = uncond + g (cond - uncond) as in k2_dpm_solver_step;
 *   D    = r[0] x - r[1] eps;   D = D (1 - mask) + init mask   if inpaint_mask != NULL and inpaint_noise == NULL (2.1);
 *   xc   = r[2] x + r[3] last + r[4] D + r[5] hist1 + r[6] hist2     (the corrected sample);
 *   x'   = r[7] xc + r[8] D + r[9] hist1;
 *   x'   = mask (r[10] init + r[11] inpaint_noise) + (1 - mask) x'   if inpaint_noise != NULL (2.2; `last` is not blended);
 *   last = xc;  hist2 = hist1;  hist1 = D.
 * last, hist1 and hist2 (fp32 [B, 4, H, W]) enter a sum only under a non-zero coefficient, so whatever they hold (even NaN)
 * cannot reach the result of a row that does not use them.  r = {1/alpha_k, sigma_k/alpha_k, a_x, a_L, a_0, a_1, a_2, b_c,
 * b_0, b_1, alpha_{k+1}, sigma_{k+1}, 0, 0, 0, 0} (kandinsky2/model/gaussian_diffusion.py: unipc_rows).  coef is device fp32:
 * with counter == NULL it is the row itself; otherwise it is a table [steps][16] and the row is counter[0] % counter[1] of the
 * device int32 counter k2_step_begin / k2_step_end maintain.  Arguments are checked before any CUDA call. */
int k2_unipc_step(const float* model_out, int C2, float* x, float* last, float* hist1, float* hist2, const float* coef,
                  const int* counter, int B, int H, int W, float guidance, int cond_first, const float* inpaint_init,
                  const float* inpaint_mask, const float* inpaint_noise, k2_stream_t stream);

/* Heun step (Karras et al. 2022, Algorithm 1 with s_churn = 0, as diffusers' HeunDiscreteScheduler runs it): one of the two
 * stages of a step per UNet evaluation, CFG closure fused.  x fp32 [B, 4, H, W] (in place) is the latent in the UNet's input
 * scale, x_ve / sqrt(sigma^2 + 1) with sigma the VE sigma; r = coef, device fp32[8] = {1/alpha, sigma, 1/sigma, c_x, c_d,
 * alpha', sigma'_vp, stage} (kandinsky2/model/gaussian_diffusion.py: HeunSchedule), staged by k2_step_begin from the step
 * counter.  Per element:
 *   eps  = uncond + g (cond - uncond) as in k2_dpm_solver_step;   d = eps  (the VE derivative (x_ve - x0) / sigma);
 *   d   += r[2] mask (r[0] x - r[1] eps - init)   if inpaint_mask != NULL and inpaint_noise == NULL (2.1: the known region
 *          replaces the x0 prediction);
 *   stage 1 (r[7] == 0):  x_prev = x;  d_prev = d;  x' = r[3] x + r[4] d        (the Euler predictor; also the last step);
 *   stage 2 (r[7] != 0):  x' = r[3] x_prev + r[4] (d_prev + d)                  (the trapezoidal corrector);
 *   x'   = mask (r[5] init + r[6] inpaint_noise) + (1 - mask) x'   if inpaint_noise != NULL (2.2, after both stages).
 * x_prev and d_prev (fp32 [B, 4, H, W], owned by the caller's step state) are not read by stage 1, so whatever they hold
 * (even NaN) cannot reach its result; stage 2 does not write them, and reads x only for the 2.1 blend.  Arguments are checked
 * before any CUDA call. */
int k2_heun_step(const float* model_out, int C2, float* x, float* x_prev, float* d_prev, const float* coef, int B, int H, int W,
                 float guidance, int cond_first, const float* inpaint_init, const float* inpaint_mask,
                 const float* inpaint_noise, k2_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * MoVQ helpers: nearest-codebook search (quntize.py:89-98; fp32, ties -> lowest index, int64 out),
 * fp32 NCHW -> NHWC transposes for the 4-channel latent, final image quantisation
 * (utils.py:57-70: ((x+1)*127.5).round().clamp(0,255) -> uint8 NHWC).
 * ------------------------------------------------------------------------------------------- */
int k2_vq_argmin(const float* z, const float* codebook, long long* idx, int n, int n_embed, int dim,
                 k2_stream_t stream);
/* y[n,o,:] = b[o] + sum_i w[o,i] x[n,i,:] on fp32 NCHW (MoVQ post_quant_conv 4->4, autoencoder.py:183) */
int k2_pointwise_nchw_f32(const float* x, const float* w, const float* b, float* y, int NB, int Ci, int Co, int HW,
                          k2_stream_t stream);
/* nearest 2x upsample of fp16 NHWC rows (movq_modules.py:93-97 F.interpolate before the conv) */
int k2_upsample2x_nhwc(const void* x, int ldx, void* y, int ldy, int NB, int H, int W, int C, k2_stream_t stream);
/* y[n, yo, xo, :] = x[n, 2*yo+oy, 2*xo+ox, :] on fp16 NHWC rows.  With (oy, ox) = (1, 1) applied to a stride-1 'same' 3x3
 * conv this is the VQGAN encoder's Downsample: pad (0,1,0,1) + conv3x3 stride 2 (vqgan_blocks.py:109-126). */
int k2_subsample2_nhwc(const void* x, int ldx, void* y, int ldy, int NB, int H, int W, int C, int oy, int ox,
                       k2_stream_t stream);
/* y[r, :] = softmax(scale * x[r, :]) over n columns, fp16 in/out, fp32 math (movq_modules.py:213-215) */
int k2_softmax_rows(const void* x, int ldx, void* y, int ldy, long long rows, int n, float scale, k2_stream_t stream);
int k2_nchw_to_nhwc_f32(const float* x, float* y, int NB, int C, int H, int W, k2_stream_t stream);
int k2_images_to_u8(const float* x_nchw, uint8_t* out_nhwc, int NB, int C, int H, int W, int crop_h,
                    int crop_w, k2_stream_t stream);
/* MoVQ SpatialNorm (movq_modules.py:61-68) + optional swish (:21-23), one read + one write of the feature map:
 *   y = act( GroupNorm(x) * (Wy.zq + by) + (Wb.zq + bb) ),  zq fp32 NHWC [NB, zh, zw, 4] nearest-resized to (H, W),
 * stats fp32 [NB, groups, 2] (mean, rstd) from k2_gn_finalize / k2_gn_stats, sn_w fp32 [C, 10] = (Wy[4], by, Wb[4], bb).
 * The per-channel normalisation and both 4 -> C modulations are folded into 10 register-resident coefficients per channel. */
int k2_sn_apply(const void* x, int C, int ldx, int NB, int H, int W, int groups, const float* stats, const float* gamma,
                const float* beta, const float* zq, int zh, int zw, const float* sn_w, int act, void* y, int ldy,
                k2_stream_t stream);
/* fp16 rows [B][T][ldx] (C columns) -> [B][C][T] (the attention values as a K-major B operand, movq_modules.py:216-219) */
int k2_transpose_f16(const void* x, int ldx, void* y, int B, int T, int C, k2_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Diffusion prior (SURVEY.md 8f rank 3; kandinsky2/model/prior.py:46-127), not on the measured denoising path and not
 * tuned (the Kandinsky 2.2 prior replays its step as one CUDA graph: kandinsky2/model/prior.py _PriorStepPlan).  The transformer's Linear layers are k2_conv_gemm flat-row GEMMs; these are the rest:
 *   k2_layernorm_f16   LayerNorm over the last dim of fp16 rows, float64 statistics, fp32 gain / bias (prior.py:46-53)
 *   k2_gelu_f16        nn.GELU (exact erf) on n fp16 elements, may run in place (prior.py:74-83)
 *   k2_attention_small QKVMultiheadAttention for T <= 128 tokens, head dim 64 (prior.py:86-103): qkv rows
 *                      [B, T, >= heads*192] with per-head [q | k | v]; additive mask = causal (if set) AND key keep-mask
 *                      (uint8 [B, T], nonzero = kept, may be NULL); fp32 softmax; out rows [B, T, >= heads*64].  A query
 *                      row that reaches no key is NaN, like torch's softmax over an all -inf row.
 * ------------------------------------------------------------------------------------------- */
int k2_layernorm_f16(const void* x, int ldx, const float* gamma, const float* beta, void* y, int ldy, int M, int N, float eps,
                     k2_stream_t stream);
int k2_gelu_f16(const void* x, void* y, long long n, k2_stream_t stream);
/* OpenAI CLIP's QuickGELU (the Kandinsky 2.1 ViT-L/14 text and image towers, kandinsky2/model/clip_vitl14.py) on n fp16
 * elements, may run in place (x == y):
 *   y[i] = fp16_rn( x / (1 + exp(-1.702 x)) )   in fp32, x = float(x[i]); within one fp16 ulp of x sigmoid(1.702 x) in float64
 * +inf -> +inf, -inf -> NaN, NaN -> NaN (torch's fp32 x * sigmoid(1.702 x)).  n positive and even, x / y 4-byte aligned;
 * arguments are checked before any CUDA call. */
int k2_quick_gelu_f16(const void* x, void* y, long long n, k2_stream_t stream);
int k2_attention_small(const void* qkv, int ldq, const unsigned char* keep_mask, int causal, void* out, int ldo, int B, int T,
                       int heads, float scale, k2_stream_t stream);
/* Token rows of the prior's sequence, bit-identical to the eager forward's `seq[:, j] = v.half()` followed by the fp16
 * `seq + positional_embedding.half()`:
 *   y[m, c] = fp16_rn( float(fp16_rn(x[m * ldx + c])) + float(pos[m * ldp + c]) )      m < M, c < N
 * x fp32, pos and y fp16; ldx = 0 / ldp = 0 repeat one source / positional row for every m.  Strides are in elements
 * (ldx, ldp: 0 or >= N; ldy >= N); x 4-byte and pos / y 2-byte aligned.  Arguments are checked before any CUDA call. */
int k2_prior_tokens(const float* x, int ldx, const void* pos, int ldp, void* y, int ldy, int M, int N, k2_stream_t stream);
/* y[m, c] = float(x[m * ldx + c]), exact: fp16 rows (ldx >= N) -> fp32 rows (ldy >= N), the `.float()` in front of the prior's
 * fp32 out_proj.  x 2-byte and y 4-byte aligned.  Arguments are checked before any CUDA call. */
int k2_f16_to_f32(const void* x, int ldx, float* y, int ldy, int M, int N, k2_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * CLIP image tower (diffusers' KandinskyV22PriorPipeline image_encoder, a transformers CLIPVisionModelWithProjection; the
 * reference builds it at kandinsky2_2_model.py:24; kandinsky2/model/clip_vision.py).  Its Linear layers are k2_conv_gemm
 * flat-row GEMMs and its LayerNorm / GELU / widening are the prior's entry points above; these two are the rest.
 *
 * k2_clip_patchify: x fp32 NCHW [B, 3, S, S] (4-byte aligned) -> out fp16 rows [B * (G^2 + 1), ldo], G = S / P, for ONE GEMM
 *   with the weight [hidden, Kp] = (patch conv weight flattened as c P^2 + ky P + kx | class_embedding | zeros) and the
 *   position embedding as the residual:
 *     row b (G^2 + 1):            1 in column 3 P^2 (the CLS slot), 0 elsewhere;
 *     row b (G^2 + 1) + 1 + t:    column c P^2 + ky P + kx = fp16_rn(x[b, c, P (t / G) + ky, P (t % G) + kx]), t < G^2;
 *   columns [3 P^2 (+1), Kp) are zero; columns >= Kp are not touched.  Needs S % P == 0, Kp >= 3 P^2 + 1, ldo >= Kp.
 * k2_attention_heads: softmax(scale q k^T) v per head, no mask, over T tokens, head width head_dim (104 only, the ViT-bigG/14
 *   geometry; anything else is refused).  qkv fp16 rows [B, T, ldq], head h reads q / k / v at h hs + q_off / k_off / v_off;
 *   out fp16 rows [B, T, ldo], head h at h ohs (only its head_dim columns are written).  Strides and offsets are multiples of 8
 *   elements, pointers 16-byte aligned, (heads - 1) hs + max offset + head_dim <= ldq, ohs >= head_dim and
 *   (heads - 1) ohs + head_dim <= ldo.  fp32 scores and softmax, P rounded to fp16 before PV (the k2_attention_d512 recipe).
 * Both check their arguments before any CUDA call.
 * ------------------------------------------------------------------------------------------- */
int k2_clip_patchify(const float* x, int B, int S, int P, void* out, int ldo, int Kp, k2_stream_t stream);
int k2_attention_heads(const void* qkv, int ldq, int hs, int q_off, int k_off, int v_off, int B, int heads, int T, int head_dim,
                       float scale, void* out, int ldo, int ohs, k2_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * CLIP text tower (diffusers' KandinskyV22PriorPipeline text_encoder, a transformers CLIPTextModelWithProjection;
 * kandinsky2/model/clip_text.py).  Its Linear layers are k2_conv_gemm flat-row GEMMs, its attention is k2_attention_small
 * (causal, no keep mask), its LayerNorm / GELU are the prior's entry points above; these two are the rest.
 *
 * k2_clip_text_embed: ids int32 [B, ldi] (T used per row), tok fp16 [V, H], pos fp16 [>= T, H] (both contiguous) ->
 *   out fp16 rows [B * T, ldo]:  out[b T + t, c] = fp16_rn( float(tok[ids[b, t], c]) + float(pos[t, c]) ),  c < H
 *   (the fp16 model's inputs_embeds + position_embeds, one rounding).  An id outside [0, V) writes a NaN row and reads no
 *   table.  H % 8 == 0, ldo >= H and a multiple of 8, tok / pos / out 16-byte aligned, ids 4-byte aligned; columns >= H are
 *   not touched.
 * k2_clip_text_pool: per sequence b the pooled position p_b, from the ids on the device:
 *     eos_id < 0:   the first t with ids[b, t] == max_t ids[b, t]   (transformers' eos_token_id == 2 rule, argmax)
 *     eos_id >= 0:  the first t with ids[b, t] == eos_id, or 0 if there is none
 *   then out[b, c] = float(hidden[(b T + p_b) ldh + c]) exactly (c < H), fp32 rows with stride ldo; index_out int32 [B] (may be
 *   NULL) receives p_b.  ldi >= T, ldh >= H, ldo >= H; ids / out / index_out 4-byte and hidden 2-byte aligned.
 * Both check their arguments before any CUDA call.
 * ------------------------------------------------------------------------------------------- */
int k2_clip_text_embed(const int* ids, int ldi, int B, int T, const void* tok, int V, const void* pos, int H, void* out, int ldo,
                       k2_stream_t stream);
int k2_clip_text_pool(const int* ids, int ldi, int B, int T, int eos_id, const void* hidden, int ldh, int H, float* out, int ldo,
                      int* index_out, k2_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * Kandinsky 2.1 text encoder (the reference's MultilingualCLIP: XLM-RoBERTa-large and a Linear, text_encoders.py:108-122;
 * kandinsky2/model/text_encoders.py).  Its Linear layers are k2_conv_gemm flat-row GEMMs, its attention is k2_attention_small
 * (not causal, the attention mask as the key keep-mask), its LayerNorm / GELU are the prior's entry points above; these two
 * are the rest.
 *
 * k2_xlmr_embed: ids int32 [B, ldi] (T used per row) -> out fp16 rows [B * T, ldo]; for row m = b T + t
 *     p = pad_id                                        if ids[b, t] == pad_id
 *       = pad_id + #{s <= t : ids[b, s] != pad_id}      otherwise   (transformers' create_position_ids_from_input_ids)
 *     x[c] = (float(word[ids[b, t], c]) + float(type_row[c])) + float(pos[p, c])      fp32, c < H
 *     out[m, c] = fp16_rn( fmaf(float((x[c] - mean) * rstd), gamma[c], beta[c]) )
 *   with mean and rstd = 1 / sqrt(var + eps) of x in float64 (two passes, as k2_layernorm_f16).  An id outside [0, V) or a
 *   position p >= P writes a NaN row and reads no table.  word fp16 [V, H], pos fp16 [P, H], type_row fp16 [H] (contiguous),
 *   gamma / beta fp32 [H].  H <= 8192, pad_id >= 0, eps > 0, ldi >= T, ldo >= H; ids / gamma / beta 4-byte and word / pos /
 *   type_row / out 2-byte aligned; columns >= H are not touched.
 * k2_masked_mean_f16: hidden fp16 rows [B * T, ldh], mask uint8 [B, ldm] (nonzero = kept) ->
 *     out[b, c] = (sum over kept t, ascending, of float(hidden[(b T + t) ldh + c]) in fp32) / count_b      fp32 [B, ldo]
 *   one division; a row with no kept token is NaN (0 / 0, as torch).  ldh >= H, ldm >= T, ldo >= H, B <= 65535; hidden
 *   2-byte and out 4-byte aligned.
 * Both check their arguments before any CUDA call.
 * ------------------------------------------------------------------------------------------- */
int k2_xlmr_embed(const int* ids, int ldi, int B, int T, int pad_id, const void* word, int V, const void* pos, int P,
                  const void* type_row, const float* gamma, const float* beta, float eps, void* out, int ldo, int H,
                  k2_stream_t stream);
int k2_masked_mean_f16(const void* hidden, int ldh, const unsigned char* mask, int ldm, int B, int T, int H, float* out,
                       int ldo, k2_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * DPT depth estimator (transformers' DPTForDepthEstimation with a plain ViT backbone, the default model of the
 * depth-estimation pipeline that builds the Kandinsky 2.2 ControlNet-depth hint; kandinsky2/model/depth.py).  Its Linear
 * layers and convolutions are k2_conv_gemm launches (ConvTranspose2d(kernel = stride = s) is one GEMM [M, C] x [C, s^2 C]
 * with the bias tiled s^2 times, followed by k2_depth_to_space_f16), its LayerNorm / GELU / attention are the ViT towers'
 * entry points above; these are the rest.  Strides are in elements; every argument is checked before any CUDA call.
 *
 * k2_relu_f16: y[m, c] = relu(x[m, c]) on fp16 rows (M rows, N columns, strides ldx / ldy >= N), bit for bit torch.relu on
 *   the GPU: a NaN keeps its bits, anything else is fp16(fmaxf(x, 0)).  x == y (in place) is allowed, other overlap is not.
 *   2-byte alignment; rows of a multiple of 8 with 16-byte aligned pointers move as 16-byte vectors.
 * k2_relu_f32: the same on fp32 rows (4-byte alignment).
 * k2_bilinear_f16: x fp16 NHWC [NB, Hi, Wi, C] rows (pixel stride ldx) -> y fp16 NHWC [NB, Ho, Wo, C] (pixel stride ldy),
 *   torch's upsample_bilinear2d without a scale factor:
 *     r = align_corners ? (out > 1 ? (in - 1) / (out - 1) : 0) : in / out                       fp32
 *     src = align_corners ? r d : max(r (d + 0.5) - 0.5, 0),  i0 = (int) src,  i1 = i0 + (i0 < in - 1),  l1 = src - i0,
 *     l0 = 1 - l1,  y = fp16_rn( l0y (l0x x[i0y, i0x] + l1x x[i0y, i1x]) + l1y (l0x x[i1y, i0x] + l1x x[i1y, i1x]) )   fp32
 *   C, ldx, ldy multiples of 8, strides >= C, 16-byte aligned pointers; columns >= C are not touched.
 * k2_depth_to_space_f16: g fp16 rows [NB H W, ldg] (ldg >= s^2 C) -> y fp16 NHWC [NB, s H, s W, C] (pixel stride ldy):
 *     y[n, s y + a, s x + b, c] = g[(n H + y) W + x, (a s + b) C + c]          a copy; a, b < s
 *   C, ldg, ldy multiples of 8, ldy >= C, 16-byte aligned pointers.
 * k2_readout_rows_f16: h fp16 rows [B T, ldh] (token 0 of each image is the CLS token) -> y fp16 rows [B (T - 1), ldy]:
 *     y[n (T - 1) + t - 1, :] = [ h[n T + t, 0:H] | h[n T, 0:H] ]               t = 1 .. T - 1, a copy
 *   (DPT's readout "project" input, cat(token, CLS)).  H, ldh, ldy multiples of 8, ldh >= H, ldy >= 2 H, 16-byte aligned.
 * ------------------------------------------------------------------------------------------- */
int k2_relu_f16(const void* x, int ldx, void* y, int ldy, int M, int N, k2_stream_t stream);
int k2_relu_f32(const float* x, int ldx, float* y, int ldy, int M, int N, k2_stream_t stream);
int k2_bilinear_f16(const void* x, int ldx, int NB, int Hi, int Wi, int C, void* y, int ldy, int Ho, int Wo, int align_corners,
                    k2_stream_t stream);
int k2_depth_to_space_f16(const void* g, int ldg, int NB, int H, int W, int C, int s, void* y, int ldy, k2_stream_t stream);
int k2_readout_rows_f16(const void* h, int ldh, int B, int T, int H, void* y, int ldy, k2_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * BiT ResNet backbone of the hybrid DPT (MiDaS v3 DPT-Hybrid, transformers' Intel/dpt-hybrid-midas; kandinsky2/model/depth.py).
 * Its 1x1 and 3x3 convolutions (weights standardised on the host) are k2_conv_gemm launches with fused GroupNorm partials,
 * a stride-2 convolution runs at stride 1 followed by k2_subsample2_nhwc; these are the rest.  Every argument is checked
 * before any CUDA call; nothing outside the output view is written.
 *
 * k2_im2col_f16: x fp32 NCHW [NB, C, H, W] (contiguous) -> y fp16 rows [NB Ho Wo, ldy] (ldy >= Kp), the k x k stride-s
 *   window of output pixel (oy, ox) with pad_top / pad_left zero rows / columns before the image (and zeros after it):
 *     y[(n Ho + oy) Wo + ox, (c k + ky) k + kx] = fp16_rn(x[n, c, oy s - pad_top + ky, ox s - pad_left + kx])
 *   columns k^2 C <= j < Kp are 0; columns >= Kp are not touched.  The column order is weight.reshape(Cout, -1)'s, so a
 *   k2_conv_gemm flat GEMM with that weight (padded to Kp) is the convolution.  Pads in [0, k).
 * k2_maxpool_f16: x fp16 NHWC [NB, H, W, C] (pixel stride ldx) -> y [NB, Ho, Wo, C] (pixel stride ldy), 3x3 window, stride 2,
 *   pad_top / pad_left (in [0, 3)) before the image and whatever Ho / Wo implies after it.  The pad value is +0, not -inf
 *   (BiT's BitMaxPool2d pads with DynamicPad2d(value=0) before max_pool2d).  Scan order ky, kx; a value replaces the running
 *   maximum when it is greater or NaN (torch's rule), so of equal values the first wins.  C, strides multiples of 8,
 *   16-byte aligned.
 * k2_gn_act_f16: y = [relu]( (x - mean) rstd gamma + beta + r ) per image and channel, groups of C / groups channels:
 *     r = 0                                                            r == NULL
 *     r = r_src                                                        r_stats == NULL
 *     r = (r_src - r_mean) r_rstd r_gamma + r_beta                     r_stats != NULL (a second GroupNorm)
 *   stats / r_stats fp32 [NB, groups, 2] (mean, rstd) as k2_gn_stats and k2_gn_finalize write them; gamma / beta fp32 [C].
 *   fp32 arithmetic (x a + b with a = gamma rstd, b = beta - mean a), one rounding.  x / r pixel strides ldx / ldr, images
 *   contiguous; y pixel stride ldy and image stride ldy_img (elements, >= (H W - 1) ldy + C), so y may be the patch rows of a
 *   wider token buffer.  C, strides multiples of 8, 16-byte aligned.
 * ------------------------------------------------------------------------------------------- */
int k2_im2col_f16(const float* x, int NB, int C, int H, int W, int k, int s, int pad_top, int pad_left, int Ho, int Wo,
                  void* y, int ldy, int Kp, k2_stream_t stream);
int k2_maxpool_f16(const void* x, int ldx, int NB, int H, int W, int C, int pad_top, int pad_left, int Ho, int Wo, void* y,
                   int ldy, k2_stream_t stream);
int k2_gn_act_f16(const void* x, int ldx, const float* stats, const float* gamma, const float* beta, const void* r, int ldr,
                  const float* r_stats, const float* r_gamma, const float* r_beta, int NB, int H, int W, int C, int groups,
                  int relu, void* y, int ldy, long long ldy_img, k2_stream_t stream);

/* ---------------------------------------------------------------------------------------------
 * LoRA adapter merge (diffusers LoRAAttnAddedKVProcessor weights folded into a packed weight, the arithmetic of diffusers'
 * fuse_lora): once per adapter load, never per step.
 *   out[n, k] = fp16_rn( float(base[n, k]) + scale * sum_j up[n, j] * down[j, k] )   n < rows, k < cols
 * base / out fp16 rows with strides ldb / ldo (elements, >= cols; columns >= cols are not touched; out may equal base);
 * up fp32 [rows, rank], down fp32 [rank, cols], both contiguous.  The sum is fp32 in ascending j, one rounding to fp16
 * (nearest-even); an element whose scaled sum is exactly zero keeps base's bits (scale 0 copies base).  The result does not
 * depend on the launch configuration.
 * ------------------------------------------------------------------------------------------- */
int k2_lora_merge(const void* base, int ldb, const float* up, const float* down, int rows, int cols, int rank, float scale,
                  void* out, int ldo, k2_stream_t stream);

#ifdef __cplusplus
}
#endif
#endif /* K2B200_H_ */
