"""Diffusion prior of Kandinsky 2.1 (reference: kandinsky2/model/prior.py) -- SURVEY.md 8f rank 3.

Parity: tests/test_gpu_zz_prior.py compares the transformer forward and the guided x0-prediction sampling loop with the
outputs of the reference's own PriorTransformer / PriorDiffusionModel classes (tests/golden/prior_tiny.pt; the oracle,
oracle/prior_oracle.py, reproduces them exactly).  tests/test_gpu_zz_prior_full.py runs the full 2.1 prior (20 layers,
width 2048, 32 heads, 81 tokens) on synthetic weights against the fp32 oracle; on an H100 (400 W), at B = 1 / 4, the forward
deviates by rel-L2 1.38e-3 / 1.31e-3 and max-abs 4.5e-3 / 5.6e-3, less than the reference's own fp16 mode does (1.67e-3 /
1.53e-3, 5.3e-3 / 5.7e-3), the fp16 residual stream stays finite (peak |h| 26), and 25-step guided sampling deviates by
rel-L2 1.7e-3.  tests/test_gpu_prior_kernels.py bounds
the three kernels against float64.  Not benchmarked.

`PriorTransformer` keeps the reference's parameter names (prior.py:191-228), so `prior_fp16.ckpt` state dicts load as they
are.  Compute: the Linear layers are flat-row wgmma GEMMs (`ops.gemm_rows`, fp16 storage / fp32 accumulate, bias and
the residual add in the epilogue), LayerNorm / GELU / the masked 81-token attention are the small kernels of
csrc/k2_prior.cu, the four single-row projections are `ops.linear`.  The residual stream is fp16 like the reference's
(`Kandinsky2_1.__init__` halves the prior when `use_fp16`).

Kandinsky 2.2 runs the same network at CLIP-bigG width (clip_dim = clip_xf_width = 1280) from a diffusers state dict
(checkpoints.diffusers_prior_to_k2).  Its sampler is diffusers' UnCLIPScheduler (UnCLIPSchedule, restated), and each sampling
step is one CUDA graph replay of _PriorStepPlan, whose model output equals `forward` bit for bit under the same GEMM
configurations; PriorEmbedder22 puts it behind the embedder protocol (tests/test_gpu_zz_prior22.py, DESIGN.md section 7).
"""
import math

import numpy as np
import torch
import torch.nn as nn

from .. import ops
from .._native import K2Error
from ..launch_plan import LaunchPlan


class _Node(nn.Module):
    pass


class PriorTransformer(nn.Module):
    def __init__(self, text_ctx, xf_width, xf_layers, xf_heads, xf_final_ln, xf_padding, clip_dim, clip_xf_width,
                 device=None):
        super().__init__()
        if xf_width % xf_heads or xf_width // xf_heads != 64:
            raise K2Error("k2b200 prior: head dimension must be 64")
        if xf_padding:
            raise K2Error("k2b200 prior: xf_padding=True is not implemented (the 2.1 config uses False)")
        self.text_ctx, self.xf_width, self.xf_layers, self.xf_heads = text_ctx, xf_width, xf_layers, xf_heads
        self.clip_dim, self.clip_xf_width, self.ext_len = clip_dim, clip_xf_width, 4
        W, n = xf_width, text_ctx + 4
        P = lambda *s: nn.Parameter(torch.zeros(*s, device=device), requires_grad=False)  # noqa: E731

        def linear(node, name, cout, cin):
            m = _Node()
            m.weight, m.bias = P(cout, cin), P(cout)
            setattr(node, name, m)

        self.positional_embedding = P(1, n, W)
        self.prd_emb = P(1, 1, W)
        self.time_embed = _Node()
        linear(self.time_embed, "0", W, W)
        linear(self.time_embed, "2", W, W)
        linear(self, "text_enc_proj", W, clip_xf_width)
        linear(self, "text_emb_proj", W, clip_dim)
        linear(self, "clip_img_proj", W, clip_dim)
        linear(self, "out_proj", clip_dim, W)
        self.transformer = _Node()
        self.transformer.resblocks = nn.ModuleList()
        for _ in range(xf_layers):
            blk = _Node()
            blk.attn = _Node()
            linear(blk.attn, "c_qkv", 3 * W, W)
            linear(blk.attn, "c_proj", W, W)
            blk.ln_1 = _Node()
            blk.ln_1.weight, blk.ln_1.bias = P(W), P(W)
            blk.mlp = _Node()
            linear(blk.mlp, "c_fc", 4 * W, W)
            linear(blk.mlp, "c_proj", W, 4 * W)
            blk.ln_2 = _Node()
            blk.ln_2.weight, blk.ln_2.bias = P(W), P(W)
            self.transformer.resblocks.append(blk)
        if xf_final_ln:
            self.final_ln = _Node()
            self.final_ln.weight, self.final_ln.bias = P(W), P(W)
        else:
            self.final_ln = None
        self._packed = None
        self._step_plans = {}

    def finalize(self):
        """Pack the GEMM weights (fp16 [N, K], K padded to 64) once per checkpoint."""
        pk = {}
        for i, blk in enumerate(self.transformer.resblocks):
            for name, m in (("qkv", blk.attn.c_qkv), ("proj", blk.attn.c_proj), ("fc", blk.mlp.c_fc), ("proj2", blk.mlp.c_proj)):
                pk[(i, name)] = (ops.pack_conv_weight(m.weight), m.bias.float().contiguous())
        pk["text_enc"] = (ops.pack_conv_weight(self.text_enc_proj.weight), self.text_enc_proj.bias.float().contiguous())
        self._packed = pk
        self._step_plans = {}
        return self

    def _step_plan(self, B):
        """The UnCLIP sampling step at B samples (2B CFG rows) as a static launch list (_PriorStepPlan), built once per B."""
        if self._packed is None:
            self.finalize()
        if B not in self._step_plans:
            self._step_plans[B] = _PriorStepPlan(self, B)
        return self._step_plans[B]

    @torch.no_grad()
    def forward(self, x, timesteps, text_emb=None, text_enc=None, mask=None, causal_mask=None):
        """x [N, clip_dim], timesteps [N], text_emb [N, clip_dim], text_enc [N, text_ctx, clip_xf_width], mask [N, text_ctx] bool
        (True = real token) -> [N, clip_dim] fp32.  `causal_mask` is accepted for signature parity; the kernel applies the
        causal structure itself."""
        if not x.is_cuda:
            raise K2Error("k2b200 prior: inputs must be CUDA tensors (no CPU fallback)")
        if self._packed is None:
            self.finalize()
        N, W, H = x.shape[0], self.xf_width, self.xf_heads
        n = self.text_ctx + self.ext_len
        keep = torch.nn.functional.pad(mask.bool(), (0, self.ext_len), value=True).to(torch.uint8).contiguous()
        lin = lambda m, v, **kw: ops.linear(v.float().contiguous(), m.weight.float().contiguous(), m.bias.float(), **kw)  # noqa: E731
        t_emb = lin(getattr(self.time_embed, "2"), lin(getattr(self.time_embed, "0"), ops.timestep_embedding(timesteps.float(), W)),
                    silu_in=True)
        wte, bte = self._packed["text_enc"]
        te16 = ops.f32_to_f16(text_enc.float().contiguous()).reshape(N * self.text_ctx, self.clip_xf_width)
        seq = torch.empty(N, n, W, dtype=torch.float16, device=x.device)
        seq[:, :self.text_ctx] = ops.gemm_rows(te16, wte, W, bias=bte).reshape(N, self.text_ctx, W)
        seq[:, self.text_ctx] = lin(self.text_emb_proj, text_emb).half()
        seq[:, self.text_ctx + 1] = t_emb.half()
        seq[:, self.text_ctx + 2] = lin(self.clip_img_proj, x).half()
        seq[:, self.text_ctx + 3] = self.prd_emb[0].half()
        h = (seq + self.positional_embedding.half()).reshape(N * n, W).contiguous()
        for i, blk in enumerate(self.transformer.resblocks):
            y = ops.layernorm_f16(h, blk.ln_1.weight.float(), blk.ln_1.bias.float())
            w, b = self._packed[(i, "qkv")]
            qkv = ops.gemm_rows(y, w, 3 * W, bias=b).reshape(N, n, 3 * W)
            a = ops.attention_small(qkv, H, keep_mask=keep, causal=True, scale=1.0 / math.sqrt(64.0)).reshape(N * n, W)
            w, b = self._packed[(i, "proj")]
            h = ops.gemm_rows(a, w, W, bias=b, residual=h)
            y = ops.layernorm_f16(h, blk.ln_2.weight.float(), blk.ln_2.bias.float())
            w, b = self._packed[(i, "fc")]
            f = ops.gelu_f16_(ops.gemm_rows(y, w, 4 * W, bias=b))
            w, b = self._packed[(i, "proj2")]
            h = ops.gemm_rows(f, w, W, bias=b, residual=h)
        last = h.reshape(N, n, W)[:, -1].contiguous()
        if self.final_ln is not None:
            last = ops.layernorm_f16(last, self.final_ln.weight.float(), self.final_ln.bias.float())
        return ops.linear(last.float(), self.out_proj.weight.float().contiguous(), self.out_proj.bias.float())


def cosine_betas(steps=1000, max_beta=0.999):
    """get_named_beta_schedule('cosine') of the reference (model/utils.py)."""
    f = lambda t: math.cos((t + 0.008) / 1.008 * math.pi / 2) ** 2  # noqa: E731
    return np.array([min(1 - f((i + 1) / steps) / f(i / steps), max_beta) for i in range(steps)], dtype=np.float64)


@torch.no_grad()
def sample_prior(model, text_emb, text_enc, mask, use_steps, guidance, clip_mean, clip_std, x_T, step_noise):
    """PriorDiffusionModel.forward (prior.py:336-384) with injected noise: x0-prediction, cosine schedule respaced to
    `use_steps`, fixed small variance, x0 clamped to +-10, classifier-free guidance with the conditional rows first.
    text_* hold 2B rows (cond | uncond); x_T [B, D]; step_noise [steps, B, D].  The per-step update acts on a [B, 768]
    tensor and is left to torch."""
    acp_full = np.cumprod(1.0 - cosine_betas(1000))
    last, betas = 1.0, []
    for i in use_steps:
        betas.append(1 - acp_full[i] / last)
        last = acp_full[i]
    betas = np.array(betas)
    acp = np.cumprod(1.0 - betas)
    acp_prev = np.append(1.0, acp[:-1])
    post_var = betas * (1.0 - acp_prev) / (1.0 - acp)
    post_logvar = np.log(np.append(post_var[1], post_var[1:]))
    c1 = betas * np.sqrt(acp_prev) / (1.0 - acp)
    c2 = (1.0 - acp_prev) * np.sqrt(1.0 - betas) / (1.0 - acp)
    B = x_T.shape[0]
    x = x_T.float()
    for n, i in enumerate(range(len(use_steps))[::-1]):
        t = torch.full((2 * B,), float(use_steps[i]), device=x.device)
        out = model(torch.cat([x, x]), t, text_emb=text_emb, text_enc=text_enc, mask=mask)
        cond, uncond = out[:B], out[B:]
        x0 = (uncond + guidance * (cond - uncond)).clamp(-10, 10)
        x = float(np.float32(c1[i])) * x0 + float(np.float32(c2[i])) * x
        if i != 0:
            x = x + math.exp(0.5 * float(np.float32(post_logvar[i]))) * step_noise[n]
    return x * clip_std + clip_mean


class PriorEmbedder:
    """The diffusion prior behind the pipelines' `embedder` protocol (kandinsky2/pipelines.py): what
    Kandinsky2_1.generate_clip_emb does (kandinsky2_1_model.py:159-182) -- CLIP text features of [prompt x B | negative
    prompt x B] -> PriorDiffusionModel sampling with classifier-free guidance -> CLIP image embedding [B, clip_dim].

    The CLIP text tower, its tokenizer and the decoder's XLM-R text encoder are conditioning PRODUCERS outside the hot path
    (SURVEY.md section 2 rows 15-16): they enter as callables, so a deployment wraps its own models and the tests use
    deterministic stand-ins:
        clip_text(list[str])  -> (txt_feat [n, clip_dim], txt_feat_seq [n, text_ctx, clip_xf_width], mask [n, text_ctx] bool)
        text_encoder(prompt, batch_size) -> (full_emb [2B, L, D1], pooled_emb [2B, D2])           (2.1 decoder only)
        clip_image(PIL.Image) -> [1, clip_dim]                                                    (mix_images with images)
    """

    def __init__(self, prior, clip_text, clip_mean, clip_std, prior_steps="25", prior_cf_scale=4.0, negative_prior_prompt="",
                 zero_image_emb=None, text_encoder=None, clip_image=None, seed=0):
        self.prior, self.clip_text, self.text_encoder, self.clip_image = prior, clip_text, text_encoder, clip_image
        self.clip_mean, self.clip_std = clip_mean, clip_std
        self.prior_steps, self.prior_cf_scale, self.negative_prior_prompt = int(prior_steps), float(prior_cf_scale), negative_prior_prompt
        self._zero = zero_image_emb
        self.seed = seed

    @torch.no_grad()
    def image_emb(self, prompt, batch_size):
        dev = self.clip_mean.device
        feat, seq, mask = self.clip_text([prompt] * batch_size + [self.negative_prior_prompt] * batch_size)
        use_steps = sorted(_space_timesteps(1000, self.prior_steps))
        import hashlib
        g = torch.Generator(device=dev).manual_seed(
            int.from_bytes(hashlib.sha256(f"{self.seed}:{prompt}".encode()).digest()[:7], "little"))
        D = self.prior.clip_dim
        x_T = torch.randn(batch_size, D, device=dev, generator=g)
        noise = torch.randn(len(use_steps), batch_size, D, device=dev, generator=g)
        return sample_prior(self.prior, feat.to(dev), seq.to(dev), mask.to(dev), use_steps, self.prior_cf_scale, self.clip_mean,
                            self.clip_std, x_T, noise).float().cpu()

    def zero_image_emb(self, batch_size):
        """CLIP embedding of a black image (create_zero_img_emb, kandinsky2_1_model.py:295-297): supplied by the deployment
        (it needs the CLIP vision tower); zeros when absent."""
        z = self._zero if self._zero is not None else torch.zeros(1, self.prior.clip_dim)
        return z.reshape(1, -1).float().cpu().repeat(batch_size, 1)

    def text_emb(self, prompt, batch_size):
        if self.text_encoder is None:
            raise K2Error("PriorEmbedder: the Kandinsky 2.1 decoder also needs the XLM-R text encoder outputs: pass text_encoder=")
        return self.text_encoder(prompt, batch_size)

    def interpolate(self, items, weights, batch_size):
        """mix_images (kandinsky2_1_model.py:346-383): weighted sum of the prior's embedding for texts and the CLIP image
        embedding for images."""
        acc = None
        for it, w in zip(items, weights):
            if isinstance(it, str):
                e = self.image_emb(it, 1)
            else:
                if self.clip_image is None:
                    raise K2Error("PriorEmbedder.interpolate: image items need clip_image=")
                e = self.clip_image(it).float().cpu()
            acc = e * w if acc is None else acc + e * w
        return acc.repeat(batch_size, 1)


def _space_timesteps(num_timesteps, count):
    """respace.py:24-72 with one section (the prior's timestep_respacing=str(prior_steps))."""
    stride = 1 if count <= 1 else (num_timesteps - 1) / (count - 1)
    cur, out = 0.0, set()
    for _ in range(count):
        out.add(round(cur))
        cur += stride
    return out


# ------------------------------------------------------------------------------------------------------------------------------
# Kandinsky 2.2 prior: diffusers' UnCLIPScheduler, the graph-replayed sampling step, and the embedder
# ------------------------------------------------------------------------------------------------------------------------------
class UnCLIPSchedule:
    """diffusers' `UnCLIPScheduler` as `kandinsky-2-2-prior` configures it (1000 training steps, squaredcos_cap_v2,
    prediction_type="sample", variance_type="fixed_small_log", clip_sample at +-10), restated (diffusers is not a dependency).

    Timesteps for N >= 2 steps: (arange(N) * 999 / (N - 1)).round() in descending order (999, 957, ..., 0 for N = 25).  Step k
    at t with t' = the next timestep (t - 1 after the last), a = acp[t], a' = acp[t'] (1 if t' < 0), beta = betas[t] if
    t' = t - 1 else 1 - a / a', alpha = 1 - beta:
        x' = (sqrt(a') beta / (1 - a)) clamp(pred, +-10) + (sqrt(alpha) (1 - a') / (1 - a)) x + sigma z,
        sigma^2 = max((1 - a') / (1 - a) beta, 1e-20), and no noise at t = 0.
    As a k2_sampler_step row (include/k2b200.h): {0, -1, c_x0, c_x, log sigma^2, log sigma^2, t > 0, 0}, so x0 = 0 x + pred
    and both variance bounds are equal.  Built in float64, cast to fp32 once.

    keep = s (KandinskyV22PriorEmb2EmbPipeline's strength): only the last s of the N steps run, `timesteps` and `rows()` are
    the tail of the full schedule's (a row's next timestep is still the full list's, as diffusers passes
    prev_timestep = timesteps[i + 1]), and the run starts from start_latent(emb, noise) at the first kept timestep."""

    def __init__(self, num_steps, num_train_timesteps=1000, clip_range=10.0, keep=None):
        num_steps = int(num_steps)
        if num_steps < 2:
            raise ValueError(f"UnCLIPSchedule: at least 2 steps (diffusers' UnCLIPScheduler divides by N - 1), got {num_steps}")
        keep = num_steps if keep is None else int(keep)
        if not 1 <= keep <= num_steps:
            raise ValueError(f"UnCLIPSchedule: keep must be in [1, {num_steps}], got {keep}")
        T = num_train_timesteps
        self.num_steps, self.keep, self.clip_range = num_steps, keep, float(clip_range)
        self.betas = cosine_betas(T)
        self.alphas_cumprod = np.cumprod(1.0 - self.betas)
        self._all = (np.arange(num_steps) * ((T - 1) / (num_steps - 1))).round()[::-1].astype(np.int64)
        self.timesteps = self._all[num_steps - keep:]

    def start_latent(self, emb, noise):
        """UnCLIPScheduler.add_noise at the first kept timestep t: sqrt(acp[t]) emb + sqrt(1 - acp[t]) noise, the coefficients
        in float64."""
        a = float(self.alphas_cumprod[int(self.timesteps[0])])
        return math.sqrt(a) * emb + math.sqrt(1.0 - a) * noise

    def rows(self):
        """float64 [keep, 8]: the k2_sampler_step row of every kept step, in loop order."""
        ts, acp, out = self._all, self.alphas_cumprod, []
        for k in range(self.num_steps - self.keep, self.num_steps):
            t = ts[k]
            tp = int(ts[k + 1]) if k + 1 < len(ts) else int(t) - 1
            a = acp[t]
            ap = acp[tp] if tp >= 0 else 1.0
            beta = self.betas[t] if tp == t - 1 else 1.0 - a / ap
            logvar = math.log(max((1.0 - ap) / (1.0 - a) * beta, 1e-20))
            out.append([0.0, -1.0, math.sqrt(ap) * beta / (1.0 - a), math.sqrt(1.0 - beta) * (1.0 - ap) / (1.0 - a), logvar, logvar,
                        1.0 if t > 0 else 0.0, 0.0])
        return np.array(out, dtype=np.float64)

    def coef_table(self):
        return self.rows().astype(np.float32)


class _PriorStepPlan(LaunchPlan):
    """One UnCLIP sampling step of the prior at B samples, on static buffers, as ONE launch list (replayed as one CUDA graph):
    k2_step_begin (x duplicated for the 2B CFG rows, this step's t / row / noise picked by the device-side counter), the time
    embedding and its two linears, clip_img_proj, the token rows 78 and 79 written into the sequence, 20 x (LayerNorm, qkv
    GEMM, attention, proj GEMM + residual, LayerNorm, fc GEMM, GELU, proj GEMM + residual), the final LayerNorm of the last
    token (a strided view), out_proj, k2_sampler_step and k2_step_end.  What does not change from step to step -- the text
    token rows, the text_emb_proj and prd_emb rows with their positional embedding, the keep mask -- is written once per call
    by bind().  Layer 0 reads the sequence buffer as its residual input.

    Every launch has the eager forward's arguments, so the model output (self.model_out[:, :clip_dim]) equals
    PriorTransformer.forward bit for bit under the same GEMM configurations (the per-shape tuner may pick split-K, which
    reorders fp32 sums; with launch_plan.TUNE_SMALL_M = 0 it only picks among bit-identical configurations)."""

    def __init__(self, model, B):
        dev = model._packed["text_enc"][0].device
        super().__init__(dev, 2 * B)
        self.m, self.B = model, B
        N, W, D, n, ctx = 2 * B, model.xf_width, model.clip_dim, model.text_ctx + model.ext_len, model.text_ctx
        if D % 4:
            raise K2Error("k2b200 prior: clip_dim must be a multiple of 4 (the sampler step sees it as [4, 1, clip_dim / 4])")
        self.N, self.n = N, n
        f32 = dict(device=dev, dtype=torch.float32)
        self.x = torch.zeros(B, D, **f32)                   # the sample, updated in place every step
        self.x_in = torch.zeros(N, D, **f32)
        self.t_in = torch.zeros(N, **f32)
        self.coef = torch.zeros(8, **f32)
        self.noise = torch.zeros(B, D, **f32)
        self.work = torch.empty(B * D + 4096, **f32)
        self.counter = torch.zeros(2, device=dev, dtype=torch.int32)
        self.ts_seq = torch.zeros(1000, **f32)
        self.coef_seq = torch.zeros(1000, 8, **f32)
        self.noise_seq = torch.zeros(1000, B, D, **f32)
        self.guidance = 4.0
        # model_out [2B, 2 * clip_dim]: out_proj writes the first clip_dim columns of each row, the variance half stays zero
        self.model_out = torch.zeros(N, 2 * D, **f32)
        self.seq = torch.zeros(N, n, W, device=dev, dtype=torch.float16)
        self.keep = torch.ones(N, n, device=dev, dtype=torch.uint8)
        self.pos16 = model.positional_embedding[0].half().contiguous()
        self._te32 = torch.empty(N * ctx, W, **f32)
        self._row32 = torch.empty(N, W, **f32)
        self._build()

    def _build(self):
        m, pk, N, n, W, B = self.m, self.m._packed, self.N, self.n, self.m.xf_width, self.B
        D, ctx, H = m.clip_dim, m.text_ctx, m.xf_heads
        S = self._add
        f32 = dict(device=self.dev, dtype=torch.float32)
        lw = lambda mod: (mod.weight.float().contiguous(), mod.bias.float())  # noqa: E731  (as forward's `lin` passes them)
        te0, te2, img, outp = (lw(getattr(m.time_embed, "0")), lw(getattr(m.time_embed, "2")), lw(m.clip_img_proj),
                               lw(m.out_proj))
        e0, e1, tok_t, tok_x = (torch.empty(N, W, **f32) for _ in range(4))
        S(lambda: ops.step_begin(self.x, self.x_in, self.t_in, self.coef, self.ts_seq, self.coef_seq, self.noise_seq, self.noise,
                                 self.counter), "step")
        S(lambda: ops.timestep_embedding(self.t_in, W, out=e0), "timestep_embedding")
        S(lambda: ops.linear(e0, *te0, out=e1), "linear", 2 * N * W * W)
        S(lambda: ops.linear(e1, *te2, silu_in=True, out=tok_t), "linear", 2 * N * W * W)
        S(lambda: ops.prior_tokens(tok_t, self.pos16[ctx + 1:ctx + 2].expand(N, W), self.seq[:, ctx + 1]), "tokens")
        S(lambda: ops.linear(self.x_in, *img, out=tok_x), "linear", 2 * N * W * D)
        S(lambda: ops.prior_tokens(tok_x, self.pos16[ctx + 2:ctx + 3].expand(N, W), self.seq[:, ctx + 2]), "tokens")
        M = N * n
        # [N, n, C] views: the tuner counts M = N * n output rows (split-K candidates for small M, launch_plan.tune)
        y, att = self._new(N, n, W), self._new(N, n, W)
        qkv, f = self._new(N, n, 3 * W), self._new(N, n, 4 * W)
        hA, hB = self._new(N, n, W), self._new(N, n, W)
        h = self.seq
        self._norms = []   # fp32 gains / biases the launches point at
        for i, blk in enumerate(m.transformer.resblocks):
            g1, b1, g2, b2 = (blk.ln_1.weight.float(), blk.ln_1.bias.float(), blk.ln_2.weight.float(), blk.ln_2.bias.float())
            self._norms += [g1, b1, g2, b2]
            S(lambda h=h, g=g1, b=b1: ops.layernorm_f16(h, g, b, out=y), "layernorm")
            w, b = pk[(i, "qkv")]
            self._gemm(y, w, 3 * W, qkv, 2 * M * 3 * W * W, bias=b)
            S(lambda: ops.attention_small(qkv, H, keep_mask=self.keep, causal=True, scale=1.0 / math.sqrt(64.0), out=att), "attention",
              4 * N * H * n * n * 64)
            w, b = pk[(i, "proj")]
            self._gemm(att, w, W, hA, 2 * M * W * W, bias=b, residual=h)
            S(lambda g=g2, b=b2: ops.layernorm_f16(hA, g, b, out=y), "layernorm")
            w, b = pk[(i, "fc")]
            self._gemm(y, w, 4 * W, f, 2 * M * 4 * W * W, bias=b)
            S(lambda: ops.gelu_f16_(f), "gelu")
            w, b = pk[(i, "proj2")]
            self._gemm(f, w, W, hB, 2 * M * 4 * W * W, bias=b, residual=hA)
            h = hB
        last = h[:, -1]
        last32 = torch.empty(N, W, **f32)
        if m.final_ln is not None:
            lnf = self._new(N, W)
            gf, bf = m.final_ln.weight.float(), m.final_ln.bias.float()
            self._norms += [gf, bf]
            S(lambda: ops.layernorm_f16(last, gf, bf, out=lnf), "layernorm")
            S(lambda: ops.f16_to_f32(lnf, out=last32), "widen")
        else:
            S(lambda: ops.f16_to_f32(last, out=last32), "widen")
        S(lambda: ops.linear(last32, *outp, out=self.model_out[:, :D]), "linear", 2 * N * W * D)
        x4, n4, mo8 = self.x.view(B, 4, 1, D // 4), self.noise.view(B, 4, 1, D // 4), self.model_out.view(N, 8, 1, D // 4)
        S(lambda: ops.sampler_step(mo8, x4, n4, self.coef, self.guidance, 0, clip=10.0, threshold_mode=0, work=self.work),
          "sampler_step")
        S(lambda: ops.step_end(self.counter), "step")

    def bind(self, text_emb, text_enc, mask):
        """This call's conditioning (2B rows, [uncond | cond]) -> the sequence rows that stay fixed for every step and the keep
        mask, with the eager forward's arithmetic (text_enc_proj GEMM, text_emb_proj linear, prd_emb, + positional rows)."""
        m, N, n, W, ctx = self.m, self.N, self.n, self.m.xf_width, self.m.text_ctx
        self.keep.copy_(torch.nn.functional.pad(mask.bool(), (0, m.ext_len), value=True).to(torch.uint8))
        wte, bte = m._packed["text_enc"]
        te16 = ops.f32_to_f16(text_enc.float().contiguous()).reshape(N * ctx, m.clip_xf_width)
        ops.f16_to_f32(ops.gemm_rows(te16, wte, W, bias=bte), out=self._te32)
        for b in range(N):
            ops.prior_tokens(self._te32[b * ctx:(b + 1) * ctx], self.pos16[:ctx], self.seq[b, :ctx])
        ops.linear(text_emb.float().contiguous(), m.text_emb_proj.weight.float().contiguous(), m.text_emb_proj.bias.float(),
                   out=self._row32)
        ops.prior_tokens(self._row32, self.pos16[ctx:ctx + 1].expand(N, W), self.seq[:, ctx])
        ops.prior_tokens(m.prd_emb[0].float().expand(N, W), self.pos16[ctx + 3:ctx + 4].expand(N, W), self.seq[:, ctx + 3])

    def set_schedule(self, sched, x_T, step_noise, guidance, use_graph=True):
        """Stage a run: the schedule's kept timesteps and rows, x_T [B, clip_dim], step_noise [keep, B, clip_dim]; resets the
        counter.  A new guidance scale drops the captured graph (the scale is a kernel argument baked into it); with use_graph
        the graph is captured here, before the state is staged, because its warm-up and first replay advance that state."""
        k = sched.keep
        if k > self.ts_seq.shape[0]:
            raise K2Error(f"k2b200 prior: at most {self.ts_seq.shape[0]} sampling steps")
        if float(guidance) != self.guidance:
            self.guidance, self.graph = float(guidance), None
        if use_graph and self.graph is None:
            self.run(True)
        self.ts_seq[:k].copy_(torch.from_numpy(sched.timesteps.astype(np.float32)))
        self.coef_seq[:k].copy_(torch.from_numpy(sched.coef_table()))
        self.noise_seq[:k].copy_(step_noise)
        self.x.copy_(x_T)
        self.counter.copy_(torch.tensor([0, k], dtype=torch.int32))


@torch.no_grad()
def sample_prior22(model, text_emb, text_enc, mask, num_steps, guidance, clip_mean, clip_std, x_T, step_noise, use_graph=True,
                   keep=None):
    """KandinskyV22PriorPipeline.__call__'s loop (diffusers, restated) with injected noise: text_* hold 2B rows [uncond | cond],
    x_T [B, clip_dim], step_noise [num_steps, B, clip_dim] (the last step draws none).  Every step is one replay of the
    prior's step graph (use_graph=False: the same launches, issued one by one).  Returns x * clip_std + clip_mean [B, clip_dim].
    CFG is uncond + g (cond - uncond); a caller without guidance passes the conditional rows twice, which makes it the
    conditional prediction exactly.  keep = s runs only the last s of the num_steps UnCLIP steps from x_T (the emb2emb
    pipeline's truncation, UnCLIPSchedule); step_noise then has s rows."""
    sched = UnCLIPSchedule(num_steps, keep=keep)
    plan = model._step_plan(x_T.shape[0])
    plan.bind(text_emb, text_enc, mask)
    plan.set_schedule(sched, x_T.float(), step_noise.float(), guidance, use_graph)
    for _ in range(sched.keep):
        plan.run(use_graph)
    return plan.x * clip_std + clip_mean


class PriorEmbedder22:
    """The Kandinsky 2.2 diffusion prior behind the pipelines' `embedder` protocol: what diffusers'
    `KandinskyV22PriorPipeline.__call__` does for the reference's Kandinsky2_2 methods (kandinsky2_2_model.py:69-80,
    99-111, 130-141, 160-172) -- CLIP text features of [negative prior prompt x B | prompt x B] -> UnCLIP sampling with
    classifier-free guidance (sample_prior22, one CUDA graph replay per step) -> CLIP image embedding [B, clip_dim].

    clip_text(list[str]) -> (text_embeds [n, clip_dim], last_hidden_state [n, text_ctx, clip_dim], mask [n, text_ctx] bool) and
    clip_image(PIL.Image) -> [1, clip_dim] are callables, as for the 2.1 PriorEmbedder.  `runs_prior` tells the 2.2 pipeline
    methods to pass their prior_steps / prior_guidance_scale / negative_prior_prompt to image_emb, interpolate and emb2emb; the
    constructor's values are the defaults.  emb2emb is KandinskyV22PriorEmb2EmbPipeline: the prior started from a noised
    image embedding.  With a guidance scale <= 1 the prior runs unguided on the prompt alone, as
    diffusers does.  x_T and the step noise come from a generator keyed by the seed and the prompt."""

    runs_prior = True

    def __init__(self, prior, clip_text, clip_mean, clip_std, zero_image_emb=None, clip_image=None, prior_steps=25,
                 prior_guidance_scale=4, negative_prior_prompt="", seed=0, use_cuda_graph=True):
        self.prior, self.clip_text, self.clip_image = prior, clip_text, clip_image
        self.clip_mean, self.clip_std = clip_mean, clip_std
        self.prior_steps, self.prior_guidance_scale = int(prior_steps), float(prior_guidance_scale)
        self.negative_prior_prompt, self.seed, self.use_cuda_graph = negative_prior_prompt, seed, use_cuda_graph
        self._zero = zero_image_emb

    @classmethod
    def from_diffusers(cls, state_dict, clip_text, device="cuda", **kwargs):
        """Build from a diffusers `PriorTransformer` state dict (kandinsky-community/kandinsky-2-2-prior, subfolder `prior`)
        via checkpoints.diffusers_prior_to_k2; the configuration is read from the tensor shapes."""
        from ..checkpoints import diffusers_prior_to_k2
        sd, mean, std = diffusers_prior_to_k2(state_dict)
        W = sd["positional_embedding"].shape[-1]
        layers = sum(1 for k in sd if k.endswith(".attn.c_qkv.weight"))
        prior = PriorTransformer(text_ctx=sd["positional_embedding"].shape[1] - 4, xf_width=W, xf_layers=layers, xf_heads=W // 64,
                                 xf_final_ln=True, xf_padding=False, clip_dim=sd["out_proj.weight"].shape[0],
                                 clip_xf_width=sd["text_enc_proj.weight"].shape[1], device=device)
        prior.load_state_dict(sd, strict=True)
        return cls(prior.finalize(), clip_text, mean.to(device).float(), std.to(device).float(), **kwargs)

    def _call_args(self, prompt, B, prior_steps, prior_guidance_scale, negative_prior_prompt):
        """(steps, guidance, CFG rows [text_embeds, hidden states, mask] on the device, the call's generator): the rows are
        [negative prior prompt x B | prompt x B], or the prompt's rows twice when guidance <= 1 (diffusers'
        do_classifier_free_guidance is False, see sample_prior22); the generator is keyed by the seed and the prompt."""
        steps = self.prior_steps if prior_steps is None else int(prior_steps)
        g = self.prior_guidance_scale if prior_guidance_scale is None else float(prior_guidance_scale)
        neg = self.negative_prior_prompt if negative_prior_prompt is None else negative_prior_prompt
        dev = self.clip_mean.device
        if g > 1.0:
            feat, seq, mask = self.clip_text([neg] * B + [prompt] * B)
        else:
            feat, seq, mask = (torch.cat([t, t]) for t in self.clip_text([prompt] * B))
        import hashlib
        gen = torch.Generator(device=dev).manual_seed(
            int.from_bytes(hashlib.sha256(f"{self.seed}:{prompt}".encode()).digest()[:7], "little"))
        return steps, g, (feat.to(dev), seq.to(dev), mask.to(dev)), gen

    @torch.no_grad()
    def image_emb(self, prompt, batch_size, prior_steps=None, prior_guidance_scale=None, negative_prior_prompt=None):
        dev, B, D = self.clip_mean.device, batch_size, self.prior.clip_dim
        steps, g, rows, gen = self._call_args(prompt, B, prior_steps, prior_guidance_scale, negative_prior_prompt)
        x_T = torch.randn(B, D, device=dev, generator=gen)
        noise = torch.randn(steps, B, D, device=dev, generator=gen)
        return sample_prior22(self.prior, *rows, steps, g, self.clip_mean, self.clip_std, x_T, noise,
                              use_graph=self.use_cuda_graph).float().cpu()

    @torch.no_grad()
    def emb2emb(self, prompt, image, batch_size, strength=0.3, prior_steps=None, prior_guidance_scale=None,
                negative_prior_prompt=None):
        """diffusers' KandinskyV22PriorEmb2EmbPipeline.__call__ (restated, unpinned): the prior started from a noised image
        embedding instead of pure noise.  image: a CLIP image embedding [1, clip_dim] (repeated to batch_size rows) or
        [batch_size, clip_dim], or a PIL image, which goes through clip_image.  Of the N = prior_steps UnCLIP steps the last
        keep = min(int(N * strength), N) run (get_timesteps), from x = UnCLIPScheduler.add_noise(image embedding, z) at the first
        kept timestep (prepare_latents: the embedding is NOT normalised by clip_mean / clip_std on the way in); the result is
        x * clip_std + clip_mean (post_process_latents), as for image_emb.  Rows, guidance and the negative prior prompt are
        image_emb's; the generator draws z [B, clip_dim] first, then the step noise [keep, B, clip_dim]."""
        steps = self.prior_steps if prior_steps is None else int(prior_steps)
        strength = float(strength)
        if not 0.0 <= strength <= 1.0:
            raise ValueError(f"PriorEmbedder22.emb2emb: strength must be in [0, 1], got {strength}")
        keep = min(int(steps * strength), steps)
        if keep == 0:
            raise ValueError(f"PriorEmbedder22.emb2emb: strength {strength} keeps no step of {steps} (int(N * strength) = 0)")
        sched = UnCLIPSchedule(steps, keep=keep)
        dev, B, D = self.clip_mean.device, batch_size, self.prior.clip_dim
        if torch.is_tensor(image):
            emb = image.float().reshape(-1, D) if image.dim() == 1 else image.float()
            if emb.dim() != 2 or emb.shape[1] != D or emb.shape[0] not in (1, B):
                raise ValueError(f"PriorEmbedder22.emb2emb: an image embedding must be [1, {D}] or [{B}, {D}], got "
                                 f"{list(image.shape)}")
        else:
            if self.clip_image is None:
                raise K2Error("PriorEmbedder22.emb2emb: a PIL image needs clip_image=")
            emb = self.clip_image(image).float().reshape(1, D)
        emb = emb.to(dev).expand(B, D)
        steps, g, rows, gen = self._call_args(prompt, B, steps, prior_guidance_scale, negative_prior_prompt)
        z = torch.randn(B, D, device=dev, generator=gen)
        noise = torch.randn(keep, B, D, device=dev, generator=gen)
        return sample_prior22(self.prior, *rows, steps, g, self.clip_mean, self.clip_std, sched.start_latent(emb, z), noise,
                              use_graph=self.use_cuda_graph, keep=keep).float().cpu()

    def zero_image_emb(self, batch_size):
        """CLIP embedding of a black image (diffusers' KandinskyV22PriorPipeline.get_zero_embed): supplied by the deployment
        (it needs the CLIP vision tower); zeros when absent."""
        z = self._zero if self._zero is not None else torch.zeros(1, self.prior.clip_dim)
        return z.reshape(1, -1).float().cpu().repeat(batch_size, 1)

    def text_emb(self, prompt, batch_size):
        raise K2Error("PriorEmbedder22: the Kandinsky 2.2 decoder takes no text input (image embeddings only)")

    def interpolate(self, items, weights, batch_size, **prior_kwargs):
        """diffusers' KandinskyV22PriorPipeline.interpolate: a text item runs the prior for batch_size rows, an image item is
        clip_image(img) repeated batch_size times; the result is the weighted sum."""
        acc = None
        for it, w in zip(items, weights):
            if isinstance(it, str):
                e = self.image_emb(it, batch_size, **prior_kwargs)
            else:
                if self.clip_image is None:
                    raise K2Error("PriorEmbedder22.interpolate: image items need clip_image=")
                e = self.clip_image(it).float().cpu().reshape(1, -1).repeat(batch_size, 1)
            acc = e * w if acc is None else acc + e * w
        return acc
