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
"""
import math

import numpy as np
import torch
import torch.nn as nn

from .. import ops
from .._native import K2Error


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

    def finalize(self):
        """Pack the GEMM weights (fp16 [N, K], K padded to 64) once per checkpoint."""
        pk = {}
        for i, blk in enumerate(self.transformer.resblocks):
            for name, m in (("qkv", blk.attn.c_qkv), ("proj", blk.attn.c_proj), ("fc", blk.mlp.c_fc), ("proj2", blk.mlp.c_proj)):
                pk[(i, name)] = (ops.pack_conv_weight(m.weight), m.bias.float().contiguous())
        pk["text_enc"] = (ops.pack_conv_weight(self.text_enc_proj.weight), self.text_enc_proj.bias.float().contiguous())
        self._packed = pk
        return self

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
