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
PriorTransformer.load_lora merges a diffusers attention-processor LoRA of the self-attention into the packed attn.qkv /
attn.proj in place (checkpoints.prior_lora_to_k2, k2_lora_merge), so the step graphs stay as they are
(tests/test_gpu_zz_prior_lora.py).
"""
import math
import os
import re

import numpy as np
import torch
import torch.nn as nn

from .. import ops
from .._native import K2Error
from ..launch_plan import LaunchPlan, tune
from .encoder import pack_layers, record_layers
from .gaussian_diffusion import SpacedDiffusion, space_timesteps

# encoder.layer_shapes names -> the reference's names inside transformer.resblocks[i]
_BLOCK_NAMES = {"ln_1": "ln_1", "ln_2": "ln_2", "attn.qkv": "attn.c_qkv", "attn.proj": "attn.c_proj", "mlp.fc1": "mlp.c_fc",
                "mlp.fc2": "mlp.c_proj"}


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
        self._lora = None        # (factors from checkpoints.prior_lora_to_k2, scale) of the loaded adapter
        self._lora_base = None   # device copies of the unmerged packed attn.qkv / attn.proj while an adapter is merged

    def finalize(self):
        """Pack the GEMM weights (fp16 [N, K], K padded to 64) once per checkpoint, the blocks' with their LayerNorm parameters
        (encoder.pack_layers)."""
        def get(i, name):
            mod, leaf = name.rsplit(".", 1)
            return self.get_parameter(f"transformer.resblocks.{i}.{_BLOCK_NAMES[mod]}.{leaf}")

        te = self.text_enc_proj
        self._packed = {"layers": pack_layers(get, self.xf_layers, te.weight.device),
                        "text_enc": (ops.pack_conv_weight(te.weight), te.bias.float().contiguous())}
        self._step_plans = {}
        self._lora_base = None
        if self._lora is not None:  # a loaded adapter survives re-packing
            self._merge_lora()
        return self

    # ---------------------------------------------------------------- LoRA adapters, merged into the packed weights
    _LORA_WEIGHTS = (("attn.qkv", "attn.c_qkv"), ("attn.proj", "attn.c_proj"))

    @property
    def lora_scale(self):
        """Scale of the loaded LoRA adapter, None when there is none."""
        return None if self._lora is None else self._lora[1]

    def load_lora(self, state_dict, scale=1.0):
        """Merge a LoRA adapter of the self-attention -- diffusers' `LoRAAttnProcessor` weights as `AttnProcsLayers` writes
        them for the 2.2 prior (checkpoints.prior_lora_to_k2) -- into the packed weights: W = W_base + scale * up @ down,
        computed by k2_lora_merge in fp32 and rounded once to fp16, two launches per layer (attn.qkv, attn.proj).  The merge
        writes the packed tensors in place, so captured step graphs keep their addresses and need no rebuild.  On first use the
        unmerged packed weights are copied on the device (restored by unload_lora).  Loading again replaces the adapter
        (adapters do not stack; a new scale means loading again).  state_dict() never changes."""
        from ..checkpoints import prior_lora_to_k2
        factors = prior_lora_to_k2(state_dict, self.xf_width, self.xf_layers)
        if not self.text_enc_proj.weight.is_cuda:
            raise K2Error("k2b200 prior: load_lora merges on the GPU; the prior is not on a CUDA device (no CPU fallback)")
        if self._packed is None:
            self.finalize()
        self._lora = (factors, float(scale))
        self._merge_lora()

    def unload_lora(self):
        """Restore the unmerged packed weights (bit-exact) and free their copy."""
        if self._lora_base is not None and self._packed is not None:
            for L, base in zip(self._packed["layers"], self._lora_base):
                for name, _ in self._LORA_WEIGHTS:
                    L[name][0].copy_(base[name])
        self._lora = None
        self._lora_base = None

    def _merge_lora(self):
        layers = self._packed["layers"]
        if self._lora_base is None:
            self._lora_base = [{name: L[name][0].clone() for name, _ in self._LORA_WEIGHTS} for L in layers]
        weights = [(f"transformer.resblocks.{i}.{target}.weight", base[name], L[name][0])
                   for i, (L, base) in enumerate(zip(layers, self._lora_base)) for name, target in self._LORA_WEIGHTS]
        ops.lora_merge_weights(weights, *self._lora)

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
        for L in self._packed["layers"]:
            y = ops.layernorm_f16(h, *L["ln_1"])
            w, b = L["attn.qkv"]
            qkv = ops.gemm_rows(y, w, 3 * W, bias=b).reshape(N, n, 3 * W)
            a = ops.attention_small(qkv, H, keep_mask=keep, causal=True, scale=1.0 / math.sqrt(64.0)).reshape(N * n, W)
            w, b = L["attn.proj"]
            h = ops.gemm_rows(a, w, W, bias=b, residual=h)
            y = ops.layernorm_f16(h, *L["ln_2"])
            w, b = L["mlp.fc1"]
            f = ops.gelu_f16_(ops.gemm_rows(y, w, 4 * W, bias=b))
            w, b = L["mlp.fc2"]
            h = ops.gemm_rows(f, w, W, bias=b, residual=h)
        last = h.reshape(N, n, W)[:, -1].contiguous()
        if self.final_ln is not None:
            last = ops.layernorm_f16(last, self.final_ln.weight.float(), self.final_ln.bias.float())
        return ops.linear(last.float(), self.out_proj.weight.float().contiguous(), self.out_proj.bias.float())


def prior_from_state_dict(sd, device="cuda"):
    """A 2.1 PriorTransformer from its state dict (the reference's names, `prior_fp16.ckpt` without the "model." prefix), the
    geometry read from the shapes (text_ctx, width, layers, heads of 64, final LayerNorm, clip_dim, clip_xf_width); packed.
    Unknown and missing keys raise K2Error naming them (the reference loads with strict=False)."""
    need = ("positional_embedding", "out_proj.weight", "text_enc_proj.weight")
    if any(k not in sd for k in need):
        raise K2Error(f"2.1 prior state dict: missing keys {[k for k in need if k not in sd]}")
    W = sd["positional_embedding"].shape[-1]
    prior = PriorTransformer(text_ctx=sd["positional_embedding"].shape[1] - 4, xf_width=W,
                             xf_layers=sum(1 for k in sd if re.fullmatch(r"transformer\.resblocks\.\d+\.attn\.c_qkv\.weight", k)),
                             xf_heads=W // 64, xf_final_ln="final_ln.weight" in sd, xf_padding="padding_embedding" in sd,
                             clip_dim=sd["out_proj.weight"].shape[0], clip_xf_width=sd["text_enc_proj.weight"].shape[1],
                             device=device)
    want = prior.state_dict()
    unknown = sorted(set(sd) - set(want))
    missing = [k for k in want if k not in sd]
    bad = [k for k in want if k in sd and tuple(sd[k].shape) != tuple(want[k].shape)]
    if unknown or missing or bad:
        raise K2Error(f"2.1 prior state dict: unknown keys {unknown}, missing keys {missing}, wrong shapes {bad}")
    prior.load_state_dict(sd, strict=True)
    return prior.finalize()


def cosine_betas(steps=1000, max_beta=0.999):
    """get_named_beta_schedule('cosine') of the reference (model/utils.py)."""
    f = lambda t: math.cos((t + 0.008) / 1.008 * math.pi / 2) ** 2  # noqa: E731
    return np.array([min(1 - f((i + 1) / steps) / f(i / steps), max_beta) for i in range(steps)], dtype=np.float64)


@torch.no_grad()
def sample_prior(model, text_emb, text_enc, mask, use_steps, guidance, clip_mean, clip_std, x_T, step_noise):
    """PriorDiffusionModel.forward (prior.py:336-384) with injected noise: x0-prediction, cosine schedule respaced to
    `use_steps`, fixed small variance, x0 clamped to +-10, classifier-free guidance with the conditional rows first.
    text_* hold 2B rows (cond | uncond); x_T [B, D]; step_noise [steps, B, D].  The per-step update acts on a [B, 768]
    tensor and is left to torch.  use_steps: base timesteps in strictly increasing order (ValueError otherwise)."""
    if any(b <= a for a, b in zip(use_steps, use_steps[1:])):
        raise ValueError("sample_prior: use_steps must be strictly increasing")
    d = SpacedDiffusion(set(use_steps), cosine_betas(1000))
    c1, c2, post_logvar = d.posterior_mean_coef1, d.posterior_mean_coef2, d.posterior_log_variance_clipped
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
    The 2.1 text_encoder comes with this package: model.text_encoders.MultilingualCLIP.from_pretrained(dir).
        clip_image(PIL.Image) -> [1, clip_dim]                                                    (mix_images with images)
    """

    def __init__(self, prior, clip_text, clip_mean, clip_std, prior_steps="25", prior_cf_scale=4.0, negative_prior_prompt="",
                 zero_image_emb=None, text_encoder=None, clip_image=None, seed=0):
        self.prior, self.clip_text, self.text_encoder, self.clip_image = prior, clip_text, text_encoder, clip_image
        self.clip_mean, self.clip_std = clip_mean, clip_std
        self.prior_steps, self.prior_cf_scale, self.negative_prior_prompt = int(prior_steps), float(prior_cf_scale), negative_prior_prompt
        self._zero = zero_image_emb
        self.seed = seed

    @classmethod
    def from_pretrained(cls, path, clip_path=None, bpe_path=None, device="cuda", **kwargs):
        """The reference's 2.1 cache folder (`get_kandinsky2` writes it to <cache_dir>/2_1) -> the embedder with every
        conditioning producer on this package's kernels:
            prior_fp16.ckpt       the PriorDiffusionModel state dict ("model." stripped; the geometry is read from the shapes)
            ViT-L-14_stats.th     (clip_mean, clip_std)
            text_encoder/         the M-CLIP text encoder (text_encoders.MultilingualCLIP.from_pretrained) -> text_encoder
            ViT-L-14.pt           the OpenAI CLIP checkpoint (clip_path; clip_vitl14.load_openai_clip) -> clip_text,
                                  clip_image and zero_image_emb (the image tower's zero_embed, computed here once)
            bpe_simple_vocab_16e6.txt.gz   clip's BPE vocabulary (bpe_path) for the CLIP tokenizer
        A missing file raises K2Error naming it, and so does a CLIP tower that does not fit the prior (its width, embedding
        width or context against the prior's clip_xf_width, clip_dim, text_ctx).  kwargs go to the constructor
        (prior_steps, prior_cf_scale, negative_prior_prompt, seed)."""
        from .clip_vitl14 import load_openai_clip
        from .text_encoders import MultilingualCLIP
        clip_path = os.path.join(path, "ViT-L-14.pt") if clip_path is None else clip_path
        bpe_path = os.path.join(path, "bpe_simple_vocab_16e6.txt.gz") if bpe_path is None else bpe_path
        files = [os.path.join(path, "prior_fp16.ckpt"), os.path.join(path, "ViT-L-14_stats.th"),
                 os.path.join(path, "text_encoder"), clip_path, bpe_path]
        for f in files:
            if not os.path.exists(f):
                raise K2Error(f"PriorEmbedder.from_pretrained: {f} not found")
        sd = torch.load(files[0], map_location="cpu", weights_only=True)
        prior = prior_from_state_dict({k[len("model."):] if k.startswith("model.") else k: v for k, v in sd.items()}, device)
        clip_mean, clip_std = torch.load(files[1], map_location="cpu", weights_only=True)
        text, image = load_openai_clip(clip_path, device, bpe_path)
        got = (text.cfg["hidden_size"], text.cfg["projection_dim"], text.tokens)
        want = (prior.clip_xf_width, prior.clip_dim, prior.text_ctx)
        if got != want:
            raise K2Error(f"PriorEmbedder.from_pretrained: the CLIP text tower gives (width, embedding width, context) {got}, "
                          f"the prior takes (clip_xf_width, clip_dim, text_ctx) {want}")
        if image.cfg["projection_dim"] != prior.clip_dim:
            raise K2Error(f"PriorEmbedder.from_pretrained: the CLIP image tower's embedding width "
                          f"{image.cfg['projection_dim']} is not the prior's clip_dim {prior.clip_dim}")
        encoder = MultilingualCLIP.from_pretrained(files[2], device=device)
        dev = torch.device(device)
        return cls(prior, text, clip_mean.reshape(-1).to(dev, torch.float32), clip_std.reshape(-1).to(dev, torch.float32),
                   zero_image_emb=image.zero_embed().float().cpu(), text_encoder=encoder, clip_image=image, **kwargs)

    @torch.no_grad()
    def image_emb(self, prompt, batch_size):
        dev = self.clip_mean.device
        feat, seq, mask = self.clip_text([prompt] * batch_size + [self.negative_prior_prompt] * batch_size)
        use_steps = sorted(space_timesteps(1000, [self.prior_steps]))
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


class _PriorNet(LaunchPlan):
    """The prior network of one UnCLIP sampling step over N CFG rows, as launches recorded into a plan: the buffers the step
    plans share (x_in, t_in, the sequence, the keep mask, model_out) and the recording of the time embedding and its two
    linears, clip_img_proj, the token rows 78 and 79 written into the sequence, the 20 pre-LayerNorm layers of
    model/encoder.py with the masked k2_attention_small as the attention, the final LayerNorm of the last token (a strided
    view) and out_proj.  Every launch has the eager forward's arguments.  _PriorStepPlan (one call at B samples) puts its
    step begin / sampler step / step end around it; batching.PriorBatcher puts the slot step's around a _PriorSlotPlan."""

    def __init__(self, model, N):
        dev = model._packed["text_enc"][0].device
        super().__init__(dev, N)
        self.m = model
        W, D, n = model.xf_width, model.clip_dim, model.text_ctx + model.ext_len
        if D % 4:
            raise K2Error("k2b200 prior: clip_dim must be a multiple of 4 (the sampler step sees it as [4, 1, clip_dim / 4])")
        self.N, self.n = N, n
        f32 = dict(device=dev, dtype=torch.float32)
        self.x_in = torch.zeros(N, D, **f32)
        self.t_in = torch.zeros(N, **f32)
        # model_out [N, 2 * clip_dim]: out_proj writes the first clip_dim columns of each row, the variance half stays zero
        self.model_out = torch.zeros(N, 2 * D, **f32)
        self.seq = torch.zeros(N, n, W, device=dev, dtype=torch.float16)
        self.keep = torch.ones(N, n, device=dev, dtype=torch.uint8)
        self.pos16 = model.positional_embedding[0].half().contiguous()

    def _record_network(self):
        m, pk, N, n, W = self.m, self.m._packed, self.N, self.n, self.m.xf_width
        D, ctx, H = m.clip_dim, m.text_ctx, m.xf_heads
        S = self._add
        f32 = dict(device=self.dev, dtype=torch.float32)
        lw = lambda mod: (mod.weight.float().contiguous(), mod.bias.float())  # noqa: E731  (as forward's `lin` passes them)
        te0, te2, img, outp = (lw(getattr(m.time_embed, "0")), lw(getattr(m.time_embed, "2")), lw(m.clip_img_proj),
                               lw(m.out_proj))
        e0, e1, tok_t, tok_x = (torch.empty(N, W, **f32) for _ in range(4))
        S(lambda: ops.timestep_embedding(self.t_in, W, out=e0), "timestep_embedding")
        S(lambda: ops.linear(e0, *te0, out=e1), "linear", 2 * N * W * W)
        S(lambda: ops.linear(e1, *te2, silu_in=True, out=tok_t), "linear", 2 * N * W * W)
        S(lambda: ops.prior_tokens(tok_t, self.pos16[ctx + 1:ctx + 2].expand(N, W), self.seq[:, ctx + 1]), "tokens")
        S(lambda: ops.linear(self.x_in, *img, out=tok_x), "linear", 2 * N * W * D)
        S(lambda: ops.prior_tokens(tok_x, self.pos16[ctx + 2:ctx + 3].expand(N, W), self.seq[:, ctx + 2]), "tokens")
        attend = lambda qkv, out: ops.attention_small(qkv, H, keep_mask=self.keep, causal=True,  # noqa: E731
                                                      scale=1.0 / math.sqrt(64.0), out=out)
        # eps 1e-5: ops.layernorm_f16's default, which forward uses
        h = record_layers(self, self.seq, pk["layers"], attend, 4 * N * H * n * n * 64, 1e-5)
        last = h[:, -1]
        last32 = torch.empty(N, W, **f32)
        if m.final_ln is not None:
            lnf = self._new(N, W)
            gf, bf = m.final_ln.weight.float(), m.final_ln.bias.float()
            S(lambda: ops.layernorm_f16(last, gf, bf, out=lnf), "layernorm")
            S(lambda: ops.f16_to_f32(lnf, out=last32), "widen")
        else:
            S(lambda: ops.f16_to_f32(last, out=last32), "widen")
        S(lambda: ops.linear(last32, *outp, out=self.model_out[:, :D]), "linear", 2 * N * W * D)

    def _fixed_rows(self, text_emb, text_enc, mask, seq, keep, te32, row32):
        """The conditioning of len(seq) CFG rows -> the sequence rows that stay fixed for every step and the keep mask, written
        into seq / keep with the eager forward's arithmetic (text_enc_proj GEMM, text_emb_proj linear, prd_emb, + positional
        rows); te32 / row32: fp32 scratch of [rows * text_ctx, W] / [rows, W]."""
        m, W, ctx = self.m, self.m.xf_width, self.m.text_ctx
        N = seq.shape[0]
        keep.copy_(torch.nn.functional.pad(mask.bool(), (0, m.ext_len), value=True).to(torch.uint8))
        wte, bte = m._packed["text_enc"]
        te16 = ops.f32_to_f16(text_enc.float().contiguous()).reshape(N * ctx, m.clip_xf_width)
        ops.f16_to_f32(ops.gemm_rows(te16, wte, W, bias=bte), out=te32)
        for b in range(N):
            ops.prior_tokens(te32[b * ctx:(b + 1) * ctx], self.pos16[:ctx], seq[b, :ctx])
        ops.linear(text_emb.float().contiguous(), m.text_emb_proj.weight.float().contiguous(), m.text_emb_proj.bias.float(),
                   out=row32)
        ops.prior_tokens(row32, self.pos16[ctx:ctx + 1].expand(N, W), seq[:, ctx])
        ops.prior_tokens(m.prd_emb[0].float().expand(N, W), self.pos16[ctx + 3:ctx + 4].expand(N, W), seq[:, ctx + 3])


class _PriorStepPlan(_PriorNet):
    """One UnCLIP sampling step of the prior at B samples, on static buffers, as ONE launch list (replayed as one CUDA graph):
    k2_step_begin (x duplicated for the 2B CFG rows, this step's t / row / noise picked by the device-side counter), the
    network of _PriorNet, k2_sampler_step and k2_step_end.  What does not change from step to step -- the text token rows,
    the text_emb_proj and prd_emb rows with their positional embedding, the keep mask -- is written once per call by bind().
    Layer 0 reads the sequence buffer as its residual input.

    Every launch has the eager forward's arguments, so the model output (self.model_out[:, :clip_dim]) equals
    PriorTransformer.forward bit for bit under the same GEMM configurations (the per-shape tuner may pick split-K, which
    reorders fp32 sums; with launch_plan.TUNE_SMALL_M = 0 it only picks among bit-identical configurations)."""

    def __init__(self, model, B):
        super().__init__(model, 2 * B)
        self.B = B
        D, W, ctx = model.clip_dim, model.xf_width, model.text_ctx
        f32 = dict(device=self.dev, dtype=torch.float32)
        self.x = torch.zeros(B, D, **f32)                   # the sample, updated in place every step
        self.coef = torch.zeros(8, **f32)
        self.noise = torch.zeros(B, D, **f32)
        self.work = torch.empty(B * D + 4096, **f32)
        self.counter = torch.zeros(2, device=self.dev, dtype=torch.int32)
        self.ts_seq = torch.zeros(1000, **f32)
        self.coef_seq = torch.zeros(1000, 8, **f32)
        self.noise_seq = torch.zeros(1000, B, D, **f32)
        self.guidance = 4.0
        self._te32 = torch.empty(self.N * ctx, W, **f32)
        self._row32 = torch.empty(self.N, W, **f32)
        self._build()

    def _build(self):
        N, B, D = self.N, self.B, self.m.clip_dim
        self._add(lambda: ops.step_begin(self.x, self.x_in, self.t_in, self.coef, self.ts_seq, self.coef_seq, self.noise_seq,
                                         self.noise, self.counter), "step")
        self._record_network()
        x4, n4, mo8 = self.x.view(B, 4, 1, D // 4), self.noise.view(B, 4, 1, D // 4), self.model_out.view(N, 8, 1, D // 4)
        self._add(lambda: ops.sampler_step(mo8, x4, n4, self.coef, self.guidance, 0, clip=10.0, threshold_mode=0,
                                           work=self.work), "sampler_step")
        self._add(lambda: ops.step_end(self.counter), "step")

    def bind(self, text_emb, text_enc, mask):
        """This call's conditioning (2B rows, [uncond | cond]) -> the sequence rows that stay fixed for every step and the keep
        mask (_fixed_rows)."""
        self._fixed_rows(text_emb, text_enc, mask, self.seq, self.keep, self._te32, self._row32)

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


class _PriorSlotPlan(_PriorNet):
    """The prior network of _PriorNet over the 2S CFG rows of S slots (unconditional row s, conditional row S + s), each slot a
    request at its own step of its own tables (batching.PriorBatcher, which launches the slot step around it).  bind_slot
    writes one slot's fixed sequence rows and keep-mask rows; what a slot's rows compute depends on its own rows alone."""

    def __init__(self, model, S):
        super().__init__(model, 2 * S)
        self.S = S
        W, n, ctx = model.xf_width, self.n, model.text_ctx
        f32 = dict(device=self.dev, dtype=torch.float32)
        # bind_slot computes a slot's rows at bind's B = 1 shapes (2 rows) here, then copies them into rows s and S + s
        self._seq2 = torch.zeros(2, n, W, device=self.dev, dtype=torch.float16)
        self._keep2 = torch.ones(2, n, device=self.dev, dtype=torch.uint8)
        self._te32 = torch.empty(2 * ctx, W, **f32)
        self._row32 = torch.empty(2, W, **f32)
        self._record_network()

    def _gemm(self, x, w, cout, out, flops, bias=None, residual=None):
        """The layers' flat-row GEMM at 2S rows, pinned to the N tile and split-K factor the batch-1 plan (_PriorStepPlan at
        B = 1: 2 CFG rows) runs it with -- the choice tune() caches for the 2-row shape, as the library then applies it.  The
        library's own cycle model picks the split-K factor from the row count, and a split changes the fp32 summation order;
        pinned, every row sums as at batch 1, so a slot computes what image_emb(prompt, 1) computes."""
        rows, n = x.shape[0], x.shape[1]
        x2, out2 = x[:2], out[:2]
        res2 = residual[:2] if residual is not None else None
        run2 = lambda cfg, info=None: ops.gemm_rows(x2, w, cout, bias=bias, residual=res2, out=out2, cfg=cfg,  # noqa: E731
                                                    info=info)
        info = [0] * 7
        run2(tune(("gemm", cout, tuple(x2.shape), residual is not None), run2, m_rows=2 * n), info)
        cfg = (info[0], 0, info[2], 1)
        got = [0] * 7
        self._add(lambda: ops.gemm_rows(x, w, cout, bias=bias, residual=residual, out=out, cfg=cfg, info=got), "conv_gemm",
                  flops)
        if (got[0], got[2]) != (cfg[0], cfg[2]):
            raise K2Error(f"k2b200 prior: the GEMM of {rows} x {n} rows to {cout} columns cannot take the batch-1 plan's N tile "
                          f"{cfg[0]} and split-K factor {cfg[2]} (it ran {got[0]} / {got[2]}); use fewer slots")
        self._parts.pop(out.data_ptr(), None)

    def bind_slot(self, s, text_emb, text_enc, mask):
        """Slot s's conditioning (2 rows, [uncond | cond]) -> its fixed sequence rows (the text tokens, the text_emb_proj and
        prd_emb rows, with their positional rows) and keep-mask rows, computed as bind computes them at B = 1 and copied into
        rows s and S + s; no other row changes, so the rows have the same bits in every slot."""
        if not 0 <= s < self.S:
            raise K2Error(f"bind_slot: slot {s} outside [0, {self.S})")
        ctx = self.m.text_ctx
        self._fixed_rows(text_emb, text_enc, mask, self._seq2, self._keep2, self._te32, self._row32)
        for src, row in ((0, s), (1, self.S + s)):
            self.seq[row, :ctx + 1].copy_(self._seq2[src, :ctx + 1])
            self.seq[row, ctx + 3].copy_(self._seq2[src, ctx + 3])
            self.keep[row].copy_(self._keep2[src])


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
    def from_diffusers(cls, state_dict, clip_text=None, device="cuda", image_encoder=None, text_encoder=None, **kwargs):
        """Build from a diffusers `PriorTransformer` state dict (kandinsky-community/kandinsky-2-2-prior, subfolder `prior`)
        via checkpoints.diffusers_prior_to_k2; the configuration is read from the tensor shapes.  image_encoder: the pipeline's
        CLIP image tower (model.clip_vision.CLIPVisionTower) or None.  A tower becomes clip_image and, unless zero_image_emb is
        passed, supplies it as the tower on all-zero pixel_values, computed here once (diffusers' get_zero_embed).
        text_encoder: the pipeline's CLIP text tower with its tokenizer (model.clip_text.CLIPTextTower), which becomes
        clip_text; exactly one of clip_text / text_encoder is given (ValueError otherwise), and a tower whose sequence length,
        hidden size or projection width does not fit the prior raises K2Error."""
        if (clip_text is None) == (text_encoder is None):
            raise ValueError("PriorEmbedder22.from_diffusers: pass exactly one of clip_text= and text_encoder=")
        if image_encoder is not None:
            if kwargs.get("clip_image") is not None:
                raise ValueError("PriorEmbedder22.from_diffusers: pass image_encoder= or clip_image=, not both")
            kwargs["clip_image"] = image_encoder
            if kwargs.get("zero_image_emb") is None:
                kwargs["zero_image_emb"] = image_encoder.zero_embed().float().cpu()
        from ..checkpoints import diffusers_prior_to_k2
        sd, mean, std = diffusers_prior_to_k2(state_dict)
        W = sd["positional_embedding"].shape[-1]
        layers = sum(1 for k in sd if k.endswith(".attn.c_qkv.weight"))
        prior = PriorTransformer(text_ctx=sd["positional_embedding"].shape[1] - 4, xf_width=W, xf_layers=layers, xf_heads=W // 64,
                                 xf_final_ln=True, xf_padding=False, clip_dim=sd["out_proj.weight"].shape[0],
                                 clip_xf_width=sd["text_enc_proj.weight"].shape[1], device=device)
        if text_encoder is not None:
            c = text_encoder.cfg
            got = (text_encoder.tokens, c["hidden_size"], c["projection_dim"])
            want = (prior.text_ctx, prior.clip_xf_width, prior.clip_dim)
            if got != want:
                raise K2Error(f"PriorEmbedder22.from_diffusers: the text encoder gives (tokens, hidden, projection) {got}, "
                              f"the prior takes (text_ctx, clip_xf_width, clip_dim) {want}")
            clip_text = text_encoder
        prior.load_state_dict(sd, strict=True)
        return cls(prior.finalize(), clip_text, mean.to(device).float(), std.to(device).float(), **kwargs)

    @classmethod
    def from_pretrained(cls, path, device="cuda", **kwargs):
        """A local `kandinsky-2-2-prior` folder (the diffusers layout) -> the embedder with its own CLIP text tower and
        tokenizer, and its CLIP image tower when the folder has one:
            prior/           diffusion_pytorch_model.{safetensors,bin}
            text_encoder/    config.json, model.{safetensors,bin}
            tokenizer/       vocab.json, merges.txt (+ special_tokens_map.json, tokenizer_config.json)
            image_encoder/   config.json, model.{safetensors,bin}           (optional)
            image_processor/ preprocessor_config.json                       (optional)
        *.safetensors are read when the safetensors package imports, else the .bin files (torch.load, weights_only).  A
        missing file raises K2Error naming it.  kwargs go to from_diffusers (prior_steps, seed, ...)."""
        from ..checkpoints import load_weights, read_json
        from .clip_text import CLIPTextTower, CLIPTokenizer
        what = "PriorEmbedder22.from_pretrained"

        def weights(sub, stem):
            return load_weights(os.path.join(path, sub), (f"{stem}.safetensors", f"{stem}.bin"), what)

        tower = CLIPTextTower.from_transformers(weights("text_encoder", "model"),
                                                read_json(os.path.join(path, "text_encoder"), "config.json", what), device,
                                                CLIPTokenizer.from_dir(os.path.join(path, "tokenizer")))
        if os.path.isdir(os.path.join(path, "image_encoder")) and kwargs.get("image_encoder") is None:
            from .clip_vision import CLIPVisionTower
            proc = (read_json(os.path.join(path, "image_processor"), "preprocessor_config.json", what)
                    if os.path.isdir(os.path.join(path, "image_processor")) else None)
            kwargs["image_encoder"] = CLIPVisionTower.from_transformers(
                weights("image_encoder", "model"), read_json(os.path.join(path, "image_encoder"), "config.json", what), device,
                proc)
        return cls.from_diffusers(weights("prior", "diffusion_pytorch_model"), device=device, text_encoder=tower, **kwargs)

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
        keep = self._emb2emb_keep(steps, strength)
        sched = UnCLIPSchedule(steps, keep=keep)
        dev, B, D = self.clip_mean.device, batch_size, self.prior.clip_dim
        emb = self._image_embedding(image, B)
        steps, g, rows, gen = self._call_args(prompt, B, steps, prior_guidance_scale, negative_prior_prompt)
        z = torch.randn(B, D, device=dev, generator=gen)
        noise = torch.randn(keep, B, D, device=dev, generator=gen)
        return sample_prior22(self.prior, *rows, steps, g, self.clip_mean, self.clip_std, sched.start_latent(emb, z), noise,
                              use_graph=self.use_cuda_graph, keep=keep).float().cpu()

    def batcher(self, max_batch):
        """A batching.PriorBatcher: image_emb(prompt, 1, ...) and emb2emb(prompt, image, 1, ...) requests submitted one at a
        time and sampled in one continuously refilled batch of max_batch slots, every slot at its own UnCLIP step, one CUDA
        graph replay per step; each result is the embedding the batch-1 call computes, left on the device."""
        from ..batching import PriorBatcher
        return PriorBatcher(self, max_batch)

    @staticmethod
    def _emb2emb_keep(steps, strength, who="PriorEmbedder22.emb2emb"):
        """The UnCLIP steps emb2emb runs of `steps` at `strength` (get_timesteps): min(int(N * strength), N); ValueError for
        a strength outside [0, 1] or one that keeps no step."""
        strength = float(strength)
        if not 0.0 <= strength <= 1.0:
            raise ValueError(f"{who}: strength must be in [0, 1], got {strength}")
        keep = min(int(steps * strength), steps)
        if keep == 0:
            raise ValueError(f"{who}: strength {strength} keeps no step of {steps} (int(N * strength) = 0)")
        return keep

    def _image_embedding(self, image, B, who="PriorEmbedder22.emb2emb"):
        """emb2emb's image -> its CLIP image embedding [B, clip_dim] on the device: a tensor [1, clip_dim] / [clip_dim]
        (repeated) or [B, clip_dim], or a PIL image through clip_image."""
        dev, D = self.clip_mean.device, self.prior.clip_dim
        if torch.is_tensor(image):
            emb = image.float().reshape(-1, D) if image.dim() == 1 else image.float()
            if emb.dim() != 2 or emb.shape[1] != D or emb.shape[0] not in (1, B):
                raise ValueError(f"{who}: an image embedding must be [1, {D}] or [{B}, {D}], got {list(image.shape)}")
        else:
            if self.clip_image is None:
                raise K2Error(f"{who}: a PIL image needs clip_image=")
            emb = self.clip_image(image).float().reshape(1, D)
        return emb.to(dev).expand(B, D)

    def zero_image_emb(self, batch_size):
        """diffusers' KandinskyV22PriorPipeline.get_zero_embed: the CLIP image tower on all-zero pixel_values, supplied by the
        deployment or by from_diffusers(image_encoder=...); zeros when absent."""
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
