"""TEST INFRASTRUCTURE (oracle): the Kandinsky 2.2 diffusion prior in diffusers' form, restated (diffusers is not installed).

  diffusers_prior_spec   <- the state dict of diffusers' `PriorTransformer` as kandinsky-community/kandinsky-2-2-prior
                            configures it (20 blocks, 32 heads of 64, embedding_dim 1280, 77 + 4 tokens, added_emb_type "prd",
                            encoder_hid_proj_type "linear", norm_in_type None)
  diffusers_prior_forward <- PriorTransformer.forward: separate to_q / to_k / to_v, the additive mask
                            (1 - mask) * -10000 plus the -10000 upper triangle, in the model dtype; norm_out over all tokens,
                            then the last token
  unclip_sample          <- KandinskyV22PriorPipeline.__call__ with UnCLIPScheduler(squaredcos_cap_v2, "sample",
                            "fixed_small_log", clip_sample_range 10) in float64, with injected noise

Restated, so unpinned.  What is pinned: after kandinsky2.checkpoints.diffusers_prior_to_k2, diffusers_prior_forward equals
oracle/prior_oracle.py's prior_forward (the reference's own network) on the CPU in fp32 (tests/test_cpu_prior22.py)."""
import math

import numpy as np
import torch
import torch.nn.functional as F

CONFIG_PRIOR22 = dict(text_ctx=77, xf_width=2048, xf_layers=20, xf_heads=32, xf_final_ln=True, xf_padding=False, clip_dim=1280,
                      clip_xf_width=1280)
CONFIG_PRIOR22_TINY = dict(text_ctx=5, xf_width=128, xf_layers=2, xf_heads=2, xf_final_ln=True, xf_padding=False, clip_dim=32,
                           clip_xf_width=32)


def diffusers_prior_spec(cfg):
    """[(diffusers key, shape)] of the 2.2 prior at cfg (this package's PriorTransformer keywords)."""
    W, D, X, n = cfg["xf_width"], cfg["clip_dim"], cfg["clip_xf_width"], cfg["text_ctx"] + 4
    spec = [("positional_embedding", (1, n, W)), ("prd_embedding", (1, 1, W)), ("clip_mean", (1, D)), ("clip_std", (1, D))]
    for name, (o, i) in (("time_embedding.linear_1", (W, W)), ("time_embedding.linear_2", (W, W)), ("proj_in", (W, D)),
                         ("embedding_proj", (W, D)), ("encoder_hidden_states_proj", (W, X)), ("proj_to_clip_embeddings", (D, W))):
        spec += [(name + ".weight", (o, i)), (name + ".bias", (o,))]
    spec += [("norm_out.weight", (W,)), ("norm_out.bias", (W,))]
    for i in range(cfg["xf_layers"]):
        p = f"transformer_blocks.{i}."
        spec += [(p + "norm1.weight", (W,)), (p + "norm1.bias", (W,)), (p + "norm3.weight", (W,)), (p + "norm3.bias", (W,))]
        for name, (o, k) in (("attn1.to_q", (W, W)), ("attn1.to_k", (W, W)), ("attn1.to_v", (W, W)), ("attn1.to_out.0", (W, W)),
                             ("ff.net.0.proj", (4 * W, W)), ("ff.net.2", (W, 4 * W))):
            spec += [(p + name + ".weight", (o, k)), (p + name + ".bias", (o,))]
    return spec


def _time_proj(t, dim):  # diffusers Timesteps(dim, flip_sin_to_cos=True, downscale_freq_shift=0)
    half = dim // 2
    freqs = torch.exp(-math.log(10000) * torch.arange(half, dtype=torch.float32, device=t.device) / half)
    args = t[:, None].float() * freqs[None]
    return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


def diffusers_prior_forward(sd, cfg, x, timesteps, text_emb, text_enc, mask, dtype=torch.float32):
    """x [N, D], timesteps [N], text_emb [N, D], text_enc [N, text_ctx, X], mask [N, text_ctx] bool (True = real token) ->
    predicted image embedding [N, D] fp32.  sd: diffusers keys, in `dtype`."""
    W, H = cfg["xf_width"], cfg["xf_heads"]
    N, d = x.shape[0], W // H
    lin = lambda name, v: F.linear(v, sd[name + ".weight"], sd[name + ".bias"])  # noqa: E731
    ln = lambda v, name: F.layer_norm(v, (W,), sd[name + ".weight"], sd[name + ".bias"])  # noqa: E731
    x, text_emb, text_enc = x.to(dtype), text_emb.to(dtype), text_enc.to(dtype)
    t_emb = lin("time_embedding.linear_2", F.silu(lin("time_embedding.linear_1", _time_proj(timesteps, W).to(dtype))))
    h = torch.cat([lin("encoder_hidden_states_proj", text_enc), lin("embedding_proj", text_emb)[:, None], t_emb[:, None],
                   lin("proj_in", x)[:, None], sd["prd_embedding"].expand(N, -1, -1)], dim=1)
    h = h + sd["positional_embedding"].to(dtype)
    n = h.shape[1]
    causal = torch.full((n, n), -10000.0, device=x.device).triu_(1)
    add = F.pad((1 - mask.to(dtype)) * -10000.0, (0, 4), value=0.0)
    add = (add[:, None, :] + causal).to(dtype)                                   # [N, n, n]
    for i in range(cfg["xf_layers"]):
        p = f"transformer_blocks.{i}."
        y = ln(h, p + "norm1")
        q, k, v = (lin(p + f"attn1.to_{c}", y).view(N, n, H, d).transpose(1, 2) for c in "qkv")
        w = (q @ k.transpose(-1, -2)) / math.sqrt(d) + add[:, None]
        a = (torch.softmax(w.float(), dim=-1).to(dtype) @ v).transpose(1, 2).reshape(N, n, W)
        h = h + lin(p + "attn1.to_out.0", a)
        y = ln(h, p + "norm3")
        h = h + lin(p + "ff.net.2", F.gelu(lin(p + "ff.net.0.proj", y)))
    h = ln(h, "norm_out")
    return lin("proj_to_clip_embeddings", h[:, -1]).float()


def unclip_timesteps(num_steps, T=1000):
    step_ratio = (T - 1) / (num_steps - 1)
    return (np.arange(num_steps) * step_ratio).round()[::-1].astype(np.int64)


def unclip_sample(model_fn, x_T, step_noise, num_steps, guidance, clip_mean, clip_std, T=1000):
    """model_fn(x [2B or B, D], t [same]) -> predicted x0.  Rows [uncond | cond] under guidance > 1, else the B conditional
    rows alone (diffusers' do_classifier_free_guidance).  The scheduler arithmetic is float64; returns float64."""
    f = lambda t: math.cos((t / T + 0.008) / 1.008 * math.pi / 2) ** 2  # noqa: E731
    betas = np.array([min(1 - f(i + 1) / f(i), 0.999) for i in range(T)])
    acp = np.cumprod(1.0 - betas)
    ts = unclip_timesteps(num_steps, T)
    x = x_T.double()
    B = x.shape[0]
    for k, t in enumerate(ts):
        cfg = guidance > 1.0
        xin = torch.cat([x, x]) if cfg else x
        pred = model_fn(xin.float(), torch.full((xin.shape[0],), float(t), device=x.device)).double()
        if cfg:
            uncond, cond = pred[:B], pred[B:]
            pred = uncond + guidance * (cond - uncond)
        prev_t = int(ts[k + 1]) if k + 1 < len(ts) else int(t) - 1
        a = acp[t]
        ap = acp[prev_t] if prev_t >= 0 else 1.0
        if prev_t == t - 1:
            beta = betas[t]
        else:
            beta = 1 - a / ap
        alpha = 1 - beta
        x0 = pred.clamp(-10, 10)
        x = (ap ** 0.5 * beta / (1 - a)) * x0 + (alpha ** 0.5 * (1 - ap) / (1 - a)) * x
        if t > 0:
            var = math.log(max((1 - ap) / (1 - a) * beta, 1e-20))
            x = x + math.exp(0.5 * var) * step_noise[k].double()
    return x * clip_std.double() + clip_mean.double()
