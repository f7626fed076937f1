"""TEST INFRASTRUCTURE (oracle): CPU restatement of the Kandinsky 2.1 diffusion prior -- SURVEY.md section 8f, rank 3 (the
step BEFORE the hot path; not implemented in the product this round, the oracle and its golden fixture are the groundwork).

  prior_forward    <- PriorTransformer.forward                      (kandinsky2/model/prior.py:159-270)
                      ResidualAttentionBlock / MultiheadAttention / QKVMultiheadAttention / MLP  (:57-127)
  prior_sample     <- PriorDiffusionModel.forward (guided_model_fn, p_sample_loop with predict_xstart, fixed small variance,
                      cosine schedule, x0 clamped to +-10)         (prior.py:336-384; gaussian_diffusion.py:223-322,352-382)

Pinned by oracle/make_golden.py (`prior_tiny.pt`: the reference classes executed on synthetic weights)."""
import math

import numpy as np
import torch
import torch.nn.functional as F

CONFIG_PRIOR = dict(text_ctx=77, xf_width=2048, xf_layers=20, xf_heads=32, xf_final_ln=True, xf_padding=False, clip_dim=768,
                    clip_xf_width=768)                                        # configs.py:101-111
CONFIG_PRIOR_TINY = dict(text_ctx=5, xf_width=128, xf_layers=2, xf_heads=2, xf_final_ln=True, xf_padding=False, clip_dim=32,
                         clip_xf_width=48)


def prior_param_spec(cfg):
    """[(state_dict key, shape)] in the reference's registration order (prior.py:191-228)."""
    W, C, X, n = cfg["xf_width"], cfg["clip_dim"], cfg["clip_xf_width"], cfg["text_ctx"] + 4
    spec = [("positional_embedding", (1, n, W)), ("prd_emb", (1, 1, W))]
    if cfg["xf_padding"]:
        spec.append(("padding_embedding", (n, W)))
    spec += [("time_embed.0.weight", (W, W)), ("time_embed.0.bias", (W,)), ("time_embed.2.weight", (W, W)),
             ("time_embed.2.bias", (W,)), ("text_enc_proj.weight", (W, X)), ("text_enc_proj.bias", (W,)),
             ("text_emb_proj.weight", (W, C)), ("text_emb_proj.bias", (W,)), ("clip_img_proj.weight", (W, C)),
             ("clip_img_proj.bias", (W,)), ("out_proj.weight", (C, W)), ("out_proj.bias", (C,))]
    for i in range(cfg["xf_layers"]):
        p = f"transformer.resblocks.{i}."
        spec += [(p + "attn.c_qkv.weight", (3 * W, W)), (p + "attn.c_qkv.bias", (3 * W,)),
                 (p + "attn.c_proj.weight", (W, W)), (p + "attn.c_proj.bias", (W,)),
                 (p + "ln_1.weight", (W,)), (p + "ln_1.bias", (W,)),
                 (p + "mlp.c_fc.weight", (4 * W, W)), (p + "mlp.c_fc.bias", (4 * W,)),
                 (p + "mlp.c_proj.weight", (W, 4 * W)), (p + "mlp.c_proj.bias", (W,)),
                 (p + "ln_2.weight", (W,)), (p + "ln_2.bias", (W,))]
    if cfg["xf_final_ln"]:
        spec += [("final_ln.weight", (W,)), ("final_ln.bias", (W,))]
    return spec


def _timestep_embedding(t, dim, max_period=10000):  # prior.py:15-35 (cos first, like model/nn.py)
    half = dim // 2
    freqs = torch.exp(-math.log(max_period) * torch.arange(half, dtype=torch.float32, device=t.device) / half)
    args = t[:, None].float() * freqs[None]
    return torch.cat([torch.cos(args), torch.sin(args)], dim=-1)


def prior_forward(sd, cfg, x, timesteps, text_emb, text_enc, mask, fp16=False):
    """x [N, clip_dim] noisy image embedding, text_emb [N, clip_dim], text_enc [N, text_ctx, clip_xf_width], mask [N, text_ctx]
    bool (True = real token) -> predicted x0 [N, clip_dim] (the last position of the causal transformer).  Runs on the
    device of the inputs.

    fp16=True: the reference's fp16 mode (Kandinsky2_1.__init__ calls prior.half() under use_fp16): sd holds fp16 tensors,
    every Linear and einsum is fp16, LayerNorm computes in fp32 and returns fp16 (prior.py:48-54 on a CUDA fp16 tensor),
    the fp32 additive mask promotes the scores to fp32 for the softmax, whose result is cast back to fp16 (prior.py:102)."""
    W, H = cfg["xf_width"], cfg["xf_heads"]
    N = x.shape[0]
    dt = torch.float16 if fp16 else torch.float32
    x, text_emb, text_enc = x.to(dt), text_emb.to(dt), text_enc.to(dt)
    lin = lambda name, v: F.linear(v, sd[name + ".weight"], sd[name + ".bias"])  # noqa: E731
    ln = lambda v, name: F.layer_norm(v.float(), (W,), sd[name + ".weight"].float(), sd[name + ".bias"].float()).to(dt)  # noqa: E731
    mask = F.pad(mask, (0, 4), value=True)                                       # ext_len = 4 extra positions
    t_emb = lin("time_embed.2", F.silu(lin("time_embed.0", _timestep_embedding(timesteps, W).to(dt))))
    seq = torch.cat([lin("text_enc_proj", text_enc), lin("text_emb_proj", text_emb)[:, None], t_emb[:, None],
                     lin("clip_img_proj", x)[:, None], sd["prd_emb"].expand(N, -1, -1)], dim=1)
    seq = seq + sd["positional_embedding"]
    if cfg["xf_padding"]:
        seq = torch.where(mask[..., None], seq, sd["padding_embedding"][None])
    n = seq.shape[1]
    causal = torch.full((n, n), float("-inf"), device=seq.device).triu_(1)
    add = torch.where(mask, 0.0, float("-inf"))[:, None, :] + causal[None]       # [N, n, n] fp32
    d = W // H
    scale = 1 / math.sqrt(math.sqrt(d))
    h = seq
    for i in range(cfg["xf_layers"]):
        p = f"transformer.resblocks.{i}."
        y = ln(h, p + "ln_1")
        qkv = lin(p + "attn.c_qkv", y).view(N, n, H, 3 * d)                      # per head [q | k | v]  (prior.py:92-95)
        q, k, v = torch.split(qkv, d, dim=-1)
        w = torch.einsum("bthc,bshc->bhts", q * scale, k * scale) + add[:, None]
        a = torch.einsum("bhts,bshc->bthc", torch.softmax(w, dim=-1).to(dt), v).reshape(N, n, W)
        h = h + lin(p + "attn.c_proj", a)
        y = ln(h, p + "ln_2")
        h = h + lin(p + "mlp.c_proj", F.gelu(lin(p + "mlp.c_fc", y)))
    if cfg["xf_final_ln"]:
        h = ln(h, "final_ln")
    return lin("out_proj", h[:, -1]).float()


def cosine_betas(steps=1000, max_beta=0.999):
    """get_named_beta_schedule('cosine') (model/utils.py / gaussian_diffusion.py betas_for_alpha_bar)."""
    f = lambda t: math.cos((t + 0.008) / 1.008 * math.pi / 2) ** 2  # noqa: E731
    return np.array([min(1 - f((i + 1) / steps) / f(i / steps), max_beta) for i in range(steps)], dtype=np.float64)


def prior_sample(model_fn, x_T, step_noise, use_steps, guidance, clip_mean, clip_std, base_steps=1000):
    """PriorDiffusionModel.forward with timestep_respacing=str(len(use_steps)): predict_xstart, FIXED_SMALL variance (posterior
    variance, log clipped), rescale_timesteps False, x0 clamped to +-10, CFG on the predicted x0 rows (cond first).
    model_fn(x[2B], t[2B]) -> x0 prediction [2B, D]; x_T [B, D]; step_noise [steps, B, D]."""
    betas_full = cosine_betas(base_steps)
    acp_full = np.cumprod(1.0 - betas_full)
    last, betas = 1.0, []
    for i in use_steps:                                    # respace.py:83-97
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
    x = x_T
    for n, i in enumerate(range(len(use_steps))[::-1]):
        t = torch.full((2 * B,), float(use_steps[i]), device=x.device)  # _WrappedModel: timestep_map[i], no rescaling
        out = model_fn(torch.cat([x, x]), t)
        cond, uncond = out[:B], out[B:]
        x0 = (uncond + guidance * (cond - uncond)).clamp(-10, 10)
        x = float(np.float32(c1[i])) * x0 + float(np.float32(c2[i])) * x
        if i != 0:                                         # nonzero_mask of p_sample
            x = x + math.exp(0.5 * float(np.float32(post_logvar[i]))) * step_noise[n]
    return x * clip_std + clip_mean
