"""TEST INFRASTRUCTURE (oracle): the two image-guided Kandinsky 2.2 loops of the reference's ControlNet notebook
(notebooks/kandinsky2_2_controlnet.ipynb), restated in float64 with injected noise (diffusers is not installed, so unpinned).

  emb2emb_sample         <- KandinskyV22PriorEmb2EmbPipeline.__call__: get_timesteps keeps the last min(int(N * strength), N) of
                            UnCLIPScheduler's N timesteps; prepare_latents starts from UnCLIPScheduler.add_noise of the image
                            embedding (NOT normalised by clip_mean / clip_std) at the first kept timestep; the step passes
                            prev_timestep = timesteps[i + 1] of the FULL list (None, i.e. t - 1, after the last);
                            post_process_latents returns x * clip_std + clip_mean
  controlnet_img2img_loop <- KandinskyV22ControlnetImg2ImgPipeline.__call__: DDPMScheduler (leading spacing, learned_range,
                            clip +-2) over timesteps[t_start:], t_start = N - min(int(N * strength), N), from
                            DDPMScheduler.add_noise of the image latent at timesteps[t_start]; the arithmetic of
                            oracle/diffusion_oracle.py's ddpm_v22_loop, the hint entering through unet_fn
"""
import math

import numpy as np
import torch

from tests import prior22_oracle as p22


def keep_of(num_steps, strength):
    """get_timesteps of both pipelines: how many of the N steps run."""
    return min(int(num_steps * strength), num_steps)


def emb2emb_sample(model_fn, image_emb, z, step_noise, num_steps, strength, guidance, clip_mean, clip_std, T=1000):
    """model_fn(x [2B or B, D], t [same]) -> predicted x0, rows [uncond | cond] under guidance > 1, else the B conditional rows
    alone.  image_emb, z [B, D]; step_noise [keep, B, D].  float64 scheduler arithmetic; returns float64."""
    f = lambda t: math.cos((t / T + 0.008) / 1.008 * math.pi / 2) ** 2  # noqa: E731
    betas = np.array([min(1 - f(i + 1) / f(i), 0.999) for i in range(T)])
    acp = np.cumprod(1.0 - betas)
    full = p22.unclip_timesteps(num_steps, T)
    t_start = max(num_steps - keep_of(num_steps, strength), 0)
    ts = full[t_start:]
    a0 = acp[int(ts[0])]
    x = a0 ** 0.5 * image_emb.double() + (1 - a0) ** 0.5 * z.double()
    B = x.shape[0]
    for i, t in enumerate(ts):
        cfg = guidance > 1.0
        xin = torch.cat([x, x]) if cfg else x
        pred = model_fn(xin.float(), torch.full((xin.shape[0],), float(t), device=x.device)).double()
        if cfg:
            uncond, cond = pred[:B], pred[B:]
            pred = uncond + guidance * (cond - uncond)
        prev_t = int(ts[i + 1]) if i + 1 < len(ts) else int(t) - 1
        a = acp[t]
        ap = acp[prev_t] if prev_t >= 0 else 1.0
        beta = betas[t] if prev_t == t - 1 else 1 - a / ap
        x0 = pred.clamp(-10, 10)
        x = (ap ** 0.5 * beta / (1 - a)) * x0 + ((1 - beta) ** 0.5 * (1 - ap) / (1 - a)) * x
        if t > 0:
            var = math.log(max((1 - ap) / (1 - a) * beta, 1e-20))
            x = x + math.exp(0.5 * var) * step_noise[i].double()
    return x * clip_std.double() + clip_mean.double()


def controlnet_img2img_loop(unet_fn, latent, noise0, steps, strength, guidance, step_noise, train_steps=1000,
                            beta_start=0.00085, beta_end=0.012):
    """unet_fn(x [2B], t [2B]) -> [2B, 8, h, w], unconditional rows first (the hint is unet_fn's business); latent, noise0
    [B, 4, h, w]; step_noise [keep, B, 4, h, w].  Returns the final latent [B, 4, h, w]."""
    betas = np.linspace(beta_start, beta_end, train_steps, dtype=np.float64)
    ac = np.cumprod(1.0 - betas)
    ratio = train_steps // steps
    timesteps = (np.arange(steps) * ratio)[::-1]
    t_start = max(steps - keep_of(steps, strength), 0)
    timesteps = timesteps[t_start:]
    a0 = ac[timesteps[0]]
    x = a0 ** 0.5 * latent + (1.0 - a0) ** 0.5 * noise0
    B = x.shape[0]
    f32 = lambda v: float(np.float32(v))  # noqa: E731
    for n, t in enumerate(timesteps):
        out = unet_fn(torch.cat([x, x], 0), torch.full((2 * B,), float(t)))
        eps, var = out[:, :4], out[:, 4:]
        e = eps[:B] + guidance * (eps[B:] - eps[:B])
        v = var[B:]
        prev_t = t - ratio
        a_t, a_prev = ac[t], (ac[prev_t] if prev_t >= 0 else 1.0)
        b_t, b_prev = 1.0 - a_t, 1.0 - a_prev
        cur_alpha = a_t / a_prev
        cur_beta = 1.0 - cur_alpha
        x0 = ((x - f32(b_t ** 0.5) * e) / f32(a_t ** 0.5)).clamp(-2.0, 2.0)
        mean = f32(a_prev ** 0.5 * cur_beta / b_t) * x0 + f32(cur_alpha ** 0.5 * b_prev / b_t) * x
        if t > 0:
            min_log = np.log(max(b_prev / b_t * cur_beta, 1e-20))
            max_log = np.log(cur_beta)
            frac = (v + 1) / 2
            mean = mean + torch.exp(0.5 * (frac * f32(max_log) + (1 - frac) * f32(min_log))) * step_noise[n]
        x = mean
    return x
