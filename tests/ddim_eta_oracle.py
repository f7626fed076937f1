"""Restatement of the reference's DDIM step with eta > 0 (kandinsky2/model/samplers.py:21-31 make_ddim_sampling_parameters,
:289-331 p_sample_ddim), and the writer of its golden fixture tests/golden/ddim_eta_tiny.pt.

Test infrastructure.  It extends the eta = 0 restatement of oracle/diffusion_oracle.py (ddim_schedule, the CFG closure) with
the noise term and leaves that module as it is.  The fixture is written by EXECUTING THE REFERENCE (needs the reference tree,
see oracle/ref_shim.py), on its own so that no existing fixture is rewritten:

    python -m tests.ddim_eta_oracle
"""
import os

import numpy as np
import torch

from oracle import diffusion_oracle as do

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "ddim_eta_tiny.pt")


def ddim_eta_schedule(num_steps, eta, base_betas=None):
    """-> (t, alphas, alphas_prev, sigmas): make_ddim_timesteps('uniform') + make_ddim_sampling_parameters(eta)."""
    t, al, alp = do.ddim_schedule(num_steps, base_betas)
    sig = eta * np.sqrt((1 - alp) / (1 - al) * (1 - al / alp))
    return t, al, alp, sig


def ddim_eta_step(x, eps, a_t, a_prev, sigma, noise):
    """p_sample_ddim (model/samplers.py:311-330): x' = sqrt(a_prev) x0 + sqrt(1 - a_prev - sigma^2) eps + sigma z."""
    pred_x0 = (x - (1.0 - a_t) ** 0.5 * eps) / a_t ** 0.5
    return a_prev ** 0.5 * pred_x0 + (1.0 - a_prev - sigma ** 2) ** 0.5 * eps + sigma * noise


def ddim_eta_sample_loop(unet_fn, x_T, num_steps, guidance, eta, step_noise):
    """DDIMSampler.sample(eta=eta) with the per-step noise injected: step_noise[n] is the noise of the n-th step run.
    unet_fn(x[2B], t[2B]) -> [2B, 8, H, W] with the cond rows first; x_T: [B, 4, H, W].  The reference casts each per-step
    scalar to fp32 (torch.full on the float64 tables)."""
    tt, al, alp, sig = ddim_eta_schedule(num_steps, eta)
    f32 = lambda v: float(np.float32(v))
    x = x_T
    for n, i in enumerate(range(len(tt))[::-1]):
        eps = do._cfg_eps(unet_fn, x, tt[i], guidance)
        x = ddim_eta_step(x, eps, f32(al[i]), f32(alp[i]), f32(sig[i]), step_noise[n])
    return x


def golden_ddim_eta(cfg=None, B=2, H=16, W=16, ntext=7, steps=4, guidance=3.0, eta=0.5, wseed=1, iseed=21):
    """The reference's own DDIMSampler.sample(..., eta=eta) on the tiny reference UNet (the set-up of oracle/make_golden.py's
    golden_sampler).  Its noise is captured by wrapping the loaded module's noise_like; the first B rows of each step's
    noise (the rows of the tracked half) are stored.  Asserts oracle == reference to 1e-4 before writing."""
    from oracle import ref_shim, synth, unet_oracle as uo
    from oracle.make_golden import build_ref_unet, unet_inputs
    cfg = uo.CONFIG_TINY if cfg is None else cfg
    model = build_ref_unet(cfg)
    sd = synth.synth_state_dict(uo.unet_param_spec(cfg), seed=wseed)
    model.load_state_dict(sd, strict=True)
    inp = unet_inputs(cfg, 2 * B, H, W, ntext, iseed)
    g = torch.Generator().manual_seed(iseed + 300)
    x_T = torch.randn(B, 4, H, W, generator=g)
    kw = dict(full_emb=inp["full_emb"], pooled_emb=inp["pooled_emb"], image_emb=inp["image_emb"])
    drawn = []
    with ref_shim.reference_modules() as R, ref_shim.cuda_as_cpu():
        mc = R.load("model.model_creation")
        sm = R.load("model.samplers")
        diffusion = mc.create_gaussian_diffusion(steps=1000, learn_sigma=True, sigma_small=False, noise_schedule="linear",
                                                 use_kl=False, predict_xstart=False, rescale_timesteps=True,
                                                 rescale_learned_sigmas=True, timestep_respacing="",
                                                 linear_start=0.00085, linear_end=0.012)

        def model_fn(x_t, ts, **kwargs):  # kandinsky2_1_model.py:222-233, sampler != "p_sampler"
            half = x_t[: len(x_t) // 2]
            combined = torch.cat([half, half], dim=0)
            eps = model(combined, ts, **kwargs)[:, :4]
            cond_eps, uncond_eps = torch.split(eps, len(eps) // 2, dim=0)
            half_eps = uncond_eps + guidance * (cond_eps - uncond_eps)
            return torch.cat([half_eps, half_eps], dim=0)

        noise_like = sm.noise_like

        def capture(*a, **k):
            z = noise_like(*a, **k)
            drawn.append(z[:B].clone())
            return z
        sm.noise_like = capture
        torch.manual_seed(iseed + 301)
        sampler = sm.DDIMSampler(model=model_fn, old_diffusion=diffusion, schedule="linear")
        model.del_cache()
        with torch.no_grad():
            out, _ = sampler.sample(steps, 2 * B, (4, H, W), conditioning=kw, x_T=torch.cat([x_T, x_T]), eta=eta,
                                    verbose=False)
        out = out[:B].clone()
        ddim_t = np.asarray(sampler.ddim_timesteps).copy()
        sigmas = np.asarray(sampler.ddim_sigmas, dtype=np.float64).copy()
    step_noise = torch.stack(drawn)
    assert step_noise.shape == (steps, B, 4, H, W), step_noise.shape
    tt, _, _, sig = ddim_eta_schedule(steps, eta)
    assert np.array_equal(ddim_t, tt) and np.allclose(sigmas, sig, rtol=1e-12, atol=0), (sigmas, sig)
    with torch.no_grad():
        orc = ddim_eta_sample_loop(lambda xx, ts: uo.unet_forward(sd, cfg, xx, ts, **kw), x_T, steps, guidance, eta,
                                   step_noise)
    err = (out - orc).abs().max().item()
    assert err <= 1e-4, f"ddim_eta_tiny: oracle deviates from the reference by {err}"
    torch.save(dict(cfg=cfg, weight_seed=wseed, cond=kw, x_T=x_T.clone(), steps=steps, guidance=guidance, eta=eta,
                    step_noise=step_noise, sigmas=sigmas, out=out), FIXTURE)
    print(f"ddim_eta_tiny: final latent std {out.std():.4f}, oracle-vs-reference max abs {err:.2e}")


if __name__ == "__main__":
    golden_ddim_eta()
