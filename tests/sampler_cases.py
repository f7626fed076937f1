"""What the tests of the schedule samplers (pipelines.SCHEDULE_SAMPLERS) share: the base tables, the tiny-UNet trajectory
fixture, the tiny pipelines, the loop bound, and one float64 oracle loop per sampler name."""
import os

import torch

from tests import dpm_oracle as do
from tests import dpm_sde_oracle as so
from tests import kdiff_oracle as ko
from tests import unipc_oracle as uo

GOLD = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")

# sigma-space sampler name -> (kdiff_oracle scheduler, Karras sigmas, the step kernel formula its rows are applied with)
KINDS = {"euler_sampler": ("euler", False, "dpm"),
         "euler_karras_sampler": ("euler", True, "dpm"),
         "euler_ancestral_sampler": ("euler_ancestral", False, "dpm"),
         "heun_sampler": ("heun", False, "heun"),
         "heun_karras_sampler": ("heun", True, "heun")}


def _schedule(name, ac, n, keep=None):
    """The schedule of a SCHEDULE_SAMPLERS name over the base table ac."""
    from kandinsky2.pipelines import SCHEDULE_SAMPLERS
    cls, kw = SCHEDULE_SAMPLERS[name]
    return cls(ac, n, keep=keep, **kw)


def _ac22():
    from kandinsky2.model.gaussian_diffusion import create_ddpm_v22
    return create_ddpm_v22(50).base_alphas_cumprod


def _base21():
    from kandinsky2.configs import CONFIG_2_1
    from kandinsky2.model.gaussian_diffusion import create_gaussian_diffusion
    return create_gaussian_diffusion(**CONFIG_2_1["diffusion_config"]).base_alphas_cumprod


def _no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


def _traj_tiny():
    """-> (the traj_tiny fixture, its synthetic weights, the product UNet built from them)"""
    from oracle import synth, unet_oracle as uo_net
    from tests.test_gpu_unet import _build
    fx = torch.load(os.path.join(GOLD, "traj_tiny.pt"), weights_only=False)
    sd = synth.synth_state_dict(uo_net.unet_param_spec(fx["cfg"]), seed=fx["weight_seed"])
    return fx, sd, _build(fx["cfg"], sd)


def oracle(name, eps, ac, n, z, step_noise=None, inpaint=None, inpaint_renoise=True):
    """The float64 oracle loop of sampler `name`, n steps over the base table ac, from the unit start noise z -> the final
    latent.  eps(x, t): the guided epsilon at the UNet input x and timestep t.  step_noise: the per-step draws of a name that
    draws noise.  inpaint = (init, mask): Kandinsky 2.2's rule (the known region re-noised with z), or 2.1's with
    inpaint_renoise=False (the known region replaces the x0 prediction; UniPC and the sigma-space names only)."""
    z = z.clone()
    if name in KINDS:
        kind, karras, _ = KINDS[name]
        return ko.sample(kind, eps, ac, n, z, karras=karras, step_noise=step_noise, inpaint=inpaint,
                         inpaint_renoise=inpaint_renoise)
    sch = _schedule(name, ac, n)
    # the oracle's own linspace grid; the Karras grid is the product's, which the CPU tests check against its restatement
    tau, alpha, sigma = do.grid(ac, n) if sch.spacing == "linspace" else (sch.timesteps, sch.alphas, sch.sigmas)
    eps_k = lambda x, k: eps(x, float(tau[k]))
    inp = None if inpaint is None else (*inpaint, z)
    if sch.step_kind == "unipc":
        return uo.solve(eps_k, z, alpha, sigma, inpaint=inp, inpaint_renoise=inpaint_renoise)
    assert inpaint is None or inpaint_renoise, "the DPM-Solver++ oracles restate the 2.2 inpainting rule only"
    if sch.draws_noise:
        return so.solve_sde(eps_k, z, alpha, sigma, step_noise, inpaint=inp)
    return do.solve(eps_k, z, alpha, sigma, inpaint=inp)


def _check(out, ref, what):
    """The bound of every tiny-UNet loop against its oracle: relative L2 < 2e-2 and max abs < 0.15 max |ref|."""
    err = (out - ref).abs().max().item()
    rel = ((out - ref).norm() / ref.norm()).item()
    print(f"{what}: rel L2 {rel:.3e}, max abs {err:.3e}")
    assert torch.isfinite(out).all()
    assert rel < 2e-2 and err < 0.15 * ref.abs().max().item(), (what, err, rel, ref.abs().max().item())


# ---- pipelines -----------------------------------------------------------------------------------------------------------
# With the random weights of the tiny configs the solver latents (no clamp on these paths) reach magnitudes that saturate the
# MoVQ decoder to black images, so the pipeline tests compare the denoised latents handed to the decoder, and the images
# where they must be identical.
def _pipe(version, task):
    from kandinsky2 import get_kandinsky2
    from tests.test_gpu_movq_sampler import _tiny_overrides
    pipe = get_kandinsky2("cuda", task_type=task, model_version=version, cache_dir="/nonexistent",
                          config_overrides=_tiny_overrides())
    pipe.seen = []
    orig = pipe._finish

    def finish(latents, h, w):
        pipe.seen.append(latents.clone())
        return orig(latents, h, w)
    pipe._finish = finish
    return pipe


def _run(pipe, method, *args, **kw):
    """-> (images, the latents the call decoded)"""
    imgs = getattr(pipe, method)(*args, **kw)
    return imgs, pipe.seen[-1]


def _same(a, b):
    return len(a) == len(b) and all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
