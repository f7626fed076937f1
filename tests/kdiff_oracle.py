"""Float64 restatement of diffusers' EulerDiscreteScheduler, EulerAncestralDiscreteScheduler and HeunDiscreteScheduler with
timestep_spacing="linspace", epsilon prediction and s_churn = 0 (Karras et al. 2022, "Elucidating the Design Space of
Diffusion-Based Generative Models"), and of the pipeline loop around them.  diffusers is not a dependency: its classes are
restated here from their published source, not pinned against it.

Test infrastructure, like tests/dpm_oracle.py.  The product's path is kandinsky2/model/gaussian_diffusion.py: EulerSchedule /
HeunSchedule (one linear row per UNet evaluation, the latent kept in the UNet's input scale) + k2_dpm_solver_step /
k2_dpm_solver_sde_step / k2_heun_step.  Here everything is written in the schedulers' own form instead: the latent is x_ve
(the variance-exploding sample), the UNet is fed scale_model_input(x_ve) = x_ve / sqrt(sigma^2 + 1), and every step goes
through pred_original_sample and the derivative as diffusers computes them.  diffusers casts its sigmas and timesteps to
float32; that cast is not restated.

apply_rows restates the step kernels' formulas in float64, so the CPU tests can run a schedule's rows against `sample`."""
import numpy as np


# ---- set_timesteps ----------------------------------------------------------------------------------------------------
def table_sigmas(ac):
    ac = np.asarray(ac, dtype=np.float64)
    return np.sqrt((1.0 - ac) / ac)


def _sigma_to_t(sigma, log_sigmas):
    """diffusers' _sigma_to_t: the fractional timestep whose log sigma interpolates the table's log sigmas linearly."""
    log_sigma = np.log(np.maximum(sigma, 1e-10))
    dists = log_sigma - log_sigmas[:, np.newaxis]
    low_idx = np.cumsum((dists >= 0), axis=0).argmax(axis=0).clip(max=log_sigmas.shape[0] - 2)
    high_idx = low_idx + 1
    low, high = log_sigmas[low_idx], log_sigmas[high_idx]
    w = np.clip((low - log_sigma) / (low - high), 0, 1)
    t = (1 - w) * low_idx + w * high_idx
    return t.reshape(np.shape(sigma))


def set_timesteps(ac, n, karras=False, heun=False):
    """-> (timesteps, sigmas): set_timesteps(n) of the Euler schedulers (heun=False: n timesteps, n + 1 sigmas) or of Heun
    (2n - 1 interleaved timesteps t0, t1, t1, ..., t_{n-1}, t_{n-1}; 2n sigmas s0, s1, s1, ..., s_{n-1}, s_{n-1}, 0)."""
    T = len(ac)
    timesteps = np.linspace(0, T - 1, n, dtype=np.float64)[::-1].copy()
    sig = table_sigmas(ac)
    log_sigmas = np.log(sig)
    sigmas = np.interp(timesteps, np.arange(0, T), sig)
    if karras:                                                   # _convert_to_karras, rho = 7
        rho = 7.0
        sigma_min, sigma_max = sigmas[-1], sigmas[0]
        ramp = np.linspace(0, 1, n)
        min_inv, max_inv = sigma_min ** (1 / rho), sigma_max ** (1 / rho)
        sigmas = (max_inv + ramp * (min_inv - max_inv)) ** rho
        timesteps = np.array([_sigma_to_t(s, log_sigmas) for s in sigmas], dtype=np.float64)
    sigmas = np.concatenate([sigmas, [0.0]])
    if heun:
        sigmas = np.concatenate([sigmas[:1], np.repeat(sigmas[1:-1], 2), sigmas[-1:]])
        timesteps = np.concatenate([timesteps[:1], np.repeat(timesteps[1:], 2)])
    return timesteps, sigmas


def init_noise_sigma(sigmas):
    """timestep_spacing "linspace": the largest sigma (not sqrt(sigma^2 + 1))."""
    return float(np.max(sigmas))


def scale_model_input(x, sigma):
    return x / ((sigma ** 2 + 1) ** 0.5)


def add_noise(original, noise, sigma):
    return original + noise * sigma


# ---- step -------------------------------------------------------------------------------------------------------------
class Scheduler:
    """The step of one of the three schedulers over its sigmas, from step index `begin` (set_begin_index).  denoise: optional
    map applied to pred_original_sample (the Kandinsky 2.1 inpainting rule)."""

    def __init__(self, kind, sigmas, begin=0):
        self.kind, self.sigmas, self.step_index = kind, sigmas, begin
        self.dt = None

    def sigma_in(self):
        return self.sigmas[self.step_index]

    def step(self, eps, sample, noise=None, denoise=None):
        s, j = self.sigmas, self.step_index
        first = self.dt is None
        if self.kind != "heun" or first:
            sigma, sigma_next = s[j], s[j + 1]
        else:
            sigma, sigma_next = s[j - 1], s[j]
        sigma_hat = sigma                                       # gamma = 0 (s_churn = 0)
        sigma_input = sigma_hat if (self.kind != "heun" or first) else sigma_next
        pred = sample - sigma_input * eps
        if denoise is not None:
            pred = denoise(pred)
        if self.kind == "euler":
            derivative = (sample - pred) / sigma_hat
            prev = sample + derivative * (sigma_next - sigma_hat)
        elif self.kind == "euler_ancestral":
            sigma_up = (sigma_next ** 2 * (sigma ** 2 - sigma_next ** 2) / sigma ** 2) ** 0.5
            sigma_down = (sigma_next ** 2 - sigma_up ** 2) ** 0.5
            derivative = (sample - pred) / sigma
            prev = sample + derivative * (sigma_down - sigma) + noise * sigma_up
        elif first:                                             # Heun, first order (the predictor, or the last step)
            derivative = (sample - pred) / sigma_hat
            self.prev_derivative, self.dt, self.sample = derivative, sigma_next - sigma_hat, sample
            prev = sample + derivative * self.dt
        else:                                                   # Heun, second order
            derivative = ((sample - pred) / sigma_next + self.prev_derivative) / 2
            prev = self.sample + derivative * self.dt
            self.prev_derivative = self.dt = self.sample = None
        self.step_index += 1
        return prev


def sample(kind, eps, ac, n, noise, karras=False, t_start=0, latent=None, step_noise=None, inpaint=None, inpaint_renoise=True):
    """The pipeline loop -> the final latent (x_ve at sigma = 0).  eps(x_in, t): the CFG epsilon at the UNet input x_in and
    timestep t.  Text2img (latent None): x = init_noise_sigma * noise.  img2img: the timesteps from index t_start * order
    (get_timesteps; order 2 for Heun), x = add_noise(latent, noise) at the first of them.  step_noise[i]: Euler ancestral's
    draw at evaluation i.  inpaint = (init, mask): inpaint_renoise=True is the KandinskyV22InpaintPipeline blend after every
    step, mask (init + sigma_next z) + (1 - mask) x with z = noise the unit start noise, the clean init after the last step;
    False the Kandinsky 2.1 rule, the known region replacing pred_original_sample."""
    heun = kind == "heun"
    timesteps, sigmas = set_timesteps(ac, n, karras=karras, heun=heun)
    begin = t_start * (2 if heun else 1)
    sch = Scheduler(kind, sigmas, begin)
    x = init_noise_sigma(sigmas) * noise if latent is None else add_noise(latent, noise, sigmas[begin])
    denoise = None
    if inpaint is not None and not inpaint_renoise:
        init, mask = inpaint
        denoise = lambda pred: pred * (1 - mask) + init * mask
    run = timesteps[begin:]
    for i, t in enumerate(run):
        e = eps(scale_model_input(x, sch.sigma_in()), t)
        x = sch.step(e, x, noise=None if step_noise is None else step_noise[i], denoise=denoise)
        if inpaint is not None and inpaint_renoise:
            init, mask = inpaint
            known = add_noise(init, noise, sch.sigmas[sch.step_index]) if i < len(run) - 1 else init
            x = mask * known + (1 - mask) * x
    return x


# ---- the kernels' formulas --------------------------------------------------------------------------------------------
def apply_rows(rows, ts, kind, eps, x, step_noise=None, inpaint=None, inpaint_renoise=True):
    """float64 run of a schedule's rows (table order, [n, 8]) with the formula of k2_dpm_solver(_sde)_step (kind "dpm") or
    k2_heun_step (kind "heun"), from the latent x in the UNet's input scale; eps(x, ts[j]) the CFG epsilon.  The 2.2 blend's
    inpaint_noise is the start latent, as _sampling_loop hands it to the kernels."""
    x = np.array(x, dtype=np.float64)
    rnoise = x.copy()
    xs = ds = None
    init, mask = inpaint if inpaint is not None else (None, None)
    blend_d = inpaint is not None and not inpaint_renoise
    for i, j in enumerate(range(len(rows))[::-1]):
        r = rows[j]
        e = eps(x, ts[j])
        if kind == "dpm":
            d0 = r[0] * x - r[1] * e
            if blend_d:
                d0 = d0 * (1 - mask) + init * mask
            xn = r[2] * x + r[3] * d0
            assert r[4] == 0.0
            if r[7] != 0.0:
                xn = xn + r[7] * step_noise[i]
        else:
            d = e
            if blend_d:
                d = d + r[2] * mask * ((r[0] * x - r[1] * e) - init)
            if r[7] == 0.0:
                xs, ds = x, d
                xn = r[3] * x + r[4] * d
            else:
                xn = r[3] * xs + r[4] * (ds + d)
        if inpaint is not None and inpaint_renoise:
            xn = mask * (r[5] * init + r[6] * rnoise) + (1 - mask) * xn
        x = xn
    return x
