"""CPU: the Kandinsky 2.1 prior's sampling tables.  sample_prior reads the respaced posterior of the cosine schedule from
SpacedDiffusion, the decoder's class; these tests pin that those arrays, and the prior's one-section timestep subset from
space_timesteps, equal the prior's own formulas (PriorDiffusionModel: respace.py:83-97 and gaussian_diffusion.py:114-165 of
the reference, restated here in float64) bit for bit."""
import numpy as np
import pytest


def _one_section(num_timesteps, count):
    """respace.py:24-72 with one section (the prior's timestep_respacing=str(prior_steps))."""
    stride = 1 if count <= 1 else (num_timesteps - 1) / (count - 1)
    cur, out = 0.0, set()
    for _ in range(count):
        out.add(round(cur))
        cur += stride
    return out


def _prior_tables(base_betas, use_steps):
    """-> (posterior_mean_coef1, posterior_mean_coef2, posterior_log_variance_clipped) of the process respaced to use_steps."""
    acp_full = np.cumprod(1.0 - base_betas)
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
    return c1, c2, post_logvar


@pytest.mark.parametrize("n", [1, 2, 25, 1000])
def test_space_timesteps_one_section(n):
    from kandinsky2.model.gaussian_diffusion import space_timesteps
    got = space_timesteps(1000, [n])
    assert got == _one_section(1000, n) and len(got) == n
    assert space_timesteps(1000, str(n)) == got          # the reference passes timestep_respacing as a string


@pytest.mark.parametrize("n", [2, 25, 1000])
def test_spaced_diffusion_gives_the_prior_tables(n):
    """Also: the cosine schedule, capped at 0.999, keeps every respaced beta inside SpacedDiffusion's (0, 1]."""
    from kandinsky2.model.gaussian_diffusion import SpacedDiffusion, space_timesteps
    from kandinsky2.model.prior import cosine_betas
    use = sorted(space_timesteps(1000, [n]))
    d = SpacedDiffusion(set(use), cosine_betas(1000))
    assert d.timestep_map == use and d.betas.dtype == np.float64
    assert (d.betas > 0).all() and (d.betas <= 1).all()
    c1, c2, logvar = _prior_tables(cosine_betas(1000), use)
    for got, want in ((d.posterior_mean_coef1, c1), (d.posterior_mean_coef2, c2), (d.posterior_log_variance_clipped, logvar)):
        assert got.dtype == np.float64 and np.array_equal(got, want)
    assert np.isfinite(logvar).all() and np.isfinite(c1).all() and np.isfinite(c2).all()


def test_sample_prior_refuses_unsorted_steps():
    """The tables are those of the sorted subset, so a list in another order (or with a repeat) would pair them with the wrong
    model timesteps: refused before the model is called."""
    from kandinsky2.model.prior import sample_prior
    for bad in ([0, 999, 500], [0, 500, 500]):
        with pytest.raises(ValueError, match="strictly increasing"):
            sample_prior(None, None, None, None, bad, 4.0, None, None, None, None)
