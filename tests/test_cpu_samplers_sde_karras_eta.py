"""CPU: the host side of the DPM-Solver++(2M) SDE variant, Karras sigma spacing and DDIM with eta > 0 -- coefficient rows
against the float64 restatements (tests/dpm_sde_oracle.py, tests/ddim_eta_oracle.py), weak convergence of the SDE on Gaussian
data, the Karras grid's known answers, the DDIM eta oracle against the reference's own sampler (tests/golden/ddim_eta_tiny.pt),
and the refusals of bad eta.  The argument checks of k2_dpm_solver_sde_step and the pipelines' sampler names are in
tests/test_cpu_schedule_samplers.py."""
import os

import numpy as np
import pytest
import torch

from tests import ddim_eta_oracle as eo
from tests import dpm_oracle as do
from tests import dpm_sde_oracle as so

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
MU, S = 0.3, 0.5   # Gaussian data x0 ~ N(MU, S^2)


def _bases():
    from kandinsky2.configs import CONFIG_2_1
    from kandinsky2.model.gaussian_diffusion import create_ddpm_v22, create_gaussian_diffusion
    return {"2.1": create_gaussian_diffusion(**CONFIG_2_1["diffusion_config"]).base_alphas_cumprod,
            "2.2": create_ddpm_v22(50).base_alphas_cumprod}


# ---- DPM-Solver++(2M) SDE rows -------------------------------------------------------------------------------------------
@pytest.mark.parametrize("spacing", ["linspace", "karras"])
@pytest.mark.parametrize("n", [10, 20, 40])
@pytest.mark.parametrize("keep", [None, 7])
def test_sde_rows_with_kernel_formula_reproduce_solve_sde(spacing, n, keep):
    """The product's float64 SDE rows applied with the kernel's formula == the paper-form SDE loop with the same injected
    noise, to 1e-12, on an epsilon that depends on x non-linearly; the rows equal the oracle's rows on the same grid."""
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule
    sch = DPMSolverSchedule(_bases()["2.2"], n, keep=keep, spacing=spacing, sde=True)
    a, s, k0 = sch.alphas, sch.sigmas, sch.k0
    rng = np.random.default_rng(n)
    x = rng.standard_normal(256)
    z = rng.standard_normal((n - k0, 256))

    def eps(x, k):
        return do.gaussian_eps(x, a[k], s[k], MU, S) + 0.1 * np.tanh(x)

    rows = sch.coef_rows()[::-1]                         # step order k = k0 .. n-1
    np.testing.assert_allclose(rows, so.sde_rows(a, s, first=k0), rtol=1e-13, atol=1e-300)
    got = so.apply_rows_sde(rows, eps, x, z, step_index=list(range(k0, n)))
    ref = so.solve_sde(eps, x, a, s, z, first=k0)
    assert np.abs(got - ref).max() < 1e-12 * max(1.0, np.abs(ref).max())


@pytest.mark.parametrize("spacing", ["linspace", "karras"])
def test_sde_schedule_structure(spacing):
    """SDE rows: the first (and first-after-truncation) row is first order with noise, interior rows are second order with
    noise, the last row lands on D with no noise; the schedule draws noise and names the SDE step; the ODE schedule's
    column 7 stays 0."""
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule
    ac = _bases()["2.1"]
    for keep in (None, 5, 1):
        sch = DPMSolverSchedule(ac, 12, keep=keep, spacing=spacing, sde=True)
        tab = sch.coef_table()[::-1]
        assert sch.draws_noise and sch.step_kind == "dpmpp_2m_sde"
        assert tuple(tab[-1, 2:5]) == (0.0, 1.0, 0.0) and tab[-1, 7] == 0.0 and tuple(tab[-1, 5:7]) == (1.0, 0.0)
        if len(tab) > 1:
            assert tab[0, 4] == 0.0 and tab[0, 7] > 0.0
            assert (tab[1:-1, 4] != 0.0).all() and (tab[:-1, 7] > 0.0).all()
        ode = DPMSolverSchedule(ac, 12, keep=keep, spacing=spacing)
        assert not ode.draws_noise and ode.step_kind == "dpmpp_2m" and (ode.coef_table()[:, 7] == 0.0).all()
        assert np.array_equal(ode.model_timesteps(), sch.model_timesteps())


def test_schedule_rejects_unknown_spacing():
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule
    with pytest.raises(ValueError):
        DPMSolverSchedule(_bases()["2.2"], 10, spacing="exponential")


def _variance_errors(ns, kind, order):
    errs = []
    for n in ns:
        a, s = do.smooth_grid(n)
        rows = so.sde_rows(a, s, order=order) if kind == "sde" else do.rows(a, s, order=order)
        mean, var = so.gaussian_moments(rows, a, s, MU, S)
        assert abs(mean - a[-1] * MU) < 1e-12              # the mean is exact for every linear solver of this family
        errs.append(abs(var - (a[-1] ** 2 * S ** 2 + s[-1] ** 2)))
    return [errs[i] / errs[i + 1] for i in range(len(errs) - 1)]


def test_sde_weak_convergence_second_order():
    """Gaussian data on the interior grid t = 999 -> 200, the output's mean and variance propagated exactly: the variance
    error of the 2M SDE falls >= 3.3x per doubling from 10 to 80 steps, ~2x with c_P forced to 0 (so the second-order term
    is what buys the order); the same propagation of the ODE rows gives ~4x and ~2x."""
    ns = [10, 20, 40, 80]
    r2, r1 = _variance_errors(ns, "sde", 2), _variance_errors(ns, "sde", 1)
    o2, o1 = _variance_errors(ns, "ode", 2), _variance_errors(ns, "ode", 1)
    assert all(r >= 3.3 for r in r2), r2
    assert all(1.8 <= r <= 2.1 for r in r1), r1
    assert all(3.5 <= r <= 4.5 for r in o2), o2
    assert all(1.8 <= r <= 2.1 for r in o1), o1


# ---- Karras spacing ------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("version", ["2.1", "2.2"])
def test_karras_known_answers(version):
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule, karras_timesteps
    ac = _bases()[version]
    t, s_hat = karras_timesteps(ac, 20)
    assert abs(s_hat[0] - 25.146115) < 1e-6 and abs(s_hat[-1] - 0.029167) < 1e-6
    assert t[0] == 999.0 and t[-1] == 0.0 and (np.diff(t) < 0).all() and (np.diff(s_hat) < 0).all()
    np.testing.assert_allclose(t[:4], [999.0, 959.957, 918.006, 872.698], atol=1e-3, rtol=0)
    np.testing.assert_allclose(t[-4:], [20.424, 7.682, 2.127, 0.0], atol=1e-3, rtol=0)
    sch = DPMSolverSchedule(ac, 20, spacing="karras")
    assert np.array_equal(sch.timesteps, t)
    assert np.array_equal(sch.model_timesteps(), t[::-1].astype(np.float32))
    np.testing.assert_allclose(sch.sigmas[:-1] / sch.alphas[:-1], s_hat, rtol=1e-14)
    np.testing.assert_allclose(sch.alphas[:-1] ** 2 + sch.sigmas[:-1] ** 2, 1.0, rtol=1e-14)
    assert (sch.alphas[-1], sch.sigmas[-1]) == (1.0, 0.0)
    # the ODE rows on the Karras grid are the paper's rows on that grid
    np.testing.assert_allclose(sch.coef_rows()[::-1], do.rows(sch.alphas, sch.sigmas), rtol=1e-13, atol=0)
    one = DPMSolverSchedule(ac, 1, spacing="karras")
    assert np.array_equal(one.timesteps, [999.0]) and one.sigmas[0] / one.alphas[0] == s_hat[0]
    for n in (2, 3, 7, 50, 200):
        tn, _ = karras_timesteps(ac, n)
        assert tn[0] == 999.0 and tn[-1] == 0.0 and (np.diff(tn) < 0).all()
    img = DPMSolverSchedule(ac, 20, keep=6, spacing="karras")
    assert img.num_timesteps == 6 and np.array_equal(img.model_timesteps(), t[14:][::-1].astype(np.float32))
    assert (img.start_latent(1.0, 0.0), img.start_latent(0.0, 1.0)) == (img.alphas[14], img.sigmas[14])


def test_karras_ode_approaches_the_flow_endpoint():
    """On Gaussian data the Karras ODE run toward sigma = 0 gets closer to the closed-form flow each time N doubles."""
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule
    ac = _bases()["2.2"]
    x = np.random.default_rng(2).standard_normal(512)
    errs = []
    for n in (10, 20, 40):
        sch = DPMSolverSchedule(ac, n, spacing="karras")
        eps = lambda x, k: do.gaussian_eps(x, sch.alphas[k], sch.sigmas[k], MU, S)
        out = do.apply_rows(sch.coef_rows()[::-1], eps, x)
        errs.append(np.abs(out - do.gaussian_flow(x, sch.alphas[0], sch.sigmas[0], 1.0, 0.0, MU, S)).max())
    assert errs[1] < errs[0] and errs[2] < errs[1], errs


# ---- DDIM with eta > 0 ---------------------------------------------------------------------------------------------------
def _ddim(eta, steps, init_step=None):
    from kandinsky2.configs import CONFIG_2_1
    from kandinsky2.model.gaussian_diffusion import DDIMSampler, create_gaussian_diffusion
    s = DDIMSampler(None, create_gaussian_diffusion(**CONFIG_2_1["diffusion_config"]))
    s.make_schedule(steps, ddim_eta=eta, init_step=init_step)
    return s


@pytest.mark.parametrize("steps", [4, 10, 50, 100])
def test_ddim_eta0_table_unchanged(steps):
    """At eta = 0 the rows are the eta-free formula's, bit for bit, with columns 4-7 zero and no noise drawn."""
    for init in (None, 500):
        s = _ddim(0.0, steps, init)
        a_t, a_p = s.ddim_alphas, s.ddim_alphas_prev
        s1 = np.sqrt(1.0 - a_t)
        ref = np.zeros((s.num_timesteps, 8))
        ref[:, 0], ref[:, 1] = 1.0 / np.sqrt(a_t), s1 / np.sqrt(a_t)
        ref[:, 2] = np.sqrt(a_p) - np.sqrt(1.0 - a_p) * np.sqrt(a_t) / s1
        ref[:, 3] = np.sqrt(1.0 - a_p) / s1
        tab = s.coef_table()
        assert tab.dtype == np.float32 and tab.tobytes() == ref.astype(np.float32).tobytes()
        assert not s.draws_noise


def test_ddim_eta_rows_apply_the_reference_step():
    """eta = 0.5: the rows applied with k2_sampler_step's formula (x0 = c0 x - c1 e; x' = c2 x0 + c3 x + c6 exp(logvar / 2) z
    with logvar = log sigma^2 whatever the variance channel) == p_sample_ddim (float64), and sigma == the reference's."""
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "ddim_eta_tiny.pt"), weights_only=False)
    s = _ddim(fx["eta"], fx["steps"])
    np.testing.assert_allclose(s.ddim_sigmas, fx["sigmas"], rtol=1e-12, atol=0)
    assert s.draws_noise
    s = _ddim(0.5, 50)
    tt, al, alp, sig = eo.ddim_eta_schedule(50, 0.5)
    assert np.array_equal(s.ddim_timesteps, tt) and (sig > 0).all()
    tab = s.coef_table().astype(np.float64)
    rng = np.random.default_rng(5)
    x, e, z, v = (rng.standard_normal(64) for _ in range(4))
    for i in range(len(tt)):
        c = tab[i]
        x0 = c[0] * x - c[1] * e
        frac = (v + 1) / 2
        got = c[2] * x0 + c[3] * x + c[6] * np.exp(0.5 * (frac * c[5] + (1 - frac) * c[4])) * z
        ref = eo.ddim_eta_step(x, e, al[i], alp[i], sig[i], z)
        np.testing.assert_allclose(got, ref, rtol=2e-5, atol=2e-5)
        assert c[6] == 1.0 and c[4] == c[5] and c[7] == 0.0


def test_ddim_eta_oracle_matches_reference_golden():
    """The eta restatement vs the output of the reference's own DDIMSampler.sample(eta=0.5) with the captured noise."""
    from oracle import synth, unet_oracle as uo
    fx = torch.load(os.path.join(ROOT, "tests", "golden", "ddim_eta_tiny.pt"), weights_only=False)
    cfg = fx["cfg"]
    sd = synth.synth_state_dict(uo.unet_param_spec(cfg), seed=fx["weight_seed"])
    with torch.no_grad():
        out = eo.ddim_eta_sample_loop(lambda xx, tt: uo.unet_forward(sd, cfg, xx, tt, **fx["cond"]), fx["x_T"], fx["steps"],
                                      fx["guidance"], fx["eta"], fx["step_noise"])
    assert (out - fx["out"]).abs().max().item() <= 1e-4


def test_ddim_eta_oracle_at_eta0_is_the_eta0_oracle():
    from oracle import diffusion_oracle as dfo
    g = torch.Generator().manual_seed(0)
    x_T = torch.randn(2, 4, 4, 4, generator=g)
    w = torch.randn(8, 4, generator=g)

    def unet(x, t):
        return torch.einsum("oc,bchw->bohw", w, torch.tanh(x)) * (1 + t[:, None, None, None] / 1000)

    a = dfo.ddim_sample_loop(unet, x_T, 5, 3.0)
    b = eo.ddim_eta_sample_loop(unet, x_T, 5, 3.0, 0.0, torch.randn(5, 2, 4, 4, 4, generator=g))
    assert torch.equal(a, b)


def test_eta_refusals():
    """PLMS refuses eta != 0, as the reference; DDIM refuses a negative eta and one whose sigma^2 exceeds 1 - a_prev."""
    from kandinsky2.model.gaussian_diffusion import PLMSSampler
    p = PLMSSampler(None, _ddim(0.0, 4).old_diffusion)
    with pytest.raises(NotImplementedError):
        p.make_schedule(10, ddim_eta=0.5)
    p.make_schedule(10, ddim_eta=0.0)
    with pytest.raises(ValueError):
        _ddim(-0.1, 10)
    with pytest.raises(ValueError):
        _ddim(5.0, 10)
    assert _ddim(1.0, 10).draws_noise
