"""CPU: the DPM-Solver++(2M) sampler's host side -- DPMSolverSchedule's timestep grid and coefficient rows against the float64
restatement of the paper (tests/dpm_oracle.py), second-order convergence on Gaussian data whose probability-flow ODE has a
closed form.  The argument checks of k2_dpm_solver_step and the pipelines' sampler names are in
tests/test_cpu_schedule_samplers.py."""
import numpy as np
import pytest

from tests import dpm_oracle as do

MU, S = 0.3, 0.5   # Gaussian data x0 ~ N(MU, S^2)


def _bases():
    from kandinsky2.configs import CONFIG_2_1
    from kandinsky2.model.gaussian_diffusion import create_ddpm_v22, create_gaussian_diffusion
    return {"2.1": create_gaussian_diffusion(**CONFIG_2_1["diffusion_config"]).base_alphas_cumprod,
            "2.2": create_ddpm_v22(50).base_alphas_cumprod}


@pytest.mark.parametrize("version", ["2.1", "2.2"])
@pytest.mark.parametrize("n", [1, 2, 3, 10, 20, 50])
def test_schedule_matches_oracle(version, n):
    """tau grid, model timesteps and fp32 rows of every run length and truncation against the oracle's rows; the last row is
    exactly (c_x, c_D, c_P) = (0, 1, 0) and every first-order row has c_P = 0."""
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule
    ac = _bases()[version]
    tau, alpha, sigma = do.grid(ac, n)
    for keep in sorted({n, max(n // 2, 1), 1}):
        sch = DPMSolverSchedule(ac, n, keep=keep)
        k0 = n - keep
        assert sch.num_timesteps == keep
        assert np.array_equal(sch.timesteps, tau)
        assert np.array_equal(sch.model_timesteps(), tau[k0:][::-1].astype(np.float32))
        tab = sch.coef_table()[::-1]          # step order k = k0 .. n-1
        ref = do.rows(alpha, sigma, first=k0)
        assert tab.dtype == np.float32 and tab.shape == (keep, 8)
        np.testing.assert_allclose(sch.coef_rows()[::-1], ref, rtol=1e-13, atol=0)
        np.testing.assert_allclose(tab, ref.astype(np.float32), rtol=2.4e-7, atol=0)
        assert tuple(tab[-1, 2:5]) == (0.0, 1.0, 0.0) and tuple(tab[-1, 5:7]) == (1.0, 0.0)
        assert tab[0, 4] == 0.0                # first step after the truncation point
        if keep >= 3:
            assert (tab[1:-1, 4] != 0.0).all()   # every interior step is second order
        a0, s0 = sch.start_latent(1.0, 0.0), sch.start_latent(0.0, 1.0)
        assert (a0, s0) == (alpha[k0], sigma[k0])


def test_schedule_rejects_bad_arguments():
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule
    ac = _bases()["2.2"]
    for n, keep in ((0, None), (10, 0), (10, 11), (1000, None)):
        with pytest.raises(ValueError):
            DPMSolverSchedule(ac, n, keep=keep)
    assert DPMSolverSchedule(ac, 999).num_timesteps == 999


@pytest.mark.parametrize("keep", [None, 7])
def test_rows_with_kernel_formula_reproduce_oracle_loop(keep):
    """The product's float64 rows applied with the kernel's formula == Algorithm 2 in the paper's form, to 1e-12, on an
    epsilon that depends on x non-linearly (so a wrong row cannot hide behind a linear model)."""
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule
    ac = _bases()["2.2"]
    n = 20
    sch = DPMSolverSchedule(ac, n, keep=keep)
    _, alpha, sigma = do.grid(ac, n)
    x = np.random.default_rng(1).standard_normal(256)

    def eps(x, k):
        return do.gaussian_eps(x, alpha[k], sigma[k], MU, S) + 0.1 * np.tanh(x)

    got = do.apply_rows(sch.coef_rows()[::-1], eps, x, step_index=list(range(sch.k0, n)))
    ref = do.solve(eps, x, alpha, sigma, first=sch.k0)
    assert np.abs(got - ref).max() < 1e-12 * max(1.0, np.abs(ref).max())


def _converge(ns, order, t_end=200.0):
    x0 = np.random.default_rng(0).standard_normal(512)
    errs = []
    for n in ns:
        a, s = do.smooth_grid(n, t_end=t_end)
        xt = a[0] * MU + np.sqrt(a[0] ** 2 * S ** 2 + s[0] ** 2) * x0
        eps = lambda x, k: do.gaussian_eps(x, a[k], s[k], MU, S)
        out = do.apply_rows(do.rows(a, s, order=order), eps, xt)
        assert np.abs(out - do.solve(eps, xt, a, s, order=order)).max() < 1e-12
        errs.append(np.abs(out - do.gaussian_flow(xt, a[0], s[0], a[-1], s[-1], MU, S)).max())
    return errs


def test_analytic_convergence_second_order():
    """From t = 999 to the interior t = 200 with N, 2N, 4N steps: the error against the closed-form flow falls 3-5x per
    doubling; with c_P forced to 0 (first order) it falls ~2x, so the second-order term is what buys the extra order."""
    e2 = _converge([10, 20, 40], order=2)
    e1 = _converge([10, 20, 40], order=1)
    r2 = [e2[i] / e2[i + 1] for i in range(2)]
    r1 = [e1[i] / e1[i + 1] for i in range(2)]
    assert all(3.0 <= r <= 5.0 for r in r2), (e2, r2)
    assert all(1.8 <= r <= 2.2 for r in r1), (e1, r1)
    assert e2[-1] < e1[-1] / 10


def test_sampler_schedule_approaches_the_flow_endpoint():
    """The product's schedule ends at sigma = 0 with x_N = D_{N-1}, a first-order last step: on Gaussian data doubling the
    steps from 25 to 50 brings the result at least 1.5x closer to the closed-form flow to sigma = 0."""
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule
    ac = _bases()["2.2"]
    x = np.random.default_rng(2).standard_normal(512)
    errs = []
    for n in (25, 50):
        sch = DPMSolverSchedule(ac, n)
        eps = lambda x, k: do.gaussian_eps(x, sch.alphas[k], sch.sigmas[k], MU, S)
        out = do.apply_rows(sch.coef_rows()[::-1], eps, x)
        errs.append(np.abs(out - do.gaussian_flow(x, sch.alphas[0], sch.sigmas[0], 1.0, 0.0, MU, S)).max())
    assert errs[1] < errs[0] / 1.5, errs
