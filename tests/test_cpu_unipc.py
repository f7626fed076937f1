"""CPU: the UniPC sampler's host side -- unipc_rows / UniPCSchedule against the float64 restatement of the paper and of diffusers'
step order (tests/unipc_oracle.py), UniP-2 bh2 without the corrector against DPMSolverSchedule, third-order convergence with
the corrector on Gaussian data whose probability-flow ODE has a closed form, both inpainting rules and the refusals of bad
schedule arguments.  The argument checks of k2_unipc_step and the pipelines' sampler names are in
tests/test_cpu_schedule_samplers.py."""
import numpy as np
import pytest

from tests import dpm_oracle as do
from tests import unipc_oracle as uo

MU, S = 0.7, 0.5   # Gaussian data x0 ~ N(MU, S^2)


def _ac(version="2.2"):
    from kandinsky2.configs import CONFIG_2_1
    from kandinsky2.model.gaussian_diffusion import create_ddpm_v22, create_gaussian_diffusion
    if version == "2.1":
        return create_gaussian_diffusion(**CONFIG_2_1["diffusion_config"]).base_alphas_cumprod
    return create_ddpm_v22(50).base_alphas_cumprod


def _eps_nonlinear(sch):
    """An epsilon that depends on x non-linearly, so a wrong coefficient cannot hide behind a linear model."""
    return lambda x, k: do.gaussian_eps(x, sch.alphas[k], sch.sigmas[k], MU, S) + 0.1 * np.tanh(x)


def _keeps(n):
    return sorted({n, max(n // 2, 1), 1})


@pytest.mark.parametrize("spacing", ["linspace", "karras"])
@pytest.mark.parametrize("n", [1, 2, 5, 10, 20, 40])
def test_rows_with_kernel_formula_reproduce_oracle_loop(n, spacing):
    """UniPCSchedule's float64 rows applied with the kernel's formula == the oracle's paper-form loop (R rho = b solved per step,
    order ramp, first-order last step), to 1e-12, for every run length, both spacings and with and without img2img truncation;
    the fp32 table is the float64 rows cast once, and the grid is DPMSolverSchedule's."""
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule, UniPCSchedule
    ac = _ac()
    x = np.random.default_rng(n).standard_normal(256)
    for keep in _keeps(n):
        sch = UniPCSchedule(ac, n, keep=keep, spacing=spacing)
        dpm = DPMSolverSchedule(ac, n, keep=keep, spacing=spacing)
        assert sch.num_timesteps == keep and sch.k0 == n - keep and sch.step_kind == "unipc" and not sch.draws_noise
        assert np.array_equal(sch.timesteps, dpm.timesteps) and np.array_equal(sch.model_timesteps(), dpm.model_timesteps())
        assert np.array_equal(sch.alphas, dpm.alphas) and np.array_equal(sch.sigmas, dpm.sigmas)
        rows = sch.coef_rows()
        tab = sch.coef_table()
        assert rows.shape == (keep, 16) and tab.dtype == np.float32 and np.array_equal(tab, rows.astype(np.float32))
        eps = _eps_nonlinear(sch)
        steps = list(range(sch.k0, n))
        got = uo.apply_rows(rows[::-1], eps, x, step_index=steps)
        ref = uo.solve(eps, x, sch.alphas, sch.sigmas, first=sch.k0)
        assert np.abs(got - ref).max() < 1e-12 * max(1.0, np.abs(ref).max()), (keep, np.abs(got - ref).max())
        a0, s0 = sch.start_latent(1.0, 0.0), sch.start_latent(0.0, 1.0)
        assert (a0, s0) == (dpm.start_latent(1.0, 0.0), dpm.start_latent(0.0, 1.0))


@pytest.mark.parametrize("keep", [None, 7])
def test_rows_structure(keep):
    """Step order: the first step has no corrector (a_x = 1, a_L..a_2 = 0) and a first-order predictor (b_1 = 0); the second has
    a first-order corrector (a_2 = 0); later ones read D_{k-2}; the last row lands on D_{N-1}: (b_c, b_0, b_1) = (0, 1, 0) and
    (alpha, sigma)_N = (1, 0); columns 12-15 are 0."""
    from kandinsky2.model.gaussian_diffusion import UniPCSchedule
    rows = UniPCSchedule(_ac(), 20, keep=keep).coef_table()[::-1]
    assert tuple(rows[0, 2:7]) == (1.0, 0.0, 0.0, 0.0, 0.0) and rows[0, 9] == 0.0
    assert rows[1, 2] == 0.0 and rows[1, 3] != 0.0 and rows[1, 5] != 0.0 and rows[1, 6] == 0.0 and rows[1, 9] != 0.0
    assert (rows[2:, 6] != 0.0).all() and (rows[1:-1, 9] != 0.0).all()
    assert tuple(rows[-1, 7:12]) == (0.0, 1.0, 0.0, 1.0, 0.0)
    assert not rows[:, 12:].any()


@pytest.mark.parametrize("spacing", ["linspace", "karras"])
@pytest.mark.parametrize("n", [1, 2, 5, 10, 20, 40])
def test_without_corrector_is_dpm_solver(n, spacing):
    """UniP-2 with bh2 is DPM-Solver++(2M): with the corrector columns forced to "no corrector" (a_x = 1, a_L..a_2 = 0) the rows
    give DPMSolverSchedule's iterates to 1e-12, and the predictor columns equal DPM's (c_x, c_D, c_P) to 1e-13 relative."""
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule, UniPCSchedule
    ac = _ac("2.1")
    x = np.random.default_rng(2 * n).standard_normal(256)
    for keep in _keeps(n):
        sch = UniPCSchedule(ac, n, keep=keep, spacing=spacing)
        dpm = DPMSolverSchedule(ac, n, keep=keep, spacing=spacing)
        rows = sch.coef_rows()[::-1].copy()
        rows[:, 2], rows[:, 3:7] = 1.0, 0.0
        eps = _eps_nonlinear(sch)
        steps = list(range(sch.k0, n))
        got = uo.apply_rows(rows, eps, x, step_index=steps)
        ref = do.apply_rows(dpm.coef_rows()[::-1], eps, x, step_index=steps)
        assert np.abs(got - ref).max() < 1e-12 * max(1.0, np.abs(ref).max()), (keep, np.abs(got - ref).max())
        np.testing.assert_allclose(rows[:, 7:10], dpm.coef_rows()[::-1][:, 2:5], rtol=1e-13, atol=0)
        assert np.abs(uo.solve(eps, x, sch.alphas, sch.sigmas, first=sch.k0, corrector=False) - ref).max() < 1e-12 * max(
            1.0, np.abs(ref).max())


def _converge(order, corrector, ns=(10, 20, 40, 80)):
    """Max-abs error against the closed-form flow from t = 999 to t = 200 on the 2.2 base table with integer linspace
    timesteps, through unipc_rows.  The predictor's last step is NOT lowered here: on an interior grid a first-order last step
    would set the global order (on the sampler's grid it lands on sigma = 0, where it is exact for D)."""
    from kandinsky2.model.gaussian_diffusion import unipc_rows
    ac = _ac()
    errs = []
    for n in ns:
        t = np.linspace(999, 200, n + 1).round().astype(np.int64)
        a, s = np.sqrt(ac[t]), np.sqrt(1.0 - ac[t])
        xt = np.linspace(-3, 3, 7) * np.sqrt(a[0] ** 2 * S ** 2 + s[0] ** 2) + a[0] * MU
        eps = lambda x, k: do.gaussian_eps(x, a[k], s[k], MU, S)
        out = uo.apply_rows(unipc_rows(a, s, order=order, corrector=corrector, lower_order_final=False), eps, xt)
        ref = uo.solve(eps, xt, a, s, order=order, corrector=corrector, lower_order_final=False)
        assert np.abs(out - ref).max() < 1e-12
        errs.append(np.abs(out - do.gaussian_flow(xt, a[0], s[0], a[-1], s[-1], MU, S)).max())
    return errs, [errs[i] / errs[i + 1] for i in range(len(errs) - 1)]


def test_gaussian_convergence_third_order_with_corrector():
    """N = 10 -> 80: the error falls > 7.5x per doubling with UniC (third order), 3.8-4.3x without it (UniP-2 = DPM++(2M)) and
    about 2x at order 1 -- 4.14e-3 / 4.97e-4 / 5.52e-5 / 6.19e-6 against 1.16e-2 / 2.86e-3 / 6.99e-4 / 1.72e-4."""
    e_pc, r_pc = _converge(2, True)
    e_p, r_p = _converge(2, False)
    e_1, r_1 = _converge(1, False)
    assert all(r > 7.5 for r in r_pc), (e_pc, r_pc)
    assert all(3.8 <= r <= 4.3 for r in r_p), (e_p, r_p)
    assert all(1.9 <= r <= 2.1 for r in r_1), (e_1, r_1)
    assert e_pc[0] < e_p[0] / 2.5 and e_pc[1] < e_p[1] / 5


def test_sampler_schedule_approaches_the_flow_endpoint():
    """The product's schedule ends at sigma = 0 with x_N = D_{N-1}: on Gaussian data doubling the steps from 10 to 20 brings the
    result closer to the closed-form flow to sigma = 0, and at 10 steps it is closer than DPM-Solver++(2M)."""
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule, UniPCSchedule
    ac = _ac()
    x = np.random.default_rng(2).standard_normal(512)
    errs = {}
    for cls in (UniPCSchedule, DPMSolverSchedule):
        for n in (10, 20):
            sch = cls(ac, n)
            eps = lambda x, k: do.gaussian_eps(x, sch.alphas[k], sch.sigmas[k], MU, S)
            app = uo.apply_rows if cls is UniPCSchedule else do.apply_rows
            out = app(sch.coef_rows()[::-1], eps, x)
            errs[cls.__name__, n] = np.abs(out - do.gaussian_flow(x, sch.alphas[0], sch.sigmas[0], 1.0, 0.0, MU, S)).max()
    assert errs["UniPCSchedule", 20] < errs["UniPCSchedule", 10] / 1.5, errs
    assert errs["UniPCSchedule", 10] < errs["DPMSolverSchedule", 10], errs


def test_inpainting_rules_in_rows_match_oracle():
    """Both inpainting rules through the rows (2.1: the known region replaces D; 2.2: the known region of x is re-noised to the
    next grid point, `last` not blended) == the oracle loop to 1e-12; the 2.2 result's known region is the clean latent."""
    from kandinsky2.model.gaussian_diffusion import UniPCSchedule
    sch = UniPCSchedule(_ac(), 12, keep=9)
    rng = np.random.default_rng(5)
    x, init, noise0 = rng.standard_normal((3, 128))
    mask = (rng.random(128) > 0.5).astype(np.float64)
    eps = _eps_nonlinear(sch)
    steps = list(range(sch.k0, 12))
    for renoise in (False, True):
        inp = (init, mask, noise0)
        got = uo.apply_rows(sch.coef_rows()[::-1], eps, x, step_index=steps, inpaint=inp, inpaint_renoise=renoise)
        ref = uo.solve(eps, x, sch.alphas, sch.sigmas, first=sch.k0, inpaint=inp, inpaint_renoise=renoise)
        assert np.abs(got - ref).max() < 1e-12 * max(1.0, np.abs(ref).max()), renoise
        if renoise:
            assert np.array_equal(got[mask == 1], init[mask == 1])


def test_schedule_rejects_bad_arguments():
    from kandinsky2.model.gaussian_diffusion import UniPCSchedule, unipc_rows
    ac = _ac()
    for n, keep, spacing in ((0, None, "linspace"), (10, 0, "linspace"), (10, 11, "linspace"), (1000, None, "linspace"),
                             (10, None, "exponential")):
        with pytest.raises(ValueError):
            UniPCSchedule(ac, n, keep=keep, spacing=spacing)
    assert UniPCSchedule(ac, 999).num_timesteps == 999
    sch = UniPCSchedule(ac, 5)
    with pytest.raises(ValueError):
        unipc_rows(sch.alphas, sch.sigmas, order=3)
    with pytest.raises(ValueError):            # a second-order step to sigma = 0 is undefined (r = 0)
        unipc_rows(sch.alphas, sch.sigmas, lower_order_final=False)
