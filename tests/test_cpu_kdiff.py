"""CPU: the sigma-space samplers' host side -- EulerSchedule / HeunSchedule rows, applied with the step kernels' formulas in
float64, against the float64 restatement of diffusers' Euler, Euler ancestral and Heun discrete schedulers and their pipeline
loop (tests/kdiff_oracle.py); the grids, the start latents, Heun's evaluation count and the refusals of bad schedule
arguments.  The argument checks of k2_heun_step and the pipelines' sampler names are in tests/test_cpu_schedule_samplers.py."""
import numpy as np
import pytest

from tests import kdiff_oracle as ko
from tests.sampler_cases import KINDS, _schedule


def _ac(version="2.2"):
    from kandinsky2.configs import CONFIG_2_1
    from kandinsky2.model.gaussian_diffusion import create_ddpm_v22, create_gaussian_diffusion
    if version == "2.1":
        return create_gaussian_diffusion(**CONFIG_2_1["diffusion_config"]).base_alphas_cumprod
    return create_ddpm_v22(50).base_alphas_cumprod


def _eps(x, t):
    """An epsilon that depends on x non-linearly and on the timestep (seen through its fp32 cast, as the UNet sees it)."""
    tt = float(np.float32(t)) / 1000.0
    return 0.4 * np.tanh(1.3 * x) + 0.2 * x * tt + 0.05 * np.cos(7.0 * tt)


def _keeps(n):
    return sorted({n, max(n // 2, 1), 1})


@pytest.mark.parametrize("version", ["2.1", "2.2"])
@pytest.mark.parametrize("n", [2, 10, 25])
@pytest.mark.parametrize("name", list(KINDS))
def test_rows_with_kernel_formula_reproduce_oracle_loop(name, n, version):
    """The float64 rows applied with the kernels' formula == diffusers' scheduler loop restated in float64, to 1e-12, for both
    base tables, with and without img2img truncation; the fp32 table is the rows cast once and the model timesteps are the
    scheduler's (fp32)."""
    kind, karras, formula = KINDS[name]
    ac = _ac(version)
    rng = np.random.default_rng(n)
    z = rng.standard_normal(256)
    latent = rng.standard_normal(256)
    for keep in _keeps(n):
        sch = _schedule(name, ac, n, keep)
        rows = sch.coef_rows()
        evals = 2 * keep - 1 if kind == "heun" else keep
        assert rows.shape == (evals, 8) and sch.num_timesteps == evals
        assert np.array_equal(sch.coef_table(), rows.astype(np.float32))
        ts = sch.model_timesteps()
        assert ts.dtype == np.float32 and ts.shape == (evals,)
        t_ref, _ = ko.set_timesteps(ac, n, karras=karras, heun=kind == "heun")
        t_start = n - keep
        # (diffusers' _sigma_to_t puts the last Karras timestep at ~1e-15 where np.interp gives 0)
        assert np.allclose(ts[::-1], t_ref[t_start * (2 if kind == "heun" else 1):], rtol=1e-7, atol=1e-9)
        step_noise = rng.standard_normal((evals, 256)) if kind == "euler_ancestral" else None
        if keep == n:
            x = sch.init_noise_scale * z
            ref = ko.sample(kind, _eps, ac, n, z, karras=karras, step_noise=step_noise)
        else:
            x = sch.start_latent(latent, z)
            ref = ko.sample(kind, _eps, ac, n, z, karras=karras, t_start=t_start, latent=latent, step_noise=step_noise)
        got = ko.apply_rows(rows, ts, formula, _eps, x, step_noise=step_noise)
        err = np.abs(got - ref).max()
        assert err < 1e-12 * max(1.0, np.abs(ref).max()), (keep, err)


@pytest.mark.parametrize("renoise", [False, True])
@pytest.mark.parametrize("name", list(KINDS))
def test_inpainting_rules_in_rows_match_oracle(name, renoise):
    """The 2.1 rule (the known region replaces pred_original_sample) and the 2.2 rule (the known region re-noised to the next
    sigma with the unit start noise, the clean latent at the end) through the rows == the oracle loop, to 1e-12; with the 2.2
    rule the known region of the result is the clean latent exactly."""
    kind, karras, formula = KINDS[name]
    ac = _ac()
    n = 10
    rng = np.random.default_rng(5)
    z, init = rng.standard_normal(256), rng.standard_normal(256)
    mask = (rng.random(256) > 0.5).astype(np.float64)
    sch = _schedule(name, ac, n)
    step_noise = rng.standard_normal((sch.num_timesteps, 256)) if kind == "euler_ancestral" else None
    got = ko.apply_rows(sch.coef_rows(), sch.model_timesteps(), formula, _eps, sch.init_noise_scale * z, step_noise=step_noise,
                        inpaint=(init, mask), inpaint_renoise=renoise)
    ref = ko.sample(kind, _eps, ac, n, z, karras=karras, step_noise=step_noise, inpaint=(init, mask), inpaint_renoise=renoise)
    assert np.abs(got - ref).max() < 1e-12 * max(1.0, np.abs(ref).max())
    if renoise:
        assert np.array_equal(got[mask == 1], init[mask == 1])


@pytest.mark.parametrize("n", [2, 10, 25])
def test_grid_endpoints_and_start(n):
    """Karras: the first sigma is the table's sigma at t = T-1, the last at t = 0 (to the last ulp); linspace: t runs from T-1
    to 0 and sigma is interpolated at the fractional t.  The start noise scale is init_noise_sigma in the UNet's input scale,
    and start_latent is add_noise at the first kept sigma in that scale."""
    from kandinsky2.model.gaussian_diffusion import EulerSchedule, HeunSchedule
    ac = _ac()
    s_tab = ko.table_sigmas(ac)
    for cls in (EulerSchedule, HeunSchedule):
        kar = cls(ac, n, spacing="karras")
        assert kar.ve_sigmas[0] == s_tab[-1] and kar.ve_sigmas[n - 1] == s_tab[0] and kar.ve_sigmas[n] == 0.0
        lin = cls(ac, n)
        assert lin.timesteps[0] == len(ac) - 1 and lin.timesteps[-1] == 0.0
        assert lin.ve_sigmas[0] == s_tab[-1] and lin.ve_sigmas[n - 1] == s_tab[0]
        for sch, karras in ((lin, False), (kar, True)):
            _, sig = ko.set_timesteps(ac, n, karras=karras)
            assert np.allclose(sch.ve_sigmas, sig, rtol=1e-13, atol=0)
            start = ko.scale_model_input(ko.init_noise_sigma(sig), sig[0])
            assert abs(sch.init_noise_scale - start) < 1e-15
            k0 = n // 2
            part = cls(ac, n, keep=n - k0, spacing=sch.spacing)
            want = ko.scale_model_input(ko.add_noise(0.7, -1.3, sig[k0]), sig[k0])
            assert abs(part.start_latent(0.7, -1.3) - want) < 1e-14


@pytest.mark.parametrize("n", [1, 2, 10, 25])
def test_heun_issues_2n_minus_1_evaluations(n):
    """Heun: 2N - 1 rows and model timesteps (2 keep - 1 after img2img truncation), stages alternating 1, 2, ..., 2, 1 in loop
    order with the last step first order, and the oracle loop calls the model as often."""
    from kandinsky2.model.gaussian_diffusion import HeunSchedule
    ac = _ac()
    for keep in _keeps(n):
        sch = HeunSchedule(ac, n, keep=keep)
        stages = sch.coef_rows()[::-1, 7]
        assert len(stages) == 2 * keep - 1 == sch.num_timesteps == len(sch.model_timesteps())
        assert list(stages) == [float(i % 2) for i in range(2 * keep - 1)]
        calls = []
        ko.sample("heun", lambda x, t: calls.append(t) or 0.0 * x, ac, n, np.zeros(4), t_start=n - keep,
                  latent=None if keep == n else np.zeros(4))
        assert len(calls) == 2 * keep - 1


def test_rows_structure():
    """Euler is DPM-Solver++ of order 1 on its grid (c_P = 0, no noise); Euler ancestral puts sigma_up in the noise column and
    its last step draws none; both land on D at the end: (c_x, c_D) = (0, 1) and (alpha, sigma_vp)_N = (1, 0).  Heun's last row
    is a first-order step to D: c_x = 1 / alpha, c_d = -sigma."""
    from kandinsky2.model.gaussian_diffusion import EulerSchedule, HeunSchedule
    ac = _ac()
    e = EulerSchedule(ac, 12).coef_rows()[::-1]
    a = EulerSchedule(ac, 12, ancestral=True).coef_rows()[::-1]
    assert not e[:, 4].any() and not e[:, 7].any() and not a[:, 4].any()
    assert (a[:-1, 7] > 0).all() and a[-1, 7] == 0.0
    for rows in (e, a):
        assert tuple(rows[-1, [2, 3, 5, 6]]) == (0.0, 1.0, 1.0, 0.0)
    sch = EulerSchedule(ac, 12)
    c_x = sch.sigmas[1:-1] / sch.sigmas[:-2]
    assert np.allclose(e[:-1, 2], c_x, rtol=1e-13, atol=0)
    h = HeunSchedule(ac, 12)
    last = h.coef_rows()[0]
    assert last[7] == 0.0 and last[3] == 1.0 / h.alphas[11] and last[4] == -h.ve_sigmas[11] and last[5] == 1.0


def test_schedule_rejects_bad_arguments():
    from kandinsky2.model.gaussian_diffusion import EulerSchedule, HeunSchedule
    ac = _ac()
    for cls in (EulerSchedule, HeunSchedule):
        for n, keep, spacing in ((0, None, "linspace"), (10, 0, "linspace"), (10, 11, "linspace"), (10, None, "exponential")):
            with pytest.raises(ValueError):
                cls(ac, n, keep=keep, spacing=spacing)
