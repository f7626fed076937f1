"""GPU: the DPM-Solver++(2M) SDE step and DDIM with eta > 0 -- k2_dpm_solver_sde_step against a float64 evaluation of its
formula, the Gaussian SDE loop through the kernel, and DDIM eta = 0.5 against the reference's own sampler
(tests/golden/ddim_eta_tiny.pt).  The SDE and Karras names' loops, pipelines and full-size runs are in
tests/test_gpu_schedule_samplers.py.  Tolerances are stated per test."""
import os

import numpy as np
import pytest
import torch

from tests import dpm_oracle as do
from tests import dpm_sde_oracle as so
from tests.sampler_cases import GOLD, _ac22

pytestmark = pytest.mark.gpu
MU, S = 0.3, 0.5


# ---- the kernel ----------------------------------------------------------------------------------------------------------
def _reference(mo, x, hist, noise, row, g, cond_first, init=None, mask=None, rnoise=None):
    """float64 evaluation of k2_dpm_solver_sde_step -> (x', x0, the magnitudes that bound their fp32 rounding)."""
    B = x.shape[0]
    mo, x, hist, noise = mo.double(), x.double(), hist.double(), noise.double()
    c, u = (mo[:B, :4], mo[B:, :4]) if cond_first else (mo[B:, :4], mo[:B, :4])
    x0 = row[0] * x - row[1] * (u + g * (c - u))
    mag_x0 = abs(row[0] * x) + abs(row[1]) * (u.abs() + abs(g) * (c.abs() + u.abs()))
    if mask is not None and rnoise is None:
        m = mask.double()
        x0 = x0 * (1 - m) + init.double() * m
        mag_x0 = mag_x0 * (1 - m) + init.double().abs() * m
    xn = row[2] * x + row[3] * x0
    mag = abs(row[2] * x) + abs(row[3]) * mag_x0
    if row[4] != 0.0:
        xn, mag = xn + row[4] * hist, mag + abs(row[4] * hist)
    if row[7] != 0.0:
        xn, mag = xn + row[7] * noise, mag + abs(row[7] * noise)
    if rnoise is not None:
        m = mask.double()
        xn = m * (row[5] * init.double() + row[6] * rnoise.double()) + (1 - m) * xn
        mag = m * (abs(row[5] * init.double()) + abs(row[6] * rnoise.double())) + (1 - m) * mag
    return xn, x0, mag, mag_x0


def _rows():
    """Step-order SDE rows of a 20-step schedule (a second-order, the first and the last row) and a random row with every
    coefficient non-zero."""
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule
    rows = DPMSolverSchedule(_ac22(), 20, sde=True).coef_table()[::-1]
    rnd = np.random.default_rng(3).uniform(0.2, 1.5, 8).astype(np.float32) * np.array([1, 1, 1, 1, -1, 1, 1, 1], np.float32)
    assert rows[7][4] != 0 and rows[7][7] != 0 and rows[0][4] == 0 and rows[-1][7] == 0
    return [rows[7], rows[0], rows[-1], rnd]


@pytest.mark.parametrize("B,HW", [(1, (8, 8)), (4, (96, 96)), (3, (5, 7))])
def test_sde_kernel_vs_float64(B, HW):
    """Both CFG orders, C2 = 8 and 4, no inpainting / 2.1 x0-replace / 2.2 renoise, and a ragged B*4*H*W: x and hist within 8
    fp32 ulps of the magnitudes.  A row with c_P = 0 never reads the history and one with c_N = 0 never reads the noise (NaN
    there changes nothing); with renoise inpainting the last step's kept region is exactly the clean latent."""
    from kandinsky2 import ops
    H, W = HW
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + H)
    init = torch.randn(B, 4, H, W, device="cuda", generator=g)
    mask = (torch.rand(B, 1, H, W, device="cuda", generator=g) > 0.5).float()
    rnoise = torch.randn(B, 4, H, W, device="cuda", generator=g)
    ulp = 2.0 ** -24
    rows = _rows()
    for C2 in (8, 4):
        mo = torch.randn(2 * B, C2, H, W, device="cuda", generator=g)
        for cond_first in (True, False):
            for mode in ("none", "x0", "renoise"):
                inp = {} if mode == "none" else dict(inpaint_init=init, inpaint_mask=mask)
                if mode == "renoise":
                    inp["inpaint_noise"] = rnoise
                for ri, row in enumerate(rows):
                    x = torch.randn(B, 4, H, W, device="cuda", generator=g)
                    hist = torch.randn(B, 4, H, W, device="cuda", generator=g)
                    z = torch.randn(B, 4, H, W, device="cuda", generator=g)
                    coef = torch.from_numpy(row.copy()).cuda()
                    ref, ref_x0, mag, mag_x0 = _reference(mo, x, hist, z, [float(v) for v in row], 4.0, cond_first,
                                                          init if inp else None, mask if inp else None,
                                                          rnoise if mode == "renoise" else None)
                    xo, ho = x.clone(), hist.clone()
                    ops.dpm_solver_step(mo, xo, ho, coef, 4.0, cond_first, noise=z, **inp)
                    assert ((xo.double() - ref).abs() <= 8 * ulp * mag + 1e-30).all(), (C2, cond_first, mode, ri)
                    assert ((ho.double() - ref_x0).abs() <= 8 * ulp * mag_x0 + 1e-30).all(), (C2, cond_first, mode, ri)
                    if row[4] == 0.0 or row[7] == 0.0:
                        nan = torch.full_like(x, float("nan"))
                        xn, hn = x.clone(), (nan.clone() if row[4] == 0.0 else hist.clone())
                        ops.dpm_solver_step(mo, xn, hn, coef, 4.0, cond_first, noise=nan if row[7] == 0.0 else z, **inp)
                        assert torch.isfinite(xn).all() and torch.equal(xn, xo) and torch.equal(hn, ho)
                    if mode == "renoise" and ri == 2:
                        keep = mask.bool().expand_as(xo)
                        assert torch.equal(xo[keep], init[keep])


def test_sde_entry_without_noise_term_is_the_ode_entry():
    """With c_N = 0 and a NaN-filled noise buffer the SDE entry gives the ODE entry's x and hist bit for bit; the ODE entry
    ignores c_N (it has no noise to read)."""
    from kandinsky2 import ops
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule
    B, H, W = 2, 24, 24
    g = torch.Generator(device="cuda").manual_seed(9)
    init = torch.randn(B, 4, H, W, device="cuda", generator=g)
    mask = (torch.rand(B, 1, H, W, device="cuda", generator=g) > 0.5).float()
    rnoise = torch.randn(B, 4, H, W, device="cuda", generator=g)
    nan = torch.full((B, 4, H, W), float("nan"), device="cuda")
    rows = list(DPMSolverSchedule(_ac22(), 10).coef_table()[::-1])
    rows.append(np.random.default_rng(1).uniform(-1, 1, 8).astype(np.float32) * np.array([1] * 7 + [0], np.float32))
    for row in rows:
        assert row[7] == 0.0
        with_cn = row.copy()
        with_cn[7] = 0.75
        for inp in ({}, dict(inpaint_init=init, inpaint_mask=mask), dict(inpaint_init=init, inpaint_mask=mask,
                                                                           inpaint_noise=rnoise)):
            for cond_first in (True, False):
                mo = torch.randn(2 * B, 8, H, W, device="cuda", generator=g)
                x = torch.randn(B, 4, H, W, device="cuda", generator=g)
                hist = torch.randn(B, 4, H, W, device="cuda", generator=g)
                xa, ha, xb, hb, xc, hc = x.clone(), hist.clone(), x.clone(), hist.clone(), x.clone(), hist.clone()
                ops.dpm_solver_step(mo, xa, ha, torch.from_numpy(row.copy()).cuda(), 3.0, cond_first, **inp)
                ops.dpm_solver_step(mo, xb, hb, torch.from_numpy(row.copy()).cuda(), 3.0, cond_first, noise=nan, **inp)
                ops.dpm_solver_step(mo, xc, hc, torch.from_numpy(with_cn).cuda(), 3.0, cond_first, **inp)
                assert torch.equal(xa, xb) and torch.equal(ha, hb) and torch.isfinite(xb).all()
                assert torch.equal(xa, xc) and torch.equal(ha, hc)


# ---- the Gaussian SDE loop through the kernel ----------------------------------------------------------------------------
def test_sde_gaussian_loop_through_kernel():
    """The interior-grid Gaussian SDE problem (t = 999 -> 200), N = 10, 20, 40 steps, run step by step through the SDE entry
    (fp32, NaN-filled history at the start) with injected noise: within 1e-5 relative of the float64 loop on the same noise."""
    from kandinsky2 import ops
    for n in (10, 20, 40):
        a, s = do.smooth_grid(n)
        rows = so.sde_rows(a, s)
        rng = np.random.default_rng(n)
        x0 = torch.from_numpy(rng.standard_normal((2, 4, 8, 8))).cuda()
        z = torch.from_numpy(rng.standard_normal((n, 2, 4, 8, 8)).astype(np.float32)).cuda()
        xt = a[0] * MU + np.sqrt(a[0] ** 2 * S ** 2 + s[0] ** 2) * x0
        x = xt.float().contiguous()
        hist = torch.full_like(x, float("nan"))
        mo = torch.zeros(4, 8, 8, 8, device="cuda")
        for k in range(n):
            eps = do.gaussian_eps(x.double(), a[k], s[k], MU, S).float()
            mo[:2, :4] = eps
            mo[2:, :4] = eps
            ops.dpm_solver_step(mo, x, hist, torch.from_numpy(rows[k].astype(np.float32)).cuda(), 3.0, True, noise=z[k])
        eps_np = lambda xx, k: do.gaussian_eps(xx, a[k], s[k], MU, S)
        zn = z.double().cpu().numpy()
        oracle = so.apply_rows_sde(rows, eps_np, xt.cpu().numpy(), zn)
        assert np.abs(oracle - so.solve_sde(eps_np, xt.cpu().numpy(), a, s, zn)).max() < 1e-12
        got = x.double().cpu().numpy()
        rel = np.linalg.norm(got - oracle) / np.linalg.norm(oracle)
        print(f"Gaussian SDE loop, {n} steps: rel {rel:.2e}")
        assert rel < 1e-5, (n, rel)


# ---- DDIM with eta > 0 against the reference -----------------------------------------------------------------------------
def test_ddim_eta_matches_reference_golden():
    """DDIMSampler.sample(eta=0.5, step_noise=the reference's captured noise) of the product (fused step, fp16 UNet) vs the
    final latents of the reference's own DDIMSampler; the bound of the eta = 0 golden test.  An eta = 0 call on the same
    sampler and model is unchanged by the eta call between, and two eta calls with the same noise are identical."""
    from kandinsky2.model.gaussian_diffusion import DDIMSampler, create_gaussian_diffusion
    from oracle import synth, unet_oracle as uo
    from tests.test_gpu_unet import _build
    fx = torch.load(os.path.join(GOLD, "ddim_eta_tiny.pt"), weights_only=False)
    cfg = fx["cfg"]
    m = _build(cfg, synth.synth_state_dict(uo.unet_param_spec(cfg), seed=fx["weight_seed"]))
    d = create_gaussian_diffusion(steps=1000, learn_sigma=True, noise_schedule="linear", rescale_timesteps=True,
                                  rescale_learned_sigmas=True, timestep_respacing="", linear_start=0.00085, linear_end=0.012)
    x_T = fx["x_T"].cuda()
    B = x_T.shape[0]
    kw = {k: v.cuda() for k, v in fx["cond"].items()}
    sampler = DDIMSampler(m, d)
    call = lambda **k: sampler.sample(fx["steps"], 2 * B, tuple(x_T.shape[1:]), conditioning=kw, x_T=torch.cat([x_T, x_T]),
                                      guidance_scale=fx["guidance"], **k)[0][:B].clone()
    e0 = call()
    out = call(eta=fx["eta"], step_noise=fx["step_noise"].cuda())
    again = call(eta=fx["eta"], step_noise=fx["step_noise"].cuda())
    e0b = call()
    ref = fx["out"].cuda()
    rel = ((out - ref).norm() / ref.norm()).item()
    print(f"DDIM eta {fx['eta']}: rel L2 vs the reference {rel:.3e}")
    assert rel < 3e-2, rel
    assert torch.equal(out, again) and torch.equal(e0, e0b) and not torch.equal(out, e0)
