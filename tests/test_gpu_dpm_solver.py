"""GPU: the DPM-Solver++(2M) step kernel -- k2_dpm_solver_step against a float64 evaluation of its formula, and the analytic
Gaussian problem solved step by step through the kernel.  The sampler's loops, pipelines and full-size runs are in
tests/test_gpu_schedule_samplers.py.  Tolerances are stated per test."""
import numpy as np
import pytest
import torch

from tests import dpm_oracle as do
from tests.sampler_cases import _ac22

pytestmark = pytest.mark.gpu
MU, S = 0.3, 0.5


# ---- the kernel ----------------------------------------------------------------------------------------------------------
def _reference(mo, x, hist, row, g, cond_first, init=None, mask=None, rnoise=None):
    """float64 evaluation of k2_dpm_solver_step and a bound of a few fp32 ulps relative to the magnitudes involved."""
    B = x.shape[0]
    mo, x, hist = mo.double(), x.double(), hist.double()
    c, u = (mo[:B, :4], mo[B:, :4]) if cond_first else (mo[B:, :4], mo[:B, :4])
    eps = u + g * (c - u)
    x0 = row[0] * x - row[1] * eps
    mag_x0 = abs(row[0] * x) + abs(row[1]) * (u.abs() + abs(g) * (c.abs() + u.abs()))
    if mask is not None and rnoise is None:
        m = mask.double()
        x0 = x0 * (1 - m) + init.double() * m
        mag_x0 = mag_x0 * (1 - m) + init.double().abs() * m
    xn = row[2] * x + row[3] * x0
    mag = abs(row[2] * x) + abs(row[3]) * mag_x0
    if row[4] != 0.0:
        xn = xn + row[4] * hist
        mag = mag + abs(row[4] * hist)
    if rnoise is not None:
        m = mask.double()
        xn = m * (row[5] * init.double() + row[6] * rnoise.double()) + (1 - m) * xn
        mag = m * (abs(row[5] * init.double()) + abs(row[6] * rnoise.double())) + (1 - m) * mag
    return xn, x0, mag, mag_x0


@pytest.mark.parametrize("B", [1, 4])
@pytest.mark.parametrize("HW", [(8, 8), (96, 96)])
def test_kernel_vs_float64(B, HW):
    """Both CFG orders, C2 = 8 and 4, every inpainting mode, a second-order row and a first-order row run on a NaN-filled
    history (finite, and equal to the result with any other history): x and hist within 8 fp32 ulps of the magnitudes."""
    from kandinsky2 import ops
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule
    H, W = HW
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + H)
    rows = DPMSolverSchedule(_ac22(), 20).coef_table()[::-1]    # step order
    second, first, last = rows[7], rows[0], rows[-1]
    assert second[4] != 0 and first[4] == 0 and last[4] == 0
    init = torch.randn(B, 4, H, W, device="cuda", generator=g)
    mask = (torch.rand(B, 1, H, W, device="cuda", generator=g) > 0.5).float()
    rnoise = torch.randn(B, 4, H, W, device="cuda", generator=g)
    ulp = 2.0 ** -24
    for C2 in (8, 4):
        mo = torch.randn(2 * B, C2, H, W, device="cuda", generator=g)
        for cond_first in (True, False):
            for mode in ("none", "x0", "renoise"):
                inp = {} if mode == "none" else dict(inpaint_init=init, inpaint_mask=mask)
                if mode == "renoise":
                    inp["inpaint_noise"] = rnoise
                for row in (second, first, last):
                    x = torch.randn(B, 4, H, W, device="cuda", generator=g)
                    hist = torch.randn(B, 4, H, W, device="cuda", generator=g)
                    coef = torch.from_numpy(row.copy()).cuda()
                    r64 = [float(v) for v in row]
                    ref, ref_x0, mag, mag_x0 = _reference(mo, x, hist, r64, 4.0, cond_first, init if inp else None,
                                                  mask if inp else None, rnoise if mode == "renoise" else None)
                    xo, ho = x.clone(), hist.clone()
                    ops.dpm_solver_step(mo, xo, ho, coef, 4.0, cond_first, **inp)
                    assert ((xo.double() - ref).abs() <= 8 * ulp * mag + 1e-30).all(), (C2, cond_first, mode, row)
                    assert ((ho.double() - ref_x0).abs() <= 8 * ulp * mag_x0 + 1e-30).all(), (C2, cond_first, mode, row)
                    if row[4] == 0.0:
                        xn, hn = x.clone(), torch.full_like(hist, float("nan"))
                        ops.dpm_solver_step(mo, xn, hn, coef, 4.0, cond_first, **inp)
                        assert torch.isfinite(xn).all() and torch.equal(xn, xo) and torch.equal(hn, ho)
                    if mode == "renoise" and row is last:   # the last step blends with the clean latent exactly
                        keep = mask.bool().expand_as(xo)
                        assert torch.equal(xo[keep], init[keep])


# ---- the analytic Gaussian problem through the kernel --------------------------------------------------------------------
def _gpu_gaussian(n, order):
    from kandinsky2 import ops
    a, s = do.smooth_grid(n)
    rows = do.rows(a, s, order=order)
    x0 = torch.from_numpy(np.random.default_rng(0).standard_normal((2, 4, 8, 8))).cuda()
    xt = (a[0] * MU + np.sqrt(a[0] ** 2 * S ** 2 + s[0] ** 2) * x0)
    x = xt.float().contiguous()
    hist = torch.full_like(x, float("nan"))
    mo = torch.zeros(4, 8, 8, 8, device="cuda")
    for k in range(n):
        eps = do.gaussian_eps(x.double(), a[k], s[k], MU, S).float()
        mo[:2, :4] = eps
        mo[2:, :4] = eps
        ops.dpm_solver_step(mo, x, hist, torch.from_numpy(rows[k].astype(np.float32)).cuda(), 3.0, True)
    xt64 = xt.cpu().numpy()
    eps_np = lambda xx, k: do.gaussian_eps(xx, a[k], s[k], MU, S)
    oracle = do.apply_rows(rows, eps_np, xt64)
    exact = do.gaussian_flow(xt64, a[0], s[0], a[-1], s[-1], MU, S)
    return x.double().cpu().numpy(), oracle, exact


def test_gaussian_loop_through_kernel():
    """The interior-grid Gaussian problem of the CPU convergence test, N = 10, 20, 40 steps, run step by step through
    ops.dpm_solver_step (fp32, NaN-filled history at the start): within 1e-5 relative of the float64 oracle loop, and the same
    convergence ratios (3-5x per doubling; ~2x with c_P = 0)."""
    for order, lo, hi in ((2, 3.0, 5.0), (1, 1.8, 2.2)):
        errs = []
        for n in (10, 20, 40):
            got, oracle, exact = _gpu_gaussian(n, order)
            rel = np.linalg.norm(got - oracle) / np.linalg.norm(oracle)
            assert rel < 1e-5, (order, n, rel)
            errs.append(np.abs(got - exact).max())
        ratios = [errs[i] / errs[i + 1] for i in range(2)]
        assert all(lo <= r <= hi for r in ratios), (order, errs, ratios)
