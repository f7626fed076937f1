"""GPU: the UniPC step kernel -- k2_unipc_step against a float64 evaluation of its formula, rows that leave operands unread run
on NaN, and the Gaussian loop through the kernel.  The sampler's loops, pipelines and full-size run are in
tests/test_gpu_schedule_samplers.py.  Tolerances are stated per test."""
import numpy as np
import pytest
import torch

from tests import dpm_oracle as do
from tests import unipc_oracle as uo
from tests.sampler_cases import _ac22

pytestmark = pytest.mark.gpu
MU, S = 0.3, 0.5


# ---- the kernel ----------------------------------------------------------------------------------------------------------
def _reference(mo, x, last, h1, h2, r, g, cond_first, init=None, mask=None, rnoise=None):
    """float64 evaluation of k2_unipc_step -> (x', last', D, and the magnitudes that bound their fp32 rounding)."""
    B = x.shape[0]
    mo, x, last, h1, h2 = mo.double(), x.double(), last.double(), h1.double(), h2.double()
    c, u = (mo[:B, :4], mo[B:, :4]) if cond_first else (mo[B:, :4], mo[:B, :4])
    d = r[0] * x - r[1] * (u + g * (c - u))
    mag_d = abs(r[0] * x) + abs(r[1]) * (u.abs() + abs(g) * (c.abs() + u.abs()))
    if mask is not None and rnoise is None:
        m = mask.double()
        d = d * (1 - m) + init.double() * m
        mag_d = mag_d * (1 - m) + init.double().abs() * m
    xc, mag_c = r[4] * d, abs(r[4]) * mag_d
    for coef, v in ((r[2], x), (r[3], last), (r[5], h1), (r[6], h2)):
        if coef != 0.0:
            xc, mag_c = xc + coef * v, mag_c + abs(coef * v)
    xn, mag = r[7] * xc + r[8] * d, abs(r[7]) * mag_c + abs(r[8]) * mag_d
    if r[9] != 0.0:
        xn, mag = xn + r[9] * h1, mag + abs(r[9] * h1)
    if rnoise is not None:
        m = mask.double()
        xn = m * (r[10] * init.double() + r[11] * rnoise.double()) + (1 - m) * xn
        mag = m * (abs(r[10] * init.double()) + abs(r[11] * rnoise.double())) + (1 - m) * mag
    return xn, xc, d, mag, mag_c, mag_d


def _rows():
    """Step-order rows of a 20-step schedule -- the first (no corrector), the second (first-order corrector), an interior one
    and the last -- and a random row with every coefficient non-zero."""
    from kandinsky2.model.gaussian_diffusion import UniPCSchedule
    rows = UniPCSchedule(_ac22(), 20).coef_table()[::-1]
    rnd = np.random.default_rng(3).uniform(0.2, 1.5, 16).astype(np.float32)
    rnd[[5, 9]] *= -1
    rnd[12:] = 0
    return [rows[0], rows[1], rows[7], rows[-1], rnd]


@pytest.mark.parametrize("B,HW", [(1, (8, 8)), (3, (5, 7)), (2, (13, 11)), (4, (96, 96))])
def test_kernel_vs_float64(B, HW):
    """Both CFG orders, C2 = 8 and 4, no inpainting / 2.1 D-replace / 2.2 renoise, ragged B*4*H*W: x, last and D within 8 fp32
    ulps of the magnitudes, the history shifted (h2 = old h1); the row read through the step counter from a staged table gives
    the same bits as the row passed alone."""
    from kandinsky2 import ops
    H, W = HW
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + H)
    init = torch.randn(B, 4, H, W, device="cuda", generator=g)
    mask = (torch.rand(B, 1, H, W, device="cuda", generator=g) > 0.5).float()
    rnoise = torch.randn(B, 4, H, W, device="cuda", generator=g)
    ulp = 2.0 ** -24
    rows = _rows()
    table = torch.from_numpy(np.stack(rows)).cuda()
    for C2 in (8, 4):
        mo = torch.randn(2 * B, C2, H, W, device="cuda", generator=g)
        for cond_first in (True, False):
            for mode in ("none", "x0", "renoise"):
                inp = {} if mode == "none" else dict(inpaint_init=init, inpaint_mask=mask)
                if mode == "renoise":
                    inp["inpaint_noise"] = rnoise
                for ri, row in enumerate(rows):
                    x, last, h1, h2 = (torch.randn(B, 4, H, W, device="cuda", generator=g) for _ in range(4))
                    r = [float(v) for v in row]
                    ref, ref_c, ref_d, mag, mag_c, mag_d = _reference(mo, x, last, h1, h2, r, 4.0, cond_first,
                                                                      init if inp else None, mask if inp else None,
                                                                      rnoise if mode == "renoise" else None)
                    xo, lo, h1o, h2o = x.clone(), last.clone(), h1.clone(), h2.clone()
                    ops.unipc_step(mo, xo, lo, h1o, h2o, torch.from_numpy(row.copy()).cuda(), 4.0, cond_first, **inp)
                    what = (C2, cond_first, mode, ri)
                    assert ((xo.double() - ref).abs() <= 8 * ulp * mag + 1e-30).all(), what
                    assert ((lo.double() - ref_c).abs() <= 8 * ulp * mag_c + 1e-30).all(), what
                    assert ((h1o.double() - ref_d).abs() <= 8 * ulp * mag_d + 1e-30).all(), what
                    assert torch.equal(h2o, h1), what
                    xs, ls, h1s, h2s = x.clone(), last.clone(), h1.clone(), h2.clone()
                    counter = torch.tensor([ri + len(rows), len(rows)], device="cuda", dtype=torch.int32)  # k mod steps
                    ops.unipc_step(mo, xs, ls, h1s, h2s, table, 4.0, cond_first, counter=counter, **inp)
                    assert torch.equal(xs, xo) and torch.equal(ls, lo) and torch.equal(h1s, h1o) and torch.equal(h2s, h2o), what
                    if mode == "renoise" and ri == 3:
                        keep = mask.bool().expand_as(xo)
                        assert torch.equal(xo[keep], init[keep])


def test_unread_operands_may_hold_nan():
    """A row without a corrector never reads last, D_{k-1} or D_{k-2}; a first-order corrector row never reads D_{k-2}; a
    first-order predictor without a corrector never reads D_{k-1}: NaN there gives the same x, last and D bits as zeros."""
    from kandinsky2 import ops
    from kandinsky2.model.gaussian_diffusion import UniPCSchedule
    B, H, W = 2, 13, 11
    rows = UniPCSchedule(_ac22(), 10).coef_table()[::-1]
    g = torch.Generator(device="cuda").manual_seed(9)
    init = torch.randn(B, 4, H, W, device="cuda", generator=g)
    mask = (torch.rand(B, 1, H, W, device="cuda", generator=g) > 0.5).float()
    rnoise = torch.randn(B, 4, H, W, device="cuda", generator=g)
    nan = torch.full((B, 4, H, W), float("nan"), device="cuda")
    cases = [(rows[0], ("last", "h1", "h2")), (rows[1], ("h2",))]
    one = UniPCSchedule(_ac22(), 1).coef_table()[0]            # the only step: first order, no corrector, lands on D
    cases.append((one, ("last", "h1", "h2")))
    for row, unread in cases:
        coef = torch.from_numpy(row.copy()).cuda()
        for inp in ({}, dict(inpaint_init=init, inpaint_mask=mask), dict(inpaint_init=init, inpaint_mask=mask,
                                                                           inpaint_noise=rnoise)):
            for cond_first in (True, False):
                mo = torch.randn(2 * B, 8, H, W, device="cuda", generator=g)
                x = torch.randn(B, 4, H, W, device="cuda", generator=g)
                base = {k: torch.randn(B, 4, H, W, device="cuda", generator=g) for k in ("last", "h1", "h2")}
                zeros = {k: (torch.zeros_like(v) if k in unread else v.clone()) for k, v in base.items()}
                nans = {k: (nan.clone() if k in unread else v.clone()) for k, v in base.items()}
                xa, xb = x.clone(), x.clone()
                ops.unipc_step(mo, xa, zeros["last"], zeros["h1"], zeros["h2"], coef, 3.0, cond_first, **inp)
                ops.unipc_step(mo, xb, nans["last"], nans["h1"], nans["h2"], coef, 3.0, cond_first, **inp)
                assert torch.isfinite(xb).all() and torch.isfinite(nans["last"]).all() and torch.isfinite(nans["h1"]).all()
                assert torch.equal(xa, xb) and torch.equal(zeros["last"], nans["last"]) and torch.equal(zeros["h1"], nans["h1"])


# ---- the Gaussian loop through the kernel --------------------------------------------------------------------------------
def test_gaussian_loop_through_kernel():
    """The Gaussian problem on the sampler's own grid (2.2 table, t = 999 -> sigma = 0), N = 10, 20, 40, run step by step
    through k2_unipc_step (fp32, NaN-filled last sample and history at the start) vs the float64 loop on the same fp32 rows:
    relative L2 within 1.5e-7 sqrt(N / 10).  The rounding of N fp32 steps grows like sqrt(N): the same loop in numpy float32
    gives 1.5e-7 / 2.0e-7 / 2.6e-7 at N = 10 / 20 / 40."""
    from kandinsky2 import ops
    from kandinsky2.model.gaussian_diffusion import UniPCSchedule
    for n in (10, 20, 40):
        sch = UniPCSchedule(_ac22(), n)
        a, s = sch.alphas, sch.sigmas
        rows = sch.coef_table()[::-1]
        rng = np.random.default_rng(n)
        x = torch.from_numpy(rng.standard_normal((2, 4, 8, 8)).astype(np.float32)).cuda()
        xt = x.double().cpu().numpy()
        last, h1, h2 = (torch.full_like(x, float("nan")) for _ in range(3))
        mo = torch.zeros(4, 8, 8, 8, device="cuda")
        for k in range(n):
            eps = do.gaussian_eps(x.double(), a[k], s[k], MU, S).float()
            mo[:2, :4] = eps
            mo[2:, :4] = eps
            ops.unipc_step(mo, x, last, h1, h2, torch.from_numpy(rows[k].copy()).cuda(), 3.0, True)
        eps_np = lambda xx, k: do.gaussian_eps(xx, a[k], s[k], MU, S)
        oracle = uo.apply_rows(rows.astype(np.float64), eps_np, xt)
        assert np.abs(uo.apply_rows(sch.coef_rows()[::-1], eps_np, xt) - uo.solve(eps_np, xt, a, s)).max() < 1e-12
        got = x.double().cpu().numpy()
        rel = np.linalg.norm(got - oracle) / np.linalg.norm(oracle)
        print(f"Gaussian UniPC loop, {n} steps: rel {rel:.2e}")
        assert rel <= 1.5e-7 * np.sqrt(n / 10), (n, rel)
