"""GPU: the Heun step kernel -- k2_heun_step against a float64 evaluation of its formula on views inside NaN-poisoned memory,
and stages that leave operands unread run on NaN.  The Euler / Heun names' loops against diffusers' schedulers restated in
tests/kdiff_oracle.py, their pipelines and full-size runs are in tests/test_gpu_schedule_samplers.py."""
import numpy as np
import pytest
import torch

from tests.sampler_cases import _ac22

pytestmark = pytest.mark.gpu
ULP = 2.0 ** -24


# ---- the kernel ----------------------------------------------------------------------------------------------------------
def _reference(mo, x, xs, ds, r, g, cond_first, init=None, mask=None, rnoise=None):
    """float64 evaluation of k2_heun_step -> (x', d, and the magnitudes that bound their fp32 rounding)."""
    B = x.shape[0]
    mo, x, xs, ds = mo.double(), x.double(), xs.double(), ds.double()
    c, u = (mo[:B, :4], mo[B:, :4]) if cond_first else (mo[B:, :4], mo[:B, :4])
    d = u + g * (c - u)
    mag_e = u.abs() + abs(g) * (c.abs() + u.abs())
    mag_d = mag_e
    if mask is not None and rnoise is None:
        m, i0 = mask.double(), init.double()
        d = d + r[2] * m * ((r[0] * x - r[1] * d) - i0)
        mag_d = mag_e + abs(r[2]) * m * (abs(r[0] * x) + abs(r[1]) * mag_e + i0.abs())
    if r[7] == 0.0:
        xn, mag = r[3] * x + r[4] * d, abs(r[3] * x) + abs(r[4]) * mag_d
    else:
        xn, mag = r[3] * xs + r[4] * (ds + d), abs(r[3] * xs) + abs(r[4]) * (ds.abs() + mag_d)
    if rnoise is not None:
        m, i0, rn = mask.double(), init.double(), rnoise.double()
        xn = m * (r[5] * i0 + r[6] * rn) + (1 - m) * xn
        mag = m * (abs(r[5] * i0) + abs(r[6] * rn)) + (1 - m) * mag
    return xn, d, mag, mag_d


def _rows():
    """Loop-order rows of a 20-step Heun schedule -- the first predictor and corrector, an interior pair, the last (first-order)
    step -- and random rows of each stage with every coefficient non-zero."""
    from kandinsky2.model.gaussian_diffusion import HeunSchedule
    rows = HeunSchedule(_ac22(), 20).coef_table()[::-1]
    rnd = np.random.default_rng(3).uniform(0.2, 1.5, (2, 8)).astype(np.float32)
    rnd[:, 4] *= -1
    rnd[0, 7], rnd[1, 7] = 0.0, 1.0
    return [rows[0], rows[1], rows[18], rows[19], rows[-1], rnd[0], rnd[1]]


class _Arena:
    """Tensors carved out of one NaN-filled allocation with NaN gaps between them, so a read outside a view shows up as NaN in
    the result and a write outside the views shows up as a non-NaN gap."""

    GAP = 37

    def __init__(self, shapes):
        sizes = [int(np.prod(s)) for s in shapes]
        self.buf = torch.full((sum(sizes) + self.GAP * (len(sizes) + 1),), float("nan"), device="cuda")
        self.views, self.used = [], torch.zeros_like(self.buf, dtype=torch.bool)
        off = self.GAP
        for s, n in zip(shapes, sizes):
            self.views.append(self.buf[off:off + n].view(s))
            self.used[off:off + n] = True
            off += n + self.GAP

    def gaps_untouched(self):
        return bool(torch.isnan(self.buf[~self.used]).all())


@pytest.mark.parametrize("B,HW", [(1, (5, 7)), (3, (13, 11)), (3, (1, 1))])
def test_kernel_vs_float64(B, HW):
    """Both CFG orders, C2 = 8 (the variance channels NaN: the eps channels are a strided view with NaN gaps) and C2 = 4, no
    inpainting / 2.1 D-replace / 2.2 renoise, odd B*H*W, every operand a view inside NaN-poisoned memory: x' within 8 fp32
    ulps of the float64 terms; stage 1 stores x exactly and d within 8 ulps; stage 2 leaves its two buffers as they were;
    nothing outside the views is written."""
    from kandinsky2 import ops
    H, W = HW
    g = torch.Generator(device="cuda").manual_seed(B * 1000 + H)
    for C2 in (8, 4):
        for cond_first in (True, False):
            for mode in ("none", "x0", "renoise"):
                for ri, row in enumerate(_rows()):
                    ar = _Arena([(2 * B, C2, H, W), (B, 4, H, W), (B, 4, H, W), (B, 4, H, W), (B, 4, H, W), (B, 1, H, W),
                                 (B, 4, H, W), (8,)])
                    mo, x, xs, ds, init, mask, rnoise, coef = ar.views
                    mo[:, :4].copy_(torch.randn(2 * B, 4, H, W, device="cuda", generator=g))
                    for t in (x, xs, ds, init, rnoise):
                        t.copy_(torch.randn(t.shape, device="cuda", generator=g))
                    mask.copy_((torch.rand(mask.shape, device="cuda", generator=g) > 0.5).float())
                    coef.copy_(torch.from_numpy(row.copy()))
                    inp = {} if mode == "none" else dict(inpaint_init=init, inpaint_mask=mask)
                    if mode == "renoise":
                        inp["inpaint_noise"] = rnoise
                    r = [float(v) for v in row]
                    ref, ref_d, mag, mag_d = _reference(mo, x, xs, ds, r, 4.0, cond_first, init if inp else None,
                                                        mask if inp else None, rnoise if mode == "renoise" else None)
                    x_in, xs_in, ds_in = x.clone(), xs.clone(), ds.clone()
                    ops.heun_step(mo, x, xs, ds, coef, 4.0, cond_first, **inp)
                    what = (C2, cond_first, mode, ri)
                    assert ((x.double() - ref).abs() <= 8 * ULP * mag + 1e-30).all(), what
                    if r[7] == 0.0:
                        assert torch.equal(xs, x_in), what
                        assert ((ds.double() - ref_d).abs() <= 8 * ULP * mag_d + 1e-30).all(), what
                    else:
                        assert torch.equal(xs, xs_in) and torch.equal(ds, ds_in), what
                    assert ar.gaps_untouched() and torch.isnan(mo[:, 4:]).all(), what
                    if mode == "renoise" and ri == 4:   # the last step blends with the clean latent exactly
                        keep = mask.bool().expand_as(x)
                        assert torch.equal(x[keep], init[keep])


def test_unread_operands_may_hold_nan():
    """Stage 1 never reads the pre-step latent or derivative buffers; stage 2 reads x only under the 2.1 rule: NaN there gives
    the same bits as any finite contents, and the stored buffers and the result stay finite."""
    from kandinsky2 import ops
    from kandinsky2.model.gaussian_diffusion import HeunSchedule
    B, H, W = 2, 13, 11
    rows = HeunSchedule(_ac22(), 10).coef_table()[::-1]
    g = torch.Generator(device="cuda").manual_seed(9)
    init = torch.randn(B, 4, H, W, device="cuda", generator=g)
    mask = (torch.rand(B, 1, H, W, device="cuda", generator=g) > 0.5).float()
    rnoise = torch.randn(B, 4, H, W, device="cuda", generator=g)
    nan = torch.full((B, 4, H, W), float("nan"), device="cuda")
    for row in (rows[0], rows[2], rows[-1], rows[1], rows[3]):
        coef = torch.from_numpy(row.copy()).cuda()
        stage2 = row[7] != 0.0
        for mode in ("none", "x0", "renoise"):
            inp = {} if mode == "none" else dict(inpaint_init=init, inpaint_mask=mask)
            if mode == "renoise":
                inp["inpaint_noise"] = rnoise
            if stage2 and mode == "x0":
                continue
            for cond_first in (True, False):
                mo = torch.randn(2 * B, 8, H, W, device="cuda", generator=g)
                x, xs, ds = (torch.randn(B, 4, H, W, device="cuda", generator=g) for _ in range(3))
                a = [x.clone(), xs.clone(), ds.clone()]
                b = [nan.clone(), xs.clone(), ds.clone()] if stage2 else [x.clone(), nan.clone(), nan.clone()]
                if stage2:
                    a[0] = torch.randn(B, 4, H, W, device="cuda", generator=g)
                ops.heun_step(mo, *a, coef, 3.0, cond_first, **inp)
                ops.heun_step(mo, *b, coef, 3.0, cond_first, **inp)
                assert all(torch.isfinite(t).all() for t in b), (row[7], mode)
                assert all(torch.equal(p, q) for p, q in zip(a, b)), (row[7], mode)
