"""GPU: the sampler kernels at their edges, against float64 evaluations of the same update rules.

  - the split threshold step (k2_sampler_step modes 2 / 3 / 4) the sharded 2.1 pipeline runs, on one GPU;
  - the dynamic threshold's percentile (claimed exact: a radix select of the two order statistics and numpy's linear
    interpolation in fp64) against np.percentile in float64 on adversarial x0;
  - the DDPM inpainting blends of 2.1 (x0 replaced by the known latent) and 2.2 (known region re-noised, coef[7] = 1 last step);
  - k2_plms_step with every history length, both CFG row orders, C2 4 / 8, with and without the e_t store;
  - k2_step_begin / k2_step_end: the step counter wraps, a NULL noise sequence leaves the noise buffer alone, nt != B.
Outputs live in guarded buffers (tests/test_gpu_kernel_bounds.py: _Guarded) whose bytes outside the view must not change."""
import numpy as np
import pytest
import torch

from tests.test_gpu_kernel_bounds import _Guarded, _assert_untouched, _bits

pytestmark = pytest.mark.gpu

COEF = [1.2, 0.7, 0.3, 0.69, -5.0, -3.0, 1.0, 0.0]   # as test_gpu_ops.py::test_sampler_step


def _inputs(B, H, W, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    r = lambda *s: torch.randn(*s, device="cuda", generator=g)
    mo, x, noise = r(2 * B, 8, H, W), r(B, 4, H, W), r(B, 4, H, W)
    init, rnoise = r(B, 4, H, W), r(B, 4, H, W)
    mask = (torch.rand(B, 1, H, W, device="cuda", generator=g) > 0.5).float()
    return mo, x, noise, init, mask, rnoise


def _ref_step(mo, x, noise, coef, g, clip, s=None, init=None, mask=None, rnoise=None, cond_first=True):
    """float64 restatement of k2_sampler_step: CFG, x0 clamp, 2.1 x0 replace, optional threshold s, learned-range posterior,
    2.2 renoise blend."""
    mo, x, noise, c = mo.double(), x.double(), noise.double(), [float(v) for v in coef]
    B = x.shape[0]
    cond, unc = (mo[:B], mo[B:]) if cond_first else (mo[B:], mo[:B])
    eps = unc[:, :4] + g * (cond[:, :4] - unc[:, :4])
    x0 = (c[0] * x - c[1] * eps).clamp(-clip, clip)
    if mask is not None and rnoise is None:
        x0 = x0 * (1 - mask.double()) + init.double() * mask.double()
    if s is not None:
        x0 = x0.clamp(-s, s) / s
    frac = (cond[:, 4:] + 1) / 2
    xp = c[2] * x0 + c[3] * x + c[6] * torch.exp(0.5 * (frac * c[5] + (1 - frac) * c[4])) * noise
    if rnoise is not None:
        m = mask.double()
        xp = m * (c[7] * init.double() + (1 - c[7] ** 2) ** 0.5 * rnoise.double()) + (1 - m) * xp
    return xp


def _percentile_s(x0):
    """The reference's dynamic threshold of sample 0 in float64, rounded to fp32 (gaussian_diffusion.py:284-294)."""
    s = np.percentile(np.abs(x0[0].double().cpu().numpy()), 99.5)
    return np.float32(max(s, 1.0))


@pytest.mark.parametrize("inpaint", [False, True])
def test_split_threshold_step_matches_fused(inpaint):
    """mode 2 (x0 + threshold of local sample 0 into work) followed by mode 3 (the update) is bit-identical to mode 1; mode 4
    (x0 only), a chosen s written into work[B*4*H*W], then mode 3 equals the float64 rule with that s."""
    from kandinsky2 import ops
    B, H, W = 2, 12, 12
    mo, x, noise, init, mask, _ = _inputs(B, H, W, 1)
    coef = torch.tensor(COEF, device="cuda")
    kw = dict(inpaint_init=init, inpaint_mask=mask) if inpaint else {}
    n = B * 4 * H * W
    fused = ops.sampler_step(mo, x.clone(), noise, coef, 4.0, 1, clip=2.0, threshold_mode=1, **kw)
    work = torch.full((n + 4096,), float("nan"), device="cuda")
    xs = x.clone()
    ops.sampler_step(mo, xs, noise, coef, 4.0, 1, clip=2.0, threshold_mode=2, work=work, **kw)
    assert torch.equal(xs, x), "mode 2 must not update x"
    s2 = work[n].item()
    ops.sampler_step(mo, xs, noise, coef, 4.0, 1, clip=2.0, threshold_mode=3, work=work, **kw)
    assert torch.equal(xs, fused)
    assert s2 == float(_percentile_s(work[:n].view(B, 4, H, W)))
    # mode 4 + a threshold of another rank's sample 0
    work.fill_(float("nan"))
    xs = x.clone()
    ops.sampler_step(mo, xs, noise, coef, 4.0, 1, clip=2.0, threshold_mode=4, work=work, **kw)
    assert torch.equal(xs, x) and torch.isnan(work[n]), "mode 4 computes x0 only"
    s = 1.37
    work[n] = s
    ops.sampler_step(mo, xs, noise, coef, 4.0, 1, clip=2.0, threshold_mode=3, work=work, **kw)
    ref = _ref_step(mo, x, noise, coef, 4.0, 2.0, s=s, init=init if inpaint else None, mask=mask if inpaint else None)
    assert (xs.double() - ref).abs().max().item() < 1e-5   # fp32 arithmetic on O(1) values, as test_sampler_step


def _adversarial(kind, H, W):
    n = 4 * H * W
    g = torch.Generator().manual_seed(H * 1000 + W)
    if kind == "ties":        # a few distinct magnitudes: both order statistics sit inside runs of equal values
        v = torch.tensor([0.5, -1.5, 2.5, -3.0, 3.0])[torch.randint(0, 5, (n,), generator=g)]
    elif kind == "equal":
        v = torch.full((n,), -1.7)
    elif kind == "below_one":  # every |x0| < 1: s = max(percentile, 1) = 1
        v = torch.rand(n, generator=g) * 1.98 - 0.99
    elif kind == "neg_zero":   # -0.0 and +0.0 (|x| drops the sign bit) below a small tail of large values
        v = torch.where(torch.rand(n, generator=g) < 0.5, torch.tensor(-0.0), torch.tensor(0.0))
        v[: n // 100 + 2] = torch.linspace(1.0, 7.0, n // 100 + 2)
    elif kind == "top_pair":   # the two order statistics differ a lot: the interpolation weight matters
        v = torch.randn(n, generator=g)
        v[torch.randperm(n, generator=g)[: n // 200 + 1]] = 50.0
    else:
        v = torch.randn(n, generator=g) * 3
    return v.reshape(1, 4, H, W)


@pytest.mark.parametrize("kind", ["ties", "equal", "below_one", "neg_zero", "top_pair", "normal"])
@pytest.mark.parametrize("H,W", [(8, 8), (12, 12), (96, 96), (10, 10), (20, 20)])
def test_percentile_threshold_exact(kind, H, W):
    """The threshold mode 2 writes equals max(np.percentile(|x0[0]|, 99.5), 1) computed in float64 and rounded to fp32.  The
    99.5 % position 0.995 (n - 1) never falls exactly on an element for n = 4 H W (n - 1 is odd); 10 x 10 and 20 x 20 put it
    0.005 past one (interpolation weight ~0), 8 x 8 / 96 x 96 use numpy's t >= 0.5 branch, 12 x 12 the t < 0.5 one, and ties
    make both order statistics equal.  coef = (1, 0, ...) and a huge clip make x0 = x exactly."""
    from kandinsky2 import ops
    B = 2
    v = _adversarial(kind, H, W).cuda()
    x = torch.cat([v, torch.randn(1, 4, H, W, device="cuda") * 100])   # sample 1 must not matter
    mo = torch.randn(2 * B, 8, H, W, device="cuda")
    coef = torch.tensor([1.0, 0.0, 0, 0, 0, 0, 0, 0], device="cuda")
    n = B * 4 * H * W
    work = torch.full((n + 4096,), float("nan"), device="cuda")
    ops.sampler_step(mo, x.clone(), torch.zeros_like(x), coef, 1.0, 1, clip=1e30, threshold_mode=2, work=work)
    x0 = work[:n].view(B, 4, H, W)
    assert torch.equal(_bits(x0[:1].abs()), _bits(v.abs()))
    got = np.float32(work[n].item())
    want = _percentile_s(v)
    assert got == want, (got, want)


@pytest.mark.parametrize("c7", [0.83, 1.0])
@pytest.mark.parametrize("mode", [0, 1])
def test_ddpm_inpaint_blends(c7, mode):
    """2.1: x0 = x0 (1 - mask) + init mask after the clamp (and before the threshold); 2.2: the known region becomes
    c init + sqrt(1 - c^2) noise0 with c = coef[7], the clean latent itself at the last step (c = 1)."""
    from kandinsky2 import ops
    B, H, W = 2, 8, 12
    mo, x, noise, init, mask, rnoise = _inputs(B, H, W, 2)
    coef = torch.tensor(COEF[:7] + [c7], device="cuda")
    for cond_first in (1, 0):
        for renoise in (False, True):
            if renoise and mode == 1:
                continue   # 2.2 runs no dynamic threshold
            out = ops.sampler_step(mo, x.clone(), noise, coef, 4.0, cond_first, clip=2.0, threshold_mode=mode, inpaint_init=init,
                                   inpaint_mask=mask, inpaint_noise=rnoise if renoise else None)
            s = None
            if mode == 1:   # the threshold of the float64 x0 (clamped, known region replaced) of sample 0
                c = [float(v) for v in coef]
                cond, unc = (mo[:B], mo[B:]) if cond_first else (mo[B:], mo[:B])
                eps = unc[:, :4].double() + 4.0 * (cond[:, :4].double() - unc[:, :4].double())
                x0 = (c[0] * x.double() - c[1] * eps).clamp(-2, 2)
                x0 = x0 * (1 - mask.double()) + init.double() * mask.double()
                s = float(max(np.percentile(np.abs(x0[0].cpu().numpy()), 99.5), 1.0))
            ref = _ref_step(mo, x, noise, coef, 4.0, 2.0, s=s, init=init, mask=mask, rnoise=rnoise if renoise else None,
                            cond_first=bool(cond_first))
            # fp32 arithmetic on O(1) values, as test_sampler_step (the threshold is the kernel's fp32 s, exact per the test above)
            assert (out.double() - ref).abs().max().item() < 1e-5, (cond_first, renoise)
            if renoise and c7 == 1.0:
                keep = mask.bool().expand_as(out)
                assert torch.equal(out[keep], init[keep]), "last step: the known region is the clean latent"


@pytest.mark.parametrize("C2", [4, 8])
@pytest.mark.parametrize("cond_first", [0, 1])
@pytest.mark.parametrize("nhist", [0, 1, 2, 3])
@pytest.mark.parametrize("store", [True, False])
def test_plms_step_vs_float64(C2, cond_first, nhist, store):
    from kandinsky2 import ops
    B, H, W = 2, 6, 10
    g = torch.Generator(device="cuda").manual_seed(C2 * 10 + nhist)
    mo = torch.randn(2 * B, C2, H, W, device="cuda", generator=g)
    x = torch.randn(B, 4, H, W, device="cuda", generator=g)
    hist = [torch.randn(B, 4, H, W, device="cuda", generator=g) for _ in range(nhist)]
    w = [55 / 24, -59 / 24, 37 / 24, -9 / 24][: nhist + 1] + [0.0] * (3 - nhist)
    coef = torch.tensor([1.3, 0.8, 0.9, 0.4] + w, device="cuda")
    n = B * 4 * H * W
    go = _Guarded((n,), 1, dtype=torch.float32, out=True)
    gs = _Guarded((n,), 1, dtype=torch.float32, out=True)
    out = go.view.view(B, 4, H, W)
    st = gs.view.view(B, 4, H, W) if store else None
    ops.plms_step(mo, x, out, hist, st, coef, 3.0, cond_first)
    torch.cuda.synchronize()
    _assert_untouched(go, gs)
    if not store:
        assert (_bits(gs.view) == gs.bits).all(), "a NULL store writes nothing"
    md = mo.double()
    cond, unc = (md[:B], md[B:]) if cond_first else (md[B:], md[:B])
    e_t = unc[:, :4] + 3.0 * (cond[:, :4] - unc[:, :4])
    c = [float(v) for v in coef]
    ep = c[4] * e_t + sum(c[5 + j] * hist[j].double() for j in range(nhist))
    ref = c[2] * (c[0] * x.double() - c[1] * ep) + c[3] * ep
    # fp32 arithmetic on O(1..10) values (Adams-Bashforth weights up to 2.5)
    assert (out.double() - ref).abs().max().item() < 2e-5 * max(1.0, ref.abs().max().item())
    if store:
        assert (st.double() - e_t).abs().max().item() < 1e-5 * max(1.0, e_t.abs().max().item())


@pytest.mark.parametrize("with_noise", [True, False])
def test_step_begin_end_counter(with_noise):
    """k = counter[0] % counter[1] with counter[0] >= counter[1] (wraps); nt != B; a NULL noise sequence leaves noise alone.
    Bit-exact copies, guard bands on x_in, t_in, coef_out and noise; step_end adds 1 to counter[0] only."""
    from kandinsky2 import ops
    B, H, W, steps, nt = 2, 5, 7, 3, 5
    n = B * 4 * H * W
    g = torch.Generator(device="cuda").manual_seed(7)
    x = torch.randn(B, 4, H, W, device="cuda", generator=g)
    ts_seq = torch.tensor([981.0, 500.5, 3.0], device="cuda")
    coef_seq = torch.randn(steps, 8, device="cuda", generator=g)
    noise_seq = torch.randn(steps, B, 4, H, W, device="cuda", generator=g) if with_noise else None
    gx = _Guarded((2 * n,), 1, dtype=torch.float32, out=True)
    gt = _Guarded((nt,), 1, dtype=torch.float32, out=True)
    gc = _Guarded((8,), 1, dtype=torch.float32, out=True)
    gn = _Guarded((n,), 1, dtype=torch.float32, out=True)
    counter = torch.tensor([7, steps], device="cuda", dtype=torch.int32)   # k = 7 % 3 = 1
    ops.step_begin(x, gx.view.view(-1), gt.view.view(-1), gc.view.view(-1), ts_seq, coef_seq, noise_seq, gn.view.view(-1),
                   counter)
    ops.step_end(counter)
    torch.cuda.synchronize()
    _assert_untouched(gx, gt, gc, gn)
    k = 1
    assert torch.equal(gx.view.view(2, -1), x.reshape(1, -1).expand(2, -1))
    assert torch.equal(gt.view.view(-1), ts_seq[k].expand(nt))
    assert torch.equal(gc.view.view(-1), coef_seq[k])
    if with_noise:
        assert torch.equal(gn.view.view(-1), noise_seq[k].reshape(-1))
    else:
        assert (_bits(gn.view) == gn.bits).all(), "noise_seq NULL: noise untouched"
    assert counter.tolist() == [8, steps]
