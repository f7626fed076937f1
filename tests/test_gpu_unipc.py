"""GPU: the UniPC sampler -- k2_unipc_step against a float64 evaluation of its formula, rows that leave operands unread run on
NaN, the Gaussian loop through the kernel, graph-replayed tiny-UNet loops against the float64 oracle loop (tests/unipc_oracle.py)
driven by the fp32 oracle UNet, graph replay against step-at-a-time execution, the pipelines' unipc sampler names, and 10
full-size cfg-2 steps.  Tolerances are stated per test; the loop bounds are those of tests/test_gpu_dpm_solver.py."""
import numpy as np
import pytest
import torch

from tests import dpm_oracle as do
from tests import unipc_oracle as uo
from tests.test_gpu_dpm_solver import _ac22, _base21, _no_tf32, _pipe, _run, _same, _traj_tiny

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


# ---- tiny-UNet trajectories ----------------------------------------------------------------------------------------------
def _check(out, ref, what):
    err = (out - ref).abs().max().item()
    rel = ((out - ref).norm() / ref.norm()).item()
    print(f"{what}: rel L2 {rel:.3e}, max abs {err:.3e}")
    assert torch.isfinite(out).all()
    assert rel < 2e-2 and err < 0.15 * ref.abs().max().item(), (what, err, rel, ref.abs().max().item())


@pytest.mark.parametrize("inpaint", [False, True])
@pytest.mark.parametrize("spacing", ["linspace", "karras"])
def test_loop_21_head_matches_oracle(spacing, inpaint):
    """2.1 head (cond rows first), 5 UniPC steps at guidance 3 through the graph-replayed loop vs the oracle loop driven by the
    fp32 oracle UNet, with and without the 2.1 inpainting rule (the known region replaces D, so the result's known region is
    exactly the clean latent)."""
    from kandinsky2.model.gaussian_diffusion import UniPCSchedule
    from oracle import unet_oracle as uo_net
    fx, sd, m = _traj_tiny()
    cfg = fx["cfg"]
    x_T = fx["x_T"].cuda()
    B = x_T.shape[0]
    kw = {k: v.cuda() for k, v in fx["cond"].items()}
    n, gs = 5, 3.0
    sch = UniPCSchedule(_base21(), n, spacing=spacing)
    extra, oinp = {}, None
    if inpaint:
        g = torch.Generator(device="cuda").manual_seed(6)
        init = torch.randn(B, 4, 16, 16, device="cuda", generator=g)
        mask = (torch.rand(B, 1, 16, 16, device="cuda", generator=g) > 0.4).float()
        extra = dict(inpaint_init=init, inpaint_mask=mask, inpaint_renoise=False)
        oinp = (init, mask, None)
    out = sch.sample(m, (2 * B, 4, 16, 16), noise=torch.cat([x_T, x_T]), model_kwargs=kw, guidance_scale=gs, cond_first=True,
                     device="cuda", **extra)[:B]
    sdc = {k: v.cuda() for k, v in sd.items()}

    def eps(x, k):
        mo = uo_net.unet_forward(sdc, cfg, torch.cat([x, x]), torch.full((2 * B,), float(sch.timesteps[k]), device="cuda"), **kw)
        return mo[B:, :4] + gs * (mo[:B, :4] - mo[B:, :4])

    with torch.no_grad():
        ref = uo.solve(eps, x_T.clone(), sch.alphas, sch.sigmas, inpaint=oinp, inpaint_renoise=False)
    _check(out, ref, f"2.1 head, {spacing}, inpaint={inpaint}")
    if inpaint:
        keep = mask.bool().expand_as(out)
        assert torch.equal(out[keep], init[keep])


@pytest.mark.parametrize("inpaint", [False, True])
@pytest.mark.parametrize("spacing", ["linspace", "karras"])
def test_loop_22_head_matches_oracle(spacing, inpaint):
    """2.2 order (unconditional rows first), 6 UniPC steps at guidance 4, with and without the renoise inpainting rule, vs the
    oracle loop; with inpainting the kept region of the result is exactly the clean latent."""
    from kandinsky2.model.gaussian_diffusion import UniPCSchedule
    from oracle import synth, unet_oracle as uo_net
    from tests.test_gpu_unet import _build
    cfg = dict(uo_net.CONFIG_TINY, inpainting=inpaint)
    sd = synth.synth_state_dict(uo_net.unet_param_spec(cfg), seed=4)
    m = _build(cfg, sd)
    g = torch.Generator().manual_seed(8)
    B, H, W, n, gs = 2, 16, 16, 6, 4.0
    x_T = torch.randn(B, 4, H, W, generator=g)
    kw = dict(full_emb=torch.randn(2 * B, 7, 96, generator=g), pooled_emb=torch.randn(2 * B, 48, generator=g),
              image_emb=torch.randn(2 * B, 48, generator=g))
    extra, oinp = {}, None
    if inpaint:
        init = torch.randn(1, 4, H, W, generator=g)
        mask = (torch.rand(1, 1, H, W, generator=g) > 0.4).float()
        kw["inpaint_image"] = (init * mask).repeat(2 * B, 1, 1, 1)
        kw["inpaint_mask"] = mask.repeat(2 * B, 1, 1, 1)
        extra = dict(inpaint_init=init.repeat(B, 1, 1, 1).cuda(), inpaint_mask=mask.repeat(B, 1, 1, 1).cuda(),
                     inpaint_renoise=True)
        oinp = (init, mask, x_T)
    sch = UniPCSchedule(_ac22(), n, spacing=spacing)
    out = sch.sample(m, (2 * B, 4, H, W), noise=torch.cat([x_T, x_T]).cuda(), model_kwargs={k: v.cuda() for k, v in kw.items()},
                     guidance_scale=gs, cond_first=False, device="cuda", **extra)[:B].cpu()

    def eps(x, k):
        mo = uo_net.unet_forward(sd, cfg, torch.cat([x, x]), torch.full((2 * B,), float(sch.timesteps[k])), **kw)
        return mo[:B, :4] + gs * (mo[B:, :4] - mo[:B, :4])

    with torch.no_grad():
        ref = uo.solve(eps, x_T.clone(), sch.alphas, sch.sigmas, inpaint=oinp, inpaint_renoise=True)
    _check(out, ref, f"2.2 head, {spacing}, inpaint={inpaint}")
    if inpaint:
        keep = mask.bool().expand(B, 4, H, W)
        assert torch.equal(out[keep], init.expand(B, 4, H, W)[keep])


@pytest.mark.parametrize("spacing", ["linspace", "karras"])
def test_graph_replay_equals_step_at_a_time(spacing):
    """The graph-replayed UniPC loop and the same steps issued one at a time (FusedStep.run with each 16-float row, eager UNet
    plan, NaN-filled last sample and history) give bit-identical latents; so does a second graph-replayed run (set_schedule
    resets the state); a DPM++(2M) run on the same model between them uses its own graph and state."""
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule, FusedStep, UniPCSchedule
    fx, _, m = _traj_tiny()
    x_T = fx["x_T"].cuda()
    B = x_T.shape[0]
    kw = {k: v.cuda() for k, v in fx["cond"].items()}
    sch = UniPCSchedule(_base21(), 6, spacing=spacing)
    dpm = DPMSolverSchedule(_base21(), 6, spacing=spacing)
    shape = (2 * B, 4, 16, 16)
    run = lambda s: s.sample(m, shape, noise=torch.cat([x_T, x_T]), model_kwargs=kw, guidance_scale=3.0, cond_first=True,
                             device="cuda")[:B].clone()
    a, d1 = run(sch), run(dpm)
    b, d2 = run(sch), run(dpm)
    coef, ts = sch._tables(torch.device("cuda"))
    assert coef.shape == (6, 16)
    m.use_cuda_graph = False
    try:
        step = FusedStep(m, B, 16, 16, kw, 3.0, True, 1e30, 0, step_kind="unipc")
        for name in ("last", "hist", "hist2"):
            step.st[name].fill_(float("nan"))
        x = x_T.clone()
        for j in range(sch.num_timesteps)[::-1]:
            step.run(x, ts[j], coef[j])
    finally:
        m.use_cuda_graph = True
    assert torch.equal(a, b) and torch.equal(a, x) and torch.isfinite(a).all()
    assert torch.equal(d1, d2) and not torch.equal(a, d1)


# ---- pipelines -----------------------------------------------------------------------------------------------------------
UNIPC_NAMES = ("unipc_sampler", "unipc_karras_sampler")


def _twice(pipe, method, *args, **kw):
    """-> the latents of the first of two identical calls, after checking both give bit-identical images and latents."""
    i1, l1 = _run(pipe, method, *args, **kw)
    i2, l2 = _run(pipe, method, *args, **kw)
    assert i1[0].size == (64, 64) and _same(i1, i2) and torch.equal(l1, l2) and torch.isfinite(l1).all(), (method, kw)
    return l1


@pytest.mark.parametrize("name", UNIPC_NAMES)
def test_pipeline_21_unipc(name):
    from PIL import Image
    kw = dict(sampler=name, h=64, w=64)
    pipe = _pipe("2.1", "text2img")
    lo = _twice(pipe, "generate_text2img", "a red cat", num_steps=6, batch_size=2, guidance_scale=4,
                **dict(kw, sampler="dpmpp_2m_sampler"))
    la = _twice(pipe, "generate_text2img", "a red cat", num_steps=6, batch_size=2, guidance_scale=4, **kw)
    lo2 = _twice(pipe, "generate_text2img", "a red cat", num_steps=6, batch_size=2, guidance_scale=4,
                 **dict(kw, sampler="dpmpp_2m_sampler"))
    assert not torch.equal(la, lo) and not torch.equal(la[0], la[1]) and torch.equal(lo, lo2)
    _twice(pipe, "mix_images", ["a cat", "a dog"], [0.3, 0.7], num_steps=5, batch_size=1, **kw)
    emb = torch.cat([pipe.embedder.image_emb("a cat", 1), pipe.embedder.zero_image_emb(1)])
    _twice(pipe, "generate_img", "a cat", emb, batch_size=1, guidance_scale=4, num_steps=5, diffusion=pipe._diffusion(name, 5),
           **kw)
    src = Image.fromarray((np.random.default_rng(0).random((70, 90, 3)) * 255).astype("uint8"))
    _twice(_pipe("2.1", "img2img"), "generate_img2img", "a dog", src, strength=0.6, num_steps=8, batch_size=1, **kw)
    lat = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(0))
    mask = torch.ones(64, 64)
    mask[:, 40:] = 0
    _twice(_pipe("2.1", "inpainting"), "generate_inpainting", "a hat", lat, mask.numpy(), num_steps=5, batch_size=1,
           guidance_scale=4, **kw)


@pytest.mark.parametrize("name", UNIPC_NAMES)
def test_pipeline_22_unipc(name):
    from PIL import Image
    kw = dict(sampler=name, h=64, w=64)
    pipe = _pipe("2.2", "text2img")
    la = _twice(pipe, "generate_text2img", "a red cat", batch_size=2, decoder_steps=6, **kw)
    lo = _twice(pipe, "generate_text2img", "a red cat", batch_size=2, decoder_steps=6, **dict(kw, sampler="dpmpp_2m_sampler"))
    assert not torch.equal(la, lo) and not torch.equal(la[0], la[1])
    _twice(pipe, "mix_images", ["a cat", "a dog"], [0.3, 0.7], batch_size=1, decoder_steps=5, **kw)
    src = Image.fromarray((np.random.default_rng(0).random((70, 90, 3)) * 255).astype("uint8"))
    _twice(_pipe("2.2", "img2img"), "generate_img2img", "a dog", src, strength=0.5, batch_size=1, decoder_steps=6, **kw)
    lat = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(0))
    mask = torch.ones(64, 64)
    mask[:, 40:] = 0
    li = _twice(_pipe("2.2", "inpainting"), "generate_inpainting", "a hat", lat, mask.numpy(), batch_size=2, decoder_steps=5,
                **kw)
    keep = torch.nn.functional.interpolate(mask[None, None], (8, 8), mode="nearest").bool().expand(2, 4, 8, 8).cuda()
    assert torch.equal(li[keep], lat.cuda().expand(2, 4, 8, 8)[keep])   # the kept region IS the encoded latent
    hint = torch.rand(1, 3, 64, 64, generator=torch.Generator().manual_seed(3))
    _twice(_pipe("2.2", "controlnet"), "generate_controlnet", "a red cat", hint, batch_size=2, decoder_steps=4, **kw)


# ---- full size -----------------------------------------------------------------------------------------------------------
def test_full_size_cfg2_unipc_matches_oracle():
    """Full-size 2.2 decoder at the cfg-2 geometry (4 images, 96x96 latents, guidance 4), 10 UniPC steps through the step graph
    vs the oracle loop with the fp32 oracle UNet: finite and within the tiny-loop bounds."""
    from kandinsky2.model.gaussian_diffusion import UniPCSchedule
    from oracle import unet_oracle as uo_net
    from tests import test_gpu_unet as tu
    _no_tf32()
    m = tu._full_model()
    B, n, gs = 4, 10, 4.0
    g = torch.Generator(device="cuda").manual_seed(47)
    x_T = torch.randn(B, 4, 96, 96, device="cuda", generator=g)
    img = torch.randn(2 * B, 1280, device="cuda", generator=g)
    sch = UniPCSchedule(_ac22(), n)
    m.del_cache()
    out = sch.sample(m, (2 * B, 4, 96, 96), noise=torch.cat([x_T, x_T]), model_kwargs=dict(image_emb=img), guidance_scale=gs,
                     cond_first=False, device="cuda")[:B].clone()
    m.del_cache()
    assert torch.isfinite(out).all()
    sd = tu._sd_as_stored(tu._full_sd())

    def eps(x, k):
        mo = uo_net.unet_forward(sd, uo_net.CONFIG_2_2, torch.cat([x, x]),
                                 torch.full((2 * B,), float(sch.timesteps[k]), device="cuda"), image_emb=img)
        return mo[:B, :4] + gs * (mo[B:, :4] - mo[:B, :4])

    with torch.no_grad():
        ref = uo.solve(eps, x_T.clone(), sch.alphas, sch.sigmas)
    err = (out - ref).abs().max().item()
    rel = ((out - ref).norm() / ref.norm()).item()
    print(f"full size cfg-2, 10 UniPC steps: rel L2 {rel:.3e}, max abs {err:.3e}")
    del sd, ref
    torch.cuda.empty_cache()
    assert rel < 2e-2 and err < 0.15 * out.abs().max().item(), (err, rel)
