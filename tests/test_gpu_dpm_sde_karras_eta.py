"""GPU: the DPM-Solver++(2M) SDE step, Karras spacing and DDIM with eta > 0 -- k2_dpm_solver_sde_step against a float64
evaluation of its formula, the Gaussian SDE loop through the kernel, graph-replayed tiny-UNet loops against the float64 oracle
loops (tests/dpm_oracle.py, tests/dpm_sde_oracle.py) driven by the fp32 oracle UNet with the same injected noise, DDIM eta = 0.5
against the reference's own sampler (tests/golden/ddim_eta_tiny.pt), and the pipelines' new sampler names.  Tolerances are
stated per test; the loop bounds are those of tests/test_gpu_dpm_solver.py."""
import os

import numpy as np
import pytest
import torch

from tests import dpm_oracle as do
from tests import dpm_sde_oracle as so
from tests.test_gpu_dpm_solver import _ac22, _base21, _no_tf32, _pipe, _run, _same, _traj_tiny

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
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


# ---- tiny-UNet trajectories ----------------------------------------------------------------------------------------------
VARIANTS = [("linspace", True), ("karras", False), ("karras", True)]


def _oracle_loop(eps, x_T, sch, step_noise, inpaint=None):
    if sch.sde:
        return so.solve_sde(eps, x_T.clone(), sch.alphas, sch.sigmas, step_noise, inpaint=inpaint)
    return do.solve(eps, x_T.clone(), sch.alphas, sch.sigmas, inpaint=inpaint)


def _check(out, ref, what):
    err = (out - ref).abs().max().item()
    rel = ((out - ref).norm() / ref.norm()).item()
    print(f"{what}: rel L2 {rel:.3e}, max abs {err:.3e}")
    assert torch.isfinite(out).all()
    assert rel < 2e-2 and err < 0.15 * ref.abs().max().item(), (what, err, rel, ref.abs().max().item())


@pytest.mark.parametrize("spacing,sde", VARIANTS)
def test_loop_21_head_matches_oracle(spacing, sde):
    """2.1 head (cond rows first), 5 steps at guidance 3 through the graph-replayed loop vs the float64-form oracle loop driven
    by the fp32 oracle UNet at the same (fractional, for Karras) timesteps, with the same injected noise."""
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule
    from oracle import unet_oracle as uo
    fx, sd, m = _traj_tiny()
    cfg = fx["cfg"]
    x_T = fx["x_T"].cuda()
    B = x_T.shape[0]
    kw = {k: v.cuda() for k, v in fx["cond"].items()}
    n, gs = 5, 3.0
    sch = DPMSolverSchedule(_base21(), n, spacing=spacing, sde=sde)
    z = torch.randn(n, B, 4, 16, 16, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    out = sch.sample(m, (2 * B, 4, 16, 16), noise=torch.cat([x_T, x_T]), model_kwargs=kw, guidance_scale=gs, cond_first=True,
                     device="cuda", step_noise=z)[:B]
    sdc = {k: v.cuda() for k, v in sd.items()}

    def eps(x, k):
        mo = uo.unet_forward(sdc, cfg, torch.cat([x, x]), torch.full((2 * B,), float(sch.timesteps[k]), device="cuda"), **kw)
        return mo[B:, :4] + gs * (mo[:B, :4] - mo[B:, :4])

    with torch.no_grad():
        ref = _oracle_loop(eps, x_T, sch, z)
    _check(out, ref, f"2.1 head, {spacing}, sde={sde}")


@pytest.mark.parametrize("inpaint", [False, True])
@pytest.mark.parametrize("spacing,sde", VARIANTS)
def test_loop_22_head_matches_oracle(spacing, sde, inpaint):
    """2.2 order (unconditional rows first), 6 steps at guidance 4, with and without the renoise inpainting rule, vs the oracle
    loop with the same noise; with inpainting the kept region of the result is exactly the clean latent."""
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule
    from oracle import synth, unet_oracle as uo
    from tests.test_gpu_unet import _build
    cfg = dict(uo.CONFIG_TINY, inpainting=inpaint)
    sd = synth.synth_state_dict(uo.unet_param_spec(cfg), seed=4)
    m = _build(cfg, sd)
    g = torch.Generator().manual_seed(8)
    B, H, W, n, gs = 2, 16, 16, 6, 4.0
    x_T = torch.randn(B, 4, H, W, generator=g)
    kw = dict(full_emb=torch.randn(2 * B, 7, 96, generator=g), pooled_emb=torch.randn(2 * B, 48, generator=g),
              image_emb=torch.randn(2 * B, 48, generator=g))
    z = torch.randn(n, B, 4, H, W, generator=g)
    extra, oinp = {}, None
    if inpaint:
        init = torch.randn(1, 4, H, W, generator=g)
        mask = (torch.rand(1, 1, H, W, generator=g) > 0.4).float()
        kw["inpaint_image"] = (init * mask).repeat(2 * B, 1, 1, 1)
        kw["inpaint_mask"] = mask.repeat(2 * B, 1, 1, 1)
        extra = dict(inpaint_init=init.repeat(B, 1, 1, 1).cuda(), inpaint_mask=mask.repeat(B, 1, 1, 1).cuda(),
                     inpaint_renoise=True)
        oinp = (init, mask, x_T)
    sch = DPMSolverSchedule(_ac22(), n, spacing=spacing, sde=sde)
    out = sch.sample(m, (2 * B, 4, H, W), noise=torch.cat([x_T, x_T]).cuda(), model_kwargs={k: v.cuda() for k, v in kw.items()},
                     guidance_scale=gs, cond_first=False, device="cuda", step_noise=z.cuda(), **extra)[:B].cpu()

    def eps(x, k):
        mo = uo.unet_forward(sd, cfg, torch.cat([x, x]), torch.full((2 * B,), float(sch.timesteps[k])), **kw)
        return mo[:B, :4] + gs * (mo[B:, :4] - mo[:B, :4])

    with torch.no_grad():
        ref = _oracle_loop(eps, x_T, sch, z, inpaint=oinp)
    _check(out, ref, f"2.2 head, {spacing}, sde={sde}, inpaint={inpaint}")
    if inpaint:
        keep = mask.bool().expand(B, 4, H, W)
        assert torch.equal(out[keep], init.expand(B, 4, H, W)[keep])


@pytest.mark.parametrize("spacing", ["linspace", "karras"])
def test_sde_graph_replay_equals_step_at_a_time(spacing):
    """The graph-replayed SDE loop and the same steps issued one at a time (FusedStep.run, eager UNet plan, the noise copied in
    by hand) give bit-identical latents; so does a second graph-replayed run.  Per-image generators reproduce their draw."""
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule, FusedStep
    fx, _, m = _traj_tiny()
    x_T = fx["x_T"].cuda()
    B = x_T.shape[0]
    kw = {k: v.cuda() for k, v in fx["cond"].items()}
    sch = DPMSolverSchedule(_base21(), 6, spacing=spacing, sde=True)
    shape = (2 * B, 4, 16, 16)
    z = torch.randn(6, B, 4, 16, 16, device="cuda", generator=torch.Generator(device="cuda").manual_seed(2))
    run = lambda **k: sch.sample(m, shape, noise=torch.cat([x_T, x_T]), model_kwargs=kw, guidance_scale=3.0, cond_first=True,
                                 device="cuda", **k)[:B].clone()
    a, b = run(step_noise=z), run(step_noise=z)
    gens = lambda: [torch.Generator(device="cuda").manual_seed(100 + i) for i in range(B)]
    c, d = run(sample_generators=gens()), run(sample_generators=gens())
    coef, ts = sch._tables(torch.device("cuda"))
    m.use_cuda_graph = False
    try:
        step = FusedStep(m, B, 16, 16, kw, 3.0, True, 1e30, 0, step_kind="dpmpp_2m_sde")
        step.st["hist"].fill_(float("nan"))
        x = x_T.clone()
        for it, j in enumerate(range(sch.num_timesteps)[::-1]):
            step.noise.copy_(z[it])
            step.run(x, ts[j], coef[j])
    finally:
        m.use_cuda_graph = True
    assert torch.equal(a, b) and torch.equal(a, x)
    assert torch.equal(c, d) and not torch.equal(a, c)


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


# ---- pipelines -----------------------------------------------------------------------------------------------------------
NEW_NAMES = ("dpmpp_2m_karras_sampler", "dpmpp_2m_sde_sampler", "dpmpp_2m_sde_karras_sampler")


def _twice(pipe, method, *args, **kw):
    """-> the latents of the first of two identical calls, after checking both give bit-identical images and latents."""
    i1, l1 = _run(pipe, method, *args, **kw)
    i2, l2 = _run(pipe, method, *args, **kw)
    assert i1[0].size == (64, 64) and _same(i1, i2) and torch.equal(l1, l2) and torch.isfinite(l1).all(), (method, kw)
    return l1


@pytest.mark.parametrize("name", NEW_NAMES)
def test_pipeline_21_new_samplers(name):
    from PIL import Image
    kw = dict(sampler=name, h=64, w=64)
    pipe = _pipe("2.1", "text2img")
    la = _twice(pipe, "generate_text2img", "a red cat", num_steps=6, batch_size=2, guidance_scale=4, **kw)
    lo = _twice(pipe, "generate_text2img", "a red cat", num_steps=6, batch_size=2, guidance_scale=4,
                **dict(kw, sampler="dpmpp_2m_sampler"))
    assert not torch.equal(la, lo) and not torch.equal(la[0], la[1])
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


@pytest.mark.parametrize("name", NEW_NAMES)
def test_pipeline_22_new_samplers(name):
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
def test_full_size_cfg2_sde_matches_oracle():
    """Full-size 2.2 decoder at the cfg-2 geometry (4 images, 96x96 latents, guidance 4), 20 DPM++ 2M SDE steps through the
    step graph vs the SDE oracle loop with the fp32 oracle UNet and the same noise: finite and within the tiny-loop bounds."""
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule
    from oracle import unet_oracle as uo
    from tests import test_gpu_unet as tu
    _no_tf32()
    m = tu._full_model()
    B, n, gs = 4, 20, 4.0
    g = torch.Generator(device="cuda").manual_seed(43)
    x_T = torch.randn(B, 4, 96, 96, device="cuda", generator=g)
    img = torch.randn(2 * B, 1280, device="cuda", generator=g)
    z = torch.randn(n, B, 4, 96, 96, device="cuda", generator=g)
    sch = DPMSolverSchedule(_ac22(), n, sde=True)
    m.del_cache()
    out = sch.sample(m, (2 * B, 4, 96, 96), noise=torch.cat([x_T, x_T]), model_kwargs=dict(image_emb=img), guidance_scale=gs,
                     cond_first=False, device="cuda", step_noise=z)[:B].clone()
    m.del_cache()
    assert torch.isfinite(out).all()
    sd = tu._sd_as_stored(tu._full_sd())

    def eps(x, k):
        mo = uo.unet_forward(sd, uo.CONFIG_2_2, torch.cat([x, x]), torch.full((2 * B,), float(sch.timesteps[k]), device="cuda"),
                             image_emb=img)
        return mo[:B, :4] + gs * (mo[B:, :4] - mo[:B, :4])

    with torch.no_grad():
        ref = so.solve_sde(eps, x_T.clone(), sch.alphas, sch.sigmas, z)
    err = (out - ref).abs().max().item()
    rel = ((out - ref).norm() / ref.norm()).item()
    print(f"full size cfg-2, 20 DPM++ 2M SDE steps: rel L2 {rel:.3e}, max abs {err:.3e}")
    del sd, ref
    torch.cuda.empty_cache()
    assert rel < 2e-2 and err < 0.15 * out.abs().max().item(), (err, rel)
