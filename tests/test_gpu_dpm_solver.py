"""GPU: the DPM-Solver++(2M) sampler -- k2_dpm_solver_step against a float64 evaluation of its formula, the analytic Gaussian
problem solved step by step through the kernel, the graph-replayed loop against the float64 oracle loop driven by the fp32
oracle UNet (tests/dpm_oracle.py), and the pipelines' sampler="dpmpp_2m_sampler" surface.  Tolerances are stated per test."""
import os

import numpy as np
import pytest
import torch

from tests import dpm_oracle as do

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")
MU, S = 0.3, 0.5


def _ac22():
    from kandinsky2.model.gaussian_diffusion import create_ddpm_v22
    return create_ddpm_v22(50).base_alphas_cumprod


def _no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


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


# ---- tiny-UNet trajectories ----------------------------------------------------------------------------------------------
def _traj_tiny():
    from oracle import synth, unet_oracle as uo
    from tests.test_gpu_unet import _build
    fx = torch.load(os.path.join(GOLD, "traj_tiny.pt"), weights_only=False)
    sd = synth.synth_state_dict(uo.unet_param_spec(fx["cfg"]), seed=fx["weight_seed"])
    return fx, sd, _build(fx["cfg"], sd)


def _base21():
    from kandinsky2.configs import CONFIG_2_1
    from kandinsky2.model.gaussian_diffusion import create_gaussian_diffusion
    return create_gaussian_diffusion(**CONFIG_2_1["diffusion_config"]).base_alphas_cumprod


def test_loop_21_head_matches_oracle():
    """2.1 head (cond rows first), 5 DPM++ steps at guidance 3 through the graph-replayed FusedStep loop vs the float64-form
    oracle loop driven by the fp32 oracle UNet.  The first step's x0 = (x - sigma eps) / alpha has 1/alpha ~ 14.6 at
    t = 999 and guidance 3 on top, which amplifies the UNet's fp16 error as in the DDIM loop test: same bounds."""
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule
    from oracle import unet_oracle as uo
    fx, sd, m = _traj_tiny()
    cfg = fx["cfg"]
    x_T = fx["x_T"].cuda()
    B = x_T.shape[0]
    kw = {k: v.cuda() for k, v in fx["cond"].items()}
    n, gs = 5, 3.0
    ac = _base21()
    out = DPMSolverSchedule(ac, n).sample(m, (2 * B, 4, 16, 16), noise=torch.cat([x_T, x_T]), model_kwargs=kw,
                                          guidance_scale=gs, cond_first=True, device="cuda")[:B]
    tau, alpha, sigma = do.grid(ac, n)
    sdc = {k: v.cuda() for k, v in sd.items()}

    def eps(x, k):
        mo = uo.unet_forward(sdc, cfg, torch.cat([x, x]), torch.full((2 * B,), float(tau[k]), device="cuda"), **kw)
        return mo[B:, :4] + gs * (mo[:B, :4] - mo[B:, :4])

    with torch.no_grad():
        ref = do.solve(eps, x_T.clone(), alpha, sigma)
    err = (out - ref).abs().max().item()
    rel = ((out - ref).norm() / ref.norm()).item()
    print(f"2.1 head, 5 DPM++ steps: rel L2 {rel:.3e}, max abs {err:.3e}")
    assert torch.isfinite(out).all()
    assert rel < 2e-2 and err < 0.15 * ref.abs().max().item(), (err, rel, ref.abs().max().item())


@pytest.mark.parametrize("inpaint", [False, True])
def test_loop_22_head_matches_oracle(inpaint):
    """2.2 order (unconditional rows first), the model and oracle forward of the 2.2 DDPM loop test, 6 DPM++ steps at guidance
    4, with and without the renoise inpainting rule.  Same bounds as above (the solver has no clamp); with inpainting the kept
    region of the result is exactly the clean latent."""
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
    extra, oinp = {}, None
    if inpaint:
        init = torch.randn(1, 4, H, W, generator=g)
        mask = (torch.rand(1, 1, H, W, generator=g) > 0.4).float()
        kw["inpaint_image"] = (init * mask).repeat(2 * B, 1, 1, 1)
        kw["inpaint_mask"] = mask.repeat(2 * B, 1, 1, 1)
        extra = dict(inpaint_init=init.repeat(B, 1, 1, 1).cuda(), inpaint_mask=mask.repeat(B, 1, 1, 1).cuda(),
                     inpaint_renoise=True)
        oinp = (init, mask, x_T)
    ac = _ac22()
    out = DPMSolverSchedule(ac, n).sample(m, (2 * B, 4, H, W), noise=torch.cat([x_T, x_T]).cuda(),
                                          model_kwargs={k: v.cuda() for k, v in kw.items()}, guidance_scale=gs,
                                          cond_first=False, device="cuda", **extra)[:B].cpu()
    tau, alpha, sigma = do.grid(ac, n)

    def eps(x, k):
        mo = uo.unet_forward(sd, cfg, torch.cat([x, x]), torch.full((2 * B,), float(tau[k])), **kw)
        return mo[:B, :4] + gs * (mo[B:, :4] - mo[:B, :4])

    with torch.no_grad():
        ref = do.solve(eps, x_T.clone(), alpha, sigma, inpaint=oinp)
    err = (out - ref).abs().max().item()
    rel = ((out - ref).norm() / ref.norm()).item()
    print(f"2.2 head, inpaint={inpaint}, 6 DPM++ steps: rel L2 {rel:.3e}, max abs {err:.3e}")
    assert rel < 2e-2 and err < 0.15 * ref.abs().max().item(), (err, rel)
    if inpaint:
        keep = mask.bool().expand(B, 4, H, W)
        assert torch.equal(out[keep], init.expand(B, 4, H, W)[keep])


def test_graph_replay_equals_step_at_a_time():
    """The graph-replayed loop and the same steps issued one at a time (FusedStep.run, eager UNet plan) give bit-identical
    latents; so does a second graph-replayed run (the history buffer is reset by set_schedule)."""
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule, FusedStep
    fx, _, m = _traj_tiny()
    x_T = fx["x_T"].cuda()
    B = x_T.shape[0]
    kw = {k: v.cuda() for k, v in fx["cond"].items()}
    sch = DPMSolverSchedule(_base21(), 6)
    shape = (2 * B, 4, 16, 16)
    a = sch.sample(m, shape, noise=torch.cat([x_T, x_T]), model_kwargs=kw, guidance_scale=3.0, cond_first=True, device="cuda")[:B]
    b = sch.sample(m, shape, noise=torch.cat([x_T, x_T]), model_kwargs=kw, guidance_scale=3.0, cond_first=True, device="cuda")[:B]
    coef, ts = sch._tables(torch.device("cuda"))
    m.use_cuda_graph = False
    try:
        step = FusedStep(m, B, 16, 16, kw, 3.0, True, 1e30, 0, step_kind="dpmpp_2m")
        step.st["hist"].fill_(float("nan"))
        x = x_T.clone()
        for j in range(sch.num_timesteps)[::-1]:
            step.run(x, ts[j], coef[j])
    finally:
        m.use_cuda_graph = True
    assert torch.equal(a, b)
    assert torch.equal(a, x)


def test_full_size_cfg2_matches_oracle():
    """Full-size 2.2 decoder at the cfg-2 geometry (4 images, 96x96 latents, guidance 4), 20 DPM++ steps through the step
    graph vs the oracle loop with the fp32 oracle UNet on the GPU: finite and within the tiny-model trajectory bounds."""
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule
    from oracle import unet_oracle as uo
    from tests import test_gpu_unet as tu
    _no_tf32()
    m = tu._full_model()
    B, n, gs = 4, 20, 4.0
    g = torch.Generator(device="cuda").manual_seed(41)
    x_T = torch.randn(B, 4, 96, 96, device="cuda", generator=g)
    img = torch.randn(2 * B, 1280, device="cuda", generator=g)
    ac = _ac22()
    m.del_cache()
    out = DPMSolverSchedule(ac, n).sample(m, (2 * B, 4, 96, 96), noise=torch.cat([x_T, x_T]), model_kwargs=dict(image_emb=img),
                                          guidance_scale=gs, cond_first=False, device="cuda")[:B].clone()
    m.del_cache()
    assert torch.isfinite(out).all()
    tau, alpha, sigma = do.grid(ac, n)
    sd = tu._sd_as_stored(tu._full_sd())

    def eps(x, k):
        mo = uo.unet_forward(sd, uo.CONFIG_2_2, torch.cat([x, x]), torch.full((2 * B,), float(tau[k]), device="cuda"),
                             image_emb=img)
        return mo[:B, :4] + gs * (mo[B:, :4] - mo[:B, :4])

    with torch.no_grad():
        ref = do.solve(eps, x_T.clone(), alpha, sigma)
    err = (out - ref).abs().max().item()
    rel = ((out - ref).norm() / ref.norm()).item()
    print(f"full size cfg-2, 20 DPM++ steps: rel L2 {rel:.3e}, max abs {err:.3e}")
    del sd, ref
    torch.cuda.empty_cache()
    assert rel < 2e-2 and err < 0.15 * out.abs().max().item(), (err, rel)


# ---- pipelines -----------------------------------------------------------------------------------------------------------
# With the random weights of the tiny configs the DPM++ latents (no clamp on this path) reach magnitudes that saturate the MoVQ
# decoder to black images, so these tests compare the denoised latents handed to the decoder, and the images where they must
# be identical.
def _pipe(version, task):
    from kandinsky2 import get_kandinsky2
    from tests.test_gpu_movq_sampler import _tiny_overrides
    pipe = get_kandinsky2("cuda", task_type=task, model_version=version, cache_dir="/nonexistent",
                          config_overrides=_tiny_overrides())
    pipe.seen = []
    orig = pipe._finish

    def finish(latents, h, w):
        pipe.seen.append(latents.clone())
        return orig(latents, h, w)
    pipe._finish = finish
    return pipe


def _run(pipe, method, *args, **kw):
    """-> (images, the latents the call decoded)"""
    imgs = getattr(pipe, method)(*args, **kw)
    return imgs, pipe.seen[-1]


def _same(a, b):
    return len(a) == len(b) and all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


def test_pipeline_21_dpm():
    dpm = dict(sampler="dpmpp_2m_sampler", h=64, w=64)
    pipe = _pipe("2.1", "text2img")
    base, lbase = _run(pipe, "generate_text2img", "a red cat", num_steps=10, batch_size=1, h=64, w=64)   # default (DDIM)
    a, la = _run(pipe, "generate_text2img", "a red cat", num_steps=8, batch_size=2, guidance_scale=4, **dpm)
    b, lb = _run(pipe, "generate_text2img", "a red cat", num_steps=8, batch_size=2, guidance_scale=4, **dpm)
    _, lc = _run(pipe, "generate_text2img", "a blue dog", num_steps=8, batch_size=2, guidance_scale=4, **dpm)
    assert len(a) == 2 and a[0].size == (64, 64) and a[0].mode == "RGB"
    assert torch.isfinite(la).all() and _same(a, b) and torch.equal(la, lb)
    assert not torch.equal(la, lc) and not torch.equal(la[0], la[1])
    mixed, _ = _run(pipe, "mix_images", ["a cat", "a dog"], [0.3, 0.7], num_steps=5, batch_size=1, **dpm)
    assert len(mixed) == 1 and mixed[0].size == (64, 64)
    again, lagain = _run(pipe, "generate_text2img", "a red cat", num_steps=10, batch_size=1, h=64, w=64)
    assert _same(base, again) and torch.equal(lbase, lagain)   # the DDIM call is untouched by the DPM++ calls between
    from PIL import Image
    src = Image.fromarray((np.random.default_rng(0).random((70, 90, 3)) * 255).astype("uint8"))
    i2i = _pipe("2.1", "img2img")
    o1, l1 = _run(i2i, "generate_img2img", "a dog", src, strength=0.6, num_steps=10, batch_size=1, **dpm)
    o2, l2 = _run(i2i, "generate_img2img", "a dog", src, strength=0.6, num_steps=10, batch_size=1, **dpm)
    o3, l3 = _run(i2i, "generate_img2img", "a dog", src, strength=0.05, num_steps=10, batch_size=1, **dpm)  # keeps 1 step
    assert o1[0].size == (64, 64) and _same(o1, o2) and torch.equal(l1, l2) and not torch.equal(l1, l3)
    inp = _pipe("2.1", "inpainting")
    lat = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(0))
    mask = torch.ones(64, 64)
    mask[:, 40:] = 0
    p1, m1 = _run(inp, "generate_inpainting", "a hat", lat, mask.numpy(), num_steps=6, batch_size=1, guidance_scale=4, **dpm)
    p2, m2 = _run(inp, "generate_inpainting", "a hat", lat, mask.numpy(), num_steps=6, batch_size=1, guidance_scale=4, **dpm)
    assert p1[0].size == (64, 64) and _same(p1, p2) and torch.equal(m1, m2) and torch.isfinite(m1).all()


def test_pipeline_22_dpm():
    dpm = dict(sampler="dpmpp_2m_sampler", h=64, w=64)
    pipe = _pipe("2.2", "text2img")
    base, lbase = _run(pipe, "generate_text2img", "a red cat", batch_size=2, decoder_steps=4, h=64, w=64)  # default (DDPM)
    a, la = _run(pipe, "generate_text2img", "a red cat", batch_size=2, decoder_steps=6, **dpm)
    b, lb = _run(pipe, "generate_text2img", "a red cat", batch_size=2, decoder_steps=6, **dpm)
    _, lc = _run(pipe, "generate_text2img", "a blue dog", batch_size=2, decoder_steps=6, **dpm)
    assert len(a) == 2 and a[0].size == (64, 64)
    assert torch.isfinite(la).all() and _same(a, b) and torch.equal(la, lb) and not torch.equal(la, lc)
    again, lagain = _run(pipe, "generate_text2img", "a red cat", batch_size=2, decoder_steps=4, h=64, w=64)
    assert _same(base, again) and torch.equal(lbase, lagain)   # the DDPM call is untouched by the DPM++ calls between
    mixed, _ = _run(pipe, "mix_images", ["a cat", "a dog"], [0.3, 0.7], batch_size=1, decoder_steps=5, **dpm)
    assert len(mixed) == 1
    i2i = _pipe("2.2", "img2img")
    from PIL import Image
    src = Image.fromarray((np.random.default_rng(0).random((70, 90, 3)) * 255).astype("uint8"))
    o1, l1 = _run(i2i, "generate_img2img", "a dog", src, strength=0.5, batch_size=1, decoder_steps=6, **dpm)
    o2, l2 = _run(i2i, "generate_img2img", "a dog", src, strength=0.5, batch_size=1, decoder_steps=6, **dpm)
    assert o1[0].size == (64, 64) and _same(o1, o2) and torch.equal(l1, l2)
    inp = _pipe("2.2", "inpainting")
    lat = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(0))
    mask = torch.ones(64, 64)
    mask[:, 40:] = 0
    d0, ld0 = _run(inp, "generate_inpainting", "a hat", lat, mask.numpy(), batch_size=2, decoder_steps=4, h=64, w=64)
    p1, m1 = _run(inp, "generate_inpainting", "a hat", lat, mask.numpy(), batch_size=2, decoder_steps=5, **dpm)
    p2, m2 = _run(inp, "generate_inpainting", "a dog", lat, mask.numpy(), batch_size=2, decoder_steps=5, **dpm)
    assert p1[0].size == (64, 64) and not torch.equal(m1, m2)
    keep = torch.nn.functional.interpolate(mask[None, None], (8, 8), mode="nearest").bool().expand(2, 4, 8, 8).cuda()
    for out in (m1, m2):
        assert torch.equal(out[keep], lat.cuda().expand(2, 4, 8, 8)[keep])   # the kept region IS the encoded latent
    d1, ld1 = _run(inp, "generate_inpainting", "a hat", lat, mask.numpy(), batch_size=2, decoder_steps=4, h=64, w=64)
    assert _same(d0, d1) and torch.equal(ld0, ld1)
    cn = _pipe("2.2", "controlnet")
    hint = torch.rand(1, 3, 64, 64, generator=torch.Generator().manual_seed(3))
    h1, k1 = _run(cn, "generate_controlnet", "a red cat", hint, batch_size=2, decoder_steps=4, **dpm)
    h2, k2 = _run(cn, "generate_controlnet", "a red cat", hint, batch_size=2, decoder_steps=4, **dpm)
    _, k3 = _run(cn, "generate_controlnet", "a red cat", 1.0 - hint, batch_size=2, decoder_steps=4, **dpm)
    assert _same(h1, h2) and torch.equal(k1, k2) and not torch.equal(k1, k3)
