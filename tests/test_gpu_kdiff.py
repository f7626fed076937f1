"""GPU: the sigma-space samplers -- k2_heun_step against a float64 evaluation of its formula on views inside NaN-poisoned memory,
stages that leave operands unread run on NaN, graph-replayed tiny-UNet loops of every Euler / Heun name against diffusers'
schedulers restated in tests/kdiff_oracle.py and driven by the fp32 oracle UNet, graph replay against step-at-a-time execution,
every pipeline method with a new name, and full-size cfg-2 runs of Heun and Euler ancestral.  The loop bounds are those of
tests/test_gpu_unipc.py."""
import numpy as np
import pytest
import torch

from tests import kdiff_oracle as ko
from tests.test_cpu_kdiff import KINDS, _schedule
from tests.test_gpu_dpm_solver import _ac22, _base21, _no_tf32, _pipe, _traj_tiny
from tests.test_gpu_unipc import _check, _twice

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


# ---- tiny-UNet trajectories ----------------------------------------------------------------------------------------------


@pytest.mark.parametrize("name", list(KINDS))
def test_loop_21_head_matches_oracle(name):
    """2.1 head (cond rows first), 5 steps at guidance 3 through the graph-replayed loop (Heun: 9 evaluations) vs diffusers'
    scheduler loop restated in kdiff_oracle, driven by the fp32 oracle UNet, from the same unit noise (and Euler ancestral's
    same per-step draws)."""
    from oracle import unet_oracle as uo_net
    fx, sd, m = _traj_tiny()
    cfg = fx["cfg"]
    z = fx["x_T"].cuda()
    B = z.shape[0]
    kw = {k: v.cuda() for k, v in fx["cond"].items()}
    n, gs = 5, 3.0
    sch = _schedule(name, _base21(), n)
    kind, karras = KINDS[name][:2]
    step_noise = None
    if sch.draws_noise:
        step_noise = torch.randn(sch.num_timesteps, B, 4, 16, 16, device="cuda", generator=torch.Generator("cuda").manual_seed(2))
    x0 = sch.init_noise_scale * z
    out = sch.sample(m, (2 * B, 4, 16, 16), noise=torch.cat([x0, x0]), model_kwargs=kw, guidance_scale=gs, cond_first=True,
                     device="cuda", step_noise=step_noise)[:B]
    sdc = {k: v.cuda() for k, v in sd.items()}

    def eps(x, t):
        mo = uo_net.unet_forward(sdc, cfg, torch.cat([x, x]), torch.full((2 * B,), float(t), device="cuda"), **kw)
        return mo[B:, :4] + gs * (mo[:B, :4] - mo[B:, :4])

    with torch.no_grad():
        ref = ko.sample(kind, eps, _base21(), n, z.clone(), karras=karras, step_noise=step_noise)
    _check(out, ref, f"2.1 head, {name}")


@pytest.mark.parametrize("inpaint", [False, True])
@pytest.mark.parametrize("name", list(KINDS))
def test_loop_22_head_matches_oracle(name, inpaint):
    """2.2 order (unconditional rows first), 6 steps at guidance 4, with and without the renoise inpainting rule, vs the oracle
    loop; with inpainting the kept region of the result is exactly the clean latent."""
    from oracle import synth, unet_oracle as uo_net
    from tests.test_gpu_unet import _build
    cfg = dict(uo_net.CONFIG_TINY, inpainting=inpaint)
    sd = synth.synth_state_dict(uo_net.unet_param_spec(cfg), seed=4)
    m = _build(cfg, sd)
    g = torch.Generator().manual_seed(8)
    B, H, W, n, gs = 2, 16, 16, 6, 4.0
    z = torch.randn(B, 4, H, W, generator=g)
    kw = dict(full_emb=torch.randn(2 * B, 7, 96, generator=g), pooled_emb=torch.randn(2 * B, 48, generator=g),
              image_emb=torch.randn(2 * B, 48, generator=g))
    sch = _schedule(name, _ac22(), n)
    kind, karras = KINDS[name][:2]
    step_noise = torch.randn(sch.num_timesteps, B, 4, H, W, generator=g) if sch.draws_noise else None
    extra, oinp = {}, None
    if inpaint:
        init = torch.randn(1, 4, H, W, generator=g)
        mask = (torch.rand(1, 1, H, W, generator=g) > 0.4).float()
        kw["inpaint_image"] = (init * mask).repeat(2 * B, 1, 1, 1)
        kw["inpaint_mask"] = mask.repeat(2 * B, 1, 1, 1)
        extra = dict(inpaint_init=init.repeat(B, 1, 1, 1).cuda(), inpaint_mask=mask.repeat(B, 1, 1, 1).cuda(),
                     inpaint_renoise=True)
        oinp = (init, mask)
    x0 = sch.init_noise_scale * z
    out = sch.sample(m, (2 * B, 4, H, W), noise=torch.cat([x0, x0]).cuda(), model_kwargs={k: v.cuda() for k, v in kw.items()},
                     guidance_scale=gs, cond_first=False, device="cuda",
                     step_noise=None if step_noise is None else step_noise.cuda(), **extra)[:B].cpu()

    def eps(x, t):
        mo = uo_net.unet_forward(sd, cfg, torch.cat([x, x]), torch.full((2 * B,), float(t)), **kw)
        return mo[:B, :4] + gs * (mo[B:, :4] - mo[:B, :4])

    with torch.no_grad():
        ref = ko.sample(kind, eps, _ac22(), n, z.clone(), karras=karras, step_noise=step_noise, inpaint=oinp)
    _check(out, ref, f"2.2 head, {name}, inpaint={inpaint}")
    if inpaint:
        keep = mask.bool().expand(B, 4, H, W)
        assert torch.equal(out[keep], init.expand(B, 4, H, W)[keep])


@pytest.mark.parametrize("name", list(KINDS))
def test_graph_replay_equals_step_at_a_time(name):
    """The graph-replayed loop and the same evaluations issued one at a time (FusedStep.run with each row, eager UNet plan,
    NaN-filled state buffers, Euler ancestral's noise copied in per step) give bit-identical latents; so does a second
    graph-replayed run (set_schedule resets the state)."""
    from kandinsky2.model.gaussian_diffusion import FusedStep
    fx, _, m = _traj_tiny()
    z = fx["x_T"].cuda()
    B = z.shape[0]
    kw = {k: v.cuda() for k, v in fx["cond"].items()}
    sch = _schedule(name, _base21(), 6)
    nz = None
    if sch.draws_noise:
        nz = torch.randn(sch.num_timesteps, B, 4, 16, 16, device="cuda", generator=torch.Generator("cuda").manual_seed(4))
    x0 = sch.init_noise_scale * z
    run = lambda: sch.sample(m, (2 * B, 4, 16, 16), noise=torch.cat([x0, x0]), model_kwargs=kw, guidance_scale=3.0,
                             cond_first=True, device="cuda", step_noise=nz)[:B].clone()
    a, b = run(), run()
    coef, ts = sch._tables(torch.device("cuda"))
    m.use_cuda_graph = False
    try:
        step = FusedStep(m, B, 16, 16, kw, 3.0, True, 1e30, 0, step_kind=sch.step_kind)
        for key in ("hist", "heun_x", "heun_d"):
            if step.st.get(key) is not None:
                step.st[key].fill_(float("nan"))
        x = x0.clone()
        for i, j in enumerate(range(sch.num_timesteps)[::-1]):
            if nz is not None:
                step.noise.copy_(nz[i])
            step.run(x, ts[j], coef[j])
    finally:
        m.use_cuda_graph = True
    assert torch.equal(a, b) and torch.equal(a, x) and torch.isfinite(a).all()


# ---- pipelines -----------------------------------------------------------------------------------------------------------
def test_pipelines_21_each_method():
    """Every 2.1 method runs end to end with a new name, deterministically; Heun img2img keeps int(N * strength) steps."""
    from PIL import Image
    pipe = _pipe("2.1", "text2img")
    la = _twice(pipe, "generate_text2img", "a red cat", num_steps=5, batch_size=2, guidance_scale=4, h=64, w=64,
                sampler="heun_sampler")
    lb = _twice(pipe, "generate_text2img", "a red cat", num_steps=5, batch_size=2, guidance_scale=4, h=64, w=64,
                sampler="euler_sampler")
    assert not torch.equal(la, lb) and not torch.equal(la[0], la[1])
    _twice(pipe, "mix_images", ["a cat", "a dog"], [0.3, 0.7], num_steps=5, batch_size=1, h=64, w=64,
           sampler="euler_ancestral_sampler")
    emb = torch.cat([pipe.embedder.image_emb("a cat", 1), pipe.embedder.zero_image_emb(1)])
    _twice(pipe, "generate_img", "a cat", emb, batch_size=1, guidance_scale=4, num_steps=5, h=64, w=64,
           diffusion=pipe._diffusion("euler_karras_sampler", 5), sampler="euler_karras_sampler")
    src = Image.fromarray((np.random.default_rng(0).random((70, 90, 3)) * 255).astype("uint8"))
    _twice(_pipe("2.1", "img2img"), "generate_img2img", "a dog", src, strength=0.6, num_steps=8, batch_size=1, h=64, w=64,
           sampler="heun_karras_sampler")
    lat = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(0))
    mask = torch.ones(64, 64)
    mask[:, 40:] = 0
    _twice(_pipe("2.1", "inpainting"), "generate_inpainting", "a hat", lat, mask.numpy(), num_steps=5, batch_size=1,
           guidance_scale=4, h=64, w=64, sampler="heun_sampler")


def test_pipelines_22_each_method():
    """Every 2.2 method runs end to end with a new name, deterministically; inpainting keeps the encoded latent exactly."""
    from PIL import Image
    pipe = _pipe("2.2", "text2img")
    la = _twice(pipe, "generate_text2img", "a red cat", batch_size=2, decoder_steps=5, h=64, w=64, sampler="heun_karras_sampler")
    assert not torch.equal(la[0], la[1])
    _twice(pipe, "mix_images", ["a cat", "a dog"], [0.3, 0.7], batch_size=1, decoder_steps=5, h=64, w=64,
           sampler="euler_karras_sampler")
    src = Image.fromarray((np.random.default_rng(0).random((70, 90, 3)) * 255).astype("uint8"))
    _twice(_pipe("2.2", "img2img"), "generate_img2img", "a dog", src, strength=0.5, batch_size=1, decoder_steps=6, h=64, w=64,
           sampler="heun_sampler")
    lat = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(0))
    mask = torch.ones(64, 64)
    mask[:, 40:] = 0
    li = _twice(_pipe("2.2", "inpainting"), "generate_inpainting", "a hat", lat, mask.numpy(), batch_size=2, decoder_steps=5,
                h=64, w=64, sampler="euler_ancestral_sampler")
    keep = torch.nn.functional.interpolate(mask[None, None], (8, 8), mode="nearest").bool().expand(2, 4, 8, 8).cuda()
    assert torch.equal(li[keep], lat.cuda().expand(2, 4, 8, 8)[keep])
    hint = torch.rand(1, 3, 64, 64, generator=torch.Generator().manual_seed(3))
    cn = _pipe("2.2", "controlnet")
    _twice(cn, "generate_controlnet", "a red cat", hint, batch_size=2, decoder_steps=4, h=64, w=64, sampler="euler_sampler")
    _twice(cn, "generate_controlnet_img2img", "a red cat", src, hint, strength=0.5, batch_size=1, decoder_steps=6, h=64, w=64,
           sampler="heun_karras_sampler")


# ---- full size -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,n", [("heun_sampler", 6), ("euler_ancestral_sampler", 10)])
def test_full_size_cfg2_matches_oracle(name, n):
    """Full-size 2.2 decoder at the cfg-2 geometry (4 images, 96x96 latents, guidance 4) through the step graph (Heun: 11
    evaluations) vs the oracle loop with the fp32 oracle UNet: finite and within the tiny-loop bounds."""
    from oracle import unet_oracle as uo_net
    from tests import test_gpu_unet as tu
    _no_tf32()
    m = tu._full_model()
    B, gs = 4, 4.0
    g = torch.Generator(device="cuda").manual_seed(53)
    z = torch.randn(B, 4, 96, 96, device="cuda", generator=g)
    img = torch.randn(2 * B, 1280, device="cuda", generator=g)
    sch = _schedule(name, _ac22(), n)
    kind, karras = KINDS[name][:2]
    nz = torch.randn(sch.num_timesteps, B, 4, 96, 96, device="cuda", generator=g) if sch.draws_noise else None
    x0 = sch.init_noise_scale * z
    m.del_cache()
    out = sch.sample(m, (2 * B, 4, 96, 96), noise=torch.cat([x0, x0]), model_kwargs=dict(image_emb=img), guidance_scale=gs,
                     cond_first=False, device="cuda", step_noise=nz)[:B].clone()
    m.del_cache()
    assert torch.isfinite(out).all()
    sd = tu._sd_as_stored(tu._full_sd())

    def eps(x, t):
        mo = uo_net.unet_forward(sd, uo_net.CONFIG_2_2, torch.cat([x, x]), torch.full((2 * B,), float(t), device="cuda"),
                                 image_emb=img)
        return mo[:B, :4] + gs * (mo[B:, :4] - mo[:B, :4])

    with torch.no_grad():
        ref = ko.sample(kind, eps, _ac22(), n, z.clone(), karras=karras, step_noise=nz)
    err = (out - ref).abs().max().item()
    rel = ((out - ref).norm() / ref.norm()).item()
    print(f"full size cfg-2, {name} x {n}: rel L2 {rel:.3e}, max abs {err:.3e}")
    del sd, ref
    torch.cuda.empty_cache()
    assert rel < 2e-2 and err < 0.15 * out.abs().max().item(), (err, rel)
