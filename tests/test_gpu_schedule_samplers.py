"""GPU: what every schedule sampler (pipelines.SCHEDULE_SAMPLERS) shares -- graph-replayed tiny-UNet loops against the
float64 oracle loop of each name (tests/sampler_cases.oracle) driven by the fp32 oracle UNet, graph replay against
step-at-a-time execution, the pipeline methods with each name, and full-size cfg-2 runs.  The kernels, and what is specific
to one schedule, are tested in the per-sampler files."""
import numpy as np
import pytest
import torch

from kandinsky2.pipelines import SCHEDULE_SAMPLERS
from tests.sampler_cases import _ac22, _base21, _check, _no_tf32, _pipe, _run, _same, _schedule, _traj_tiny, oracle

pytestmark = pytest.mark.gpu
NAMES = list(SCHEDULE_SAMPLERS)
DPM = ("dpmpp_2m_sampler", "dpmpp_2m_karras_sampler", "dpmpp_2m_sde_sampler", "dpmpp_2m_sde_karras_sampler")
UNIPC = ("unipc_sampler", "unipc_karras_sampler")
# name -> the seeds of its per-step noise in the 2.1 loop and in the graph-replay test, for the names that draw noise
NOISE_SEEDS = {"dpmpp_2m_sde_sampler": (5, 2), "dpmpp_2m_sde_karras_sampler": (5, 2), "euler_ancestral_sampler": (2, 4)}


# ---- tiny-UNet trajectories ----------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,inpaint", [(n, False) for n in NAMES] + [(n, True) for n in UNIPC])
def test_loop_21_head_matches_oracle(name, inpaint):
    """2.1 head (cond rows first), 5 steps at guidance 3 through the graph-replayed loop (Heun: 9 evaluations) vs the oracle
    loop driven by the fp32 oracle UNet at the same timesteps, from the same start noise and with the same per-step draws.
    The first step's x0 = (x - sigma eps) / alpha has 1/alpha ~ 14.6 at t = 999 and guidance 3 on top, which amplifies the
    UNet's fp16 error as in the DDIM loop test: same bounds.  UniPC also with the 2.1 inpainting rule (the known region
    replaces D), after which the result's known region is exactly the clean latent."""
    from oracle import unet_oracle as uo_net
    fx, sd, m = _traj_tiny()
    cfg = fx["cfg"]
    z = fx["x_T"].cuda()
    B = z.shape[0]
    kw = {k: v.cuda() for k, v in fx["cond"].items()}
    n, gs = 5, 3.0
    sch = _schedule(name, _base21(), n)
    assert sch.draws_noise == (name in NOISE_SEEDS)
    step_noise = None
    if sch.draws_noise:
        g = torch.Generator(device="cuda").manual_seed(NOISE_SEEDS[name][0])
        step_noise = torch.randn(sch.num_timesteps, B, 4, 16, 16, device="cuda", generator=g)
    extra, oinp = {}, None
    if inpaint:
        g = torch.Generator(device="cuda").manual_seed(6)
        init = torch.randn(B, 4, 16, 16, device="cuda", generator=g)
        mask = (torch.rand(B, 1, 16, 16, device="cuda", generator=g) > 0.4).float()
        extra, oinp = dict(inpaint_init=init, inpaint_mask=mask, inpaint_renoise=False), (init, mask)
    x0 = sch.init_noise_scale * z
    out = sch.sample(m, (2 * B, 4, 16, 16), noise=torch.cat([x0, x0]), model_kwargs=kw, guidance_scale=gs, cond_first=True,
                     device="cuda", step_noise=step_noise, **extra)[:B]
    sdc = {k: v.cuda() for k, v in sd.items()}

    def eps(x, t):
        mo = uo_net.unet_forward(sdc, cfg, torch.cat([x, x]), torch.full((2 * B,), float(t), device="cuda"), **kw)
        return mo[B:, :4] + gs * (mo[:B, :4] - mo[B:, :4])

    with torch.no_grad():
        ref = oracle(name, eps, _base21(), n, z, step_noise=step_noise, inpaint=oinp, inpaint_renoise=False)
    _check(out, ref, f"2.1 head, {name}, inpaint={inpaint}")
    if inpaint:
        keep = mask.bool().expand_as(out)
        assert torch.equal(out[keep], init[keep])


@pytest.mark.parametrize("inpaint", [False, True])
@pytest.mark.parametrize("name", NAMES)
def test_loop_22_head_matches_oracle(name, inpaint):
    """2.2 order (unconditional rows first), the model and oracle forward of the 2.2 DDPM loop test, 6 steps at guidance 4,
    with and without the renoise inpainting rule, vs the oracle loop with the same per-step draws; with inpainting the kept
    region of the result is exactly the clean latent."""
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
    step_noise = None
    if sch.draws_noise or name == "dpmpp_2m_karras_sampler":   # that one ignores its draw, which keeps its inpainting inputs
        step_noise = torch.randn(sch.num_timesteps, B, 4, H, W, generator=g)
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
        ref = oracle(name, eps, _ac22(), n, z, step_noise=step_noise, inpaint=oinp)
    _check(out, ref, f"2.2 head, {name}, inpaint={inpaint}")
    if inpaint:
        keep = mask.bool().expand(B, 4, H, W)
        assert torch.equal(out[keep], init.expand(B, 4, H, W)[keep])


@pytest.mark.parametrize("name", NAMES)
def test_graph_replay_equals_step_at_a_time(name):
    """The graph-replayed loop and the same evaluations issued one at a time (FusedStep.run with each row, eager UNet plan,
    every state buffer of the step kind NaN-filled, the per-step noise copied in by hand) give bit-identical latents; so does
    a second graph-replayed run (set_schedule resets the state), with a run of another step kind between the two, which
    uses its own graph and state.  Per-image generators reproduce their draw."""
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule, FusedStep, UniPCSchedule
    fx, _, m = _traj_tiny()
    z = fx["x_T"].cuda()
    B = z.shape[0]
    kw = {k: v.cuda() for k, v in fx["cond"].items()}
    sch = _schedule(name, _base21(), 6)
    other = (DPMSolverSchedule if sch.step_kind == "unipc" else UniPCSchedule)(_base21(), 6, spacing=sch.spacing)
    nz = None
    if sch.draws_noise:
        nz = torch.randn(sch.num_timesteps, B, 4, 16, 16, device="cuda",
                         generator=torch.Generator(device="cuda").manual_seed(NOISE_SEEDS[name][1]))
    x0 = sch.init_noise_scale * z
    run = lambda s, **k: s.sample(m, (2 * B, 4, 16, 16), noise=torch.cat([x0, x0]), model_kwargs=kw, guidance_scale=3.0,
                                  cond_first=True, device="cuda", **k)[:B].clone()
    a, d1 = run(sch, step_noise=nz), run(other)
    b, d2 = run(sch, step_noise=nz), run(other)
    coef, ts = sch._tables(torch.device("cuda"))
    assert coef.shape == sch.coef_table().shape
    m.use_cuda_graph = False
    try:
        step = FusedStep(m, B, 16, 16, kw, 3.0, True, 1e30, 0, step_kind=sch.step_kind)
        for key in ("hist", "last", "hist2", "heun_x", "heun_d"):
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
    assert torch.equal(d1, d2) and not torch.equal(a, d1)
    if sch.draws_noise:
        gens = lambda: [torch.Generator(device="cuda").manual_seed(100 + i) for i in range(B)]
        c, d = run(sch, sample_generators=gens()), run(sch, sample_generators=gens())
        assert torch.equal(c, d) and not torch.equal(a, c)


# ---- pipelines -----------------------------------------------------------------------------------------------------------
def _inputs(pipe):
    from PIL import Image
    mask = torch.ones(64, 64)
    mask[:, 40:] = 0
    src = Image.fromarray((np.random.default_rng(0).random((70, 90, 3)) * 255).astype("uint8"))
    return dict(pipe=pipe, mask=mask, src=src, lat=torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(0)),
                hint=torch.rand(1, 3, 64, 64, generator=torch.Generator().manual_seed(3)))


def _emb(pipe):
    return torch.cat([pipe.embedder.image_emb("a cat", 1), pipe.embedder.zero_image_emb(1)])


# (version, task) -> [(method, its positional arguments from _inputs, its keywords, the sampler names it runs with)].  None
# is the version's default sampler (DDIM / DDPM).  Every call runs at 64x64.
PIPELINE_CALLS = {
    ("2.1", "text2img"): [
        ("generate_text2img", lambda i: ("a red cat",), dict(num_steps=10, batch_size=1), (None,)),
        ("generate_text2img", lambda i: ("a red cat",), dict(num_steps=8, batch_size=2, guidance_scale=4), DPM[:1]),
        ("generate_text2img", lambda i: ("a blue dog",), dict(num_steps=8, batch_size=2, guidance_scale=4), DPM[:1]),
        ("generate_text2img", lambda i: ("a red cat",), dict(num_steps=6, batch_size=2, guidance_scale=4), DPM + UNIPC),
        ("generate_text2img", lambda i: ("a red cat",), dict(num_steps=5, batch_size=2, guidance_scale=4),
         ("heun_sampler", "euler_sampler")),
        ("mix_images", lambda i: (["a cat", "a dog"], [0.3, 0.7]), dict(num_steps=5, batch_size=1),
         DPM + UNIPC + ("euler_ancestral_sampler",)),
        ("generate_img", lambda i: ("a cat", _emb(i["pipe"])), dict(batch_size=1, guidance_scale=4, num_steps=5),
         DPM[1:] + UNIPC + ("euler_karras_sampler",))],
    ("2.1", "img2img"): [
        ("generate_img2img", lambda i: ("a dog", i["src"]), dict(strength=0.6, num_steps=10, batch_size=1), DPM[:1]),
        ("generate_img2img", lambda i: ("a dog", i["src"]), dict(strength=0.05, num_steps=10, batch_size=1), DPM[:1]),
        ("generate_img2img", lambda i: ("a dog", i["src"]), dict(strength=0.6, num_steps=8, batch_size=1),
         DPM[1:] + UNIPC + ("heun_karras_sampler",))],
    ("2.1", "inpainting"): [
        ("generate_inpainting", lambda i: ("a hat", i["lat"], i["mask"].numpy()),
         dict(num_steps=6, batch_size=1, guidance_scale=4), DPM[:1]),
        ("generate_inpainting", lambda i: ("a hat", i["lat"], i["mask"].numpy()),
         dict(num_steps=5, batch_size=1, guidance_scale=4), DPM[1:] + UNIPC + ("heun_sampler",))],
    ("2.2", "text2img"): [
        ("generate_text2img", lambda i: ("a red cat",), dict(batch_size=2, decoder_steps=4), (None,)),
        ("generate_text2img", lambda i: ("a red cat",), dict(batch_size=2, decoder_steps=6), DPM + UNIPC),
        ("generate_text2img", lambda i: ("a blue dog",), dict(batch_size=2, decoder_steps=6), DPM[:1]),
        ("generate_text2img", lambda i: ("a red cat",), dict(batch_size=2, decoder_steps=5), ("heun_karras_sampler",)),
        ("mix_images", lambda i: (["a cat", "a dog"], [0.3, 0.7]), dict(batch_size=1, decoder_steps=5),
         DPM + UNIPC + ("euler_karras_sampler",))],
    ("2.2", "img2img"): [
        ("generate_img2img", lambda i: ("a dog", i["src"]), dict(strength=0.5, batch_size=1, decoder_steps=6),
         DPM + UNIPC + ("heun_sampler",))],
    ("2.2", "inpainting"): [
        ("generate_inpainting", lambda i: ("a hat", i["lat"], i["mask"].numpy()), dict(batch_size=2, decoder_steps=4),
         (None,)),
        ("generate_inpainting", lambda i: ("a hat", i["lat"], i["mask"].numpy()), dict(batch_size=2, decoder_steps=5),
         DPM + UNIPC + ("euler_ancestral_sampler",)),
        ("generate_inpainting", lambda i: ("a dog", i["lat"], i["mask"].numpy()), dict(batch_size=2, decoder_steps=5),
         DPM[:1])],
    ("2.2", "controlnet"): [
        ("generate_controlnet", lambda i: ("a red cat", i["hint"]), dict(batch_size=2, decoder_steps=4),
         DPM + UNIPC + ("euler_sampler",)),
        ("generate_controlnet", lambda i: ("a red cat", 1.0 - i["hint"]), dict(batch_size=2, decoder_steps=4), DPM[:1]),
        ("generate_controlnet_img2img", lambda i: ("a red cat", i["src"], i["hint"]),
         dict(strength=0.5, batch_size=1, decoder_steps=6), ("heun_karras_sampler",))],
}


@pytest.mark.parametrize("version", ["2.1", "2.2"])
@pytest.mark.parametrize("name", NAMES)
def test_pipeline_calls(name, version):
    """On each pipe the name has calls on: its calls, the same calls with their row's first name (the one the row's other
    names are compared with) and the default sampler's calls, each run twice with all the others between.  Both runs give
    the same images and latents, so a DDIM / DDPM call is untouched by the solver calls and each sampler's calls by the other
    sampler's.  64x64 RGB images, one per batch row, finite latents.  Every call's latents differ from every other call's
    (another prompt, hint, strength, step count or sampler; img2img at strength 0.05 keeps one step) and between batch rows.
    2.2 inpainting with a schedule sampler keeps the encoded latent exactly in the known region."""
    for (pipe_version, task), rows in PIPELINE_CALLS.items():
        if pipe_version != version or not any(name in names for *_, names in rows):
            continue
        pipe = _pipe(version, task)
        inputs = _inputs(pipe)
        calls = []
        for method, args, kw, names in rows:
            for sampler in dict.fromkeys(s for s in names if s is None or (name in names and s in (names[0], name))):
                k = dict(kw, h=64, w=64)
                if sampler is not None:
                    k["sampler"] = sampler
                if method == "generate_img":
                    k["diffusion"] = pipe._diffusion(sampler, kw["num_steps"])
                calls.append((method, args(inputs), k))
        first, second = ([_run(pipe, method, *args, **k) for method, args, k in calls] for _ in range(2))
        keep = torch.nn.functional.interpolate(inputs["mask"][None, None], (8, 8), mode="nearest").bool()
        keep = keep.expand(2, 4, 8, 8).cuda()
        for (method, _, k), (i1, l1), (i2, l2) in zip(calls, first, second):
            what = (task, method, k.get("sampler"), {key: v for key, v in k.items() if isinstance(v, (int, float))})
            assert _same(i1, i2) and torch.equal(l1, l2), what
            assert len(i1) == k["batch_size"] and all(im.size == (64, 64) and im.mode == "RGB" for im in i1), what
            assert torch.isfinite(l1).all(), what
            if k["batch_size"] > 1:
                assert not torch.equal(l1[0], l1[1]), what
            if (version, method) == ("2.2", "generate_inpainting") and "sampler" in k:
                assert torch.equal(l1[keep], inputs["lat"].cuda().expand(2, 4, 8, 8)[keep]), what
        for j, (_, lj) in enumerate(first):
            for (method, _, k), (_, li) in zip(calls[:j], first[:j]):
                assert not torch.equal(li, lj), (task, calls[j][0], calls[j][2].get("sampler"), method, k.get("sampler"))


# ---- full size -----------------------------------------------------------------------------------------------------------
@pytest.mark.parametrize("name,n,seed", [("dpmpp_2m_sampler", 20, 41), ("dpmpp_2m_sde_sampler", 20, 43),
                                         ("unipc_sampler", 10, 47), ("heun_sampler", 6, 53),
                                         ("euler_ancestral_sampler", 10, 53)])
def test_full_size_cfg2_matches_oracle(name, n, seed):
    """Full-size 2.2 decoder at the cfg-2 geometry (4 images, 96x96 latents, guidance 4) through the step graph (Heun x 6: 11
    evaluations) vs the oracle loop with the fp32 oracle UNet on the GPU and the same per-step draws: finite and within the
    tiny-loop bounds."""
    from oracle import unet_oracle as uo_net
    from tests import test_gpu_unet as tu
    _no_tf32()
    m = tu._full_model()
    B, gs = 4, 4.0
    g = torch.Generator(device="cuda").manual_seed(seed)
    z = torch.randn(B, 4, 96, 96, device="cuda", generator=g)
    img = torch.randn(2 * B, 1280, device="cuda", generator=g)
    sch = _schedule(name, _ac22(), n)
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
        ref = oracle(name, eps, _ac22(), n, z, step_noise=nz)
    err = (out - ref).abs().max().item()
    rel = ((out - ref).norm() / ref.norm()).item()
    print(f"full size cfg-2, {name} x {n}: rel L2 {rel:.3e}, max abs {err:.3e}")
    del sd, ref
    torch.cuda.empty_cache()
    assert rel < 2e-2 and err < 0.15 * out.abs().max().item(), (err, rel)
