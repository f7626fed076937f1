"""CPU: the host side of img2img and ControlNet requests on the continuously refilled batch (kandinsky2/batching.py) -- the
per-request tables of an img2img request against the rows the sampling loops stage, the 2.1 img2img start rule against its
earlier inline form, and what submit and Kandinsky2_2.batcher refuse."""
import numpy as np
import pytest
import torch

SAMPLERS_22 = ("ddpm_sampler", "dpmpp_2m_sampler", "dpmpp_2m_karras_sampler")
SAMPLERS_21 = ("p_sampler", "ddim_sampler", "dpmpp_2m_sampler", "dpmpp_2m_karras_sampler")
STRENGTHS = (0.0, 0.3, 0.5, 0.8, 0.98, 0.999, 1.0)


def _bare_pipe(version, task_type="text2img", grid=(8, 8)):
    """A pipeline object without models: its schedules and img2img start rule run on the CPU, its MoVQ encoder is a stub that
    returns a zero latent of `grid`."""
    from kandinsky2.configs import CONFIG_2_1, CONFIG_2_2
    from kandinsky2.pipelines import Kandinsky2_1, Kandinsky2_2
    cls = Kandinsky2_1 if version == "2.1" else Kandinsky2_2
    pipe = cls.__new__(cls)
    pipe.config = CONFIG_2_1 if version == "2.1" else CONFIG_2_2
    pipe.task_type, pipe.device, pipe.base_seed, pipe.scale = task_type, torch.device("cpu"), 1234, 1
    pipe._encode_image = lambda image, h, w: torch.zeros((1, 4) + grid)
    return pipe


def _staged(pipe, sampler, steps, init_step, monkeypatch):
    """(timesteps, coefficient rows, step noise or None) the sampling loop stages for pipe's img2img at init_step: the schedule
    _decode builds, run by the loop _decode calls for it, with the fused step replaced by a recorder."""
    from kandinsky2.model import gaussian_diffusion as gd
    from kandinsky2.pipelines import _sampler_schedule
    got = {}

    class Recorder:
        def __init__(self, model, B, H, W, *args, **kw):
            self.noise, self.x = torch.zeros(B, 4, H, W), torch.zeros(B, 4, H, W)

        def set_schedule(self, ts, coef, noise_seq):
            got.update(ts=ts, coef=coef, noise=noise_seq)

        def latent(self):
            return self.x

        def advance(self, xs):
            pass

    monkeypatch.setattr(gd, "FusedStep", Recorder)
    model = torch.nn.Linear(1, 1)
    shape, noise = (2, 4, 2, 2), torch.zeros(2, 4, 2, 2)
    gens = [torch.Generator().manual_seed(9)]
    sched = _sampler_schedule(sampler, pipe._diffusion(sampler, steps), steps, init_step)
    if isinstance(sched, gd._SolverSchedule):
        sched.sample(model, shape, noise=noise, device="cpu", sample_generators=gens if sched.draws_noise else None)
    elif isinstance(sched, gd.DDIMSampler):
        sched.model = model
        sched.sample(steps, 2, shape[1:], x_T=noise, init_step=init_step)
    else:
        sched.p_sample_loop(model, shape, noise=noise, device="cpu", init_step=init_step, sample_generators=gens)
    return got["ts"], got["coef"], got["noise"]


@pytest.mark.parametrize("version,sampler", [("2.2", s) for s in SAMPLERS_22] + [("2.1", s) for s in SAMPLERS_21])
@pytest.mark.parametrize("steps", [2, 7, 50])
def test_img2img_request_tables_are_the_rows_the_loop_stages(version, sampler, steps, monkeypatch):
    """request_tables(pipe, sampler, steps, init_step), init_step the pipeline's _img2img_start gives at each strength, is what
    the img2img loop stages, and the DDPM noise the batcher draws from the request's generator is the loop's: as many rows, the
    same stream.  The strengths reach keep = 1 and every row of the schedule."""
    from kandinsky2.batching import request_tables
    pipe = _bare_pipe(version)
    full = request_tables(pipe, sampler, steps)[0].shape[0]
    keeps = set()
    for strength in STRENGTHS:
        _, init_step = pipe._img2img_start(torch.zeros(1, 4, 2, 2), pipe._diffusion(sampler, steps), steps, strength, sampler)
        if init_step < 1:   # the 2.1 rule keeps no step at this strength: submit refuses it
            continue
        ts, coef = request_tables(pipe, sampler, steps, init_step)
        want_ts, want_coef, noise = _staged(pipe, sampler, steps, init_step, monkeypatch)
        assert torch.equal(ts, want_ts.cpu()) and torch.equal(coef, want_coef.cpu()), strength
        n = ts.shape[0]
        keeps.add(n)
        if noise is not None:
            drawn = torch.randn(n, 4, 2, 2, generator=torch.Generator().manual_seed(9))
            assert noise.shape[0] == n and torch.equal(noise[:, 0], drawn)
    assert 1 in keeps and full in keeps, keeps


@pytest.mark.parametrize("sampler", SAMPLERS_21)
@pytest.mark.parametrize("strength", [0.0, 0.3, 0.7, 0.999])
def test_21_img2img_start_is_the_earlier_inline_rule(sampler, strength):
    """Kandinsky2_1._img2img_start gives the start latent and step generate_img2img computed inline before it, bit for bit, and
    base_seed replaces the pipeline's seed of the noise."""
    from kandinsky2.pipelines import SCHEDULE_SAMPLERS
    from kandinsky2.utils import q_sample
    pipe = _bare_pipe("2.1")
    image = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(3))
    steps = 25
    diffusion = pipe._diffusion(sampler, steps)
    x, start = pipe._img2img_start(image, diffusion, steps, strength, sampler)
    if sampler in SCHEDULE_SAMPLERS:
        want_x, want_start = pipe._dpm_img2img_start(image, diffusion, steps, strength, sampler)
    else:
        want_start = int(diffusion.num_timesteps * (1 - strength))
        dc = pipe.config["diffusion_config"]
        want_x = q_sample(image, diffusion.timestep_map[want_start - 1], schedule_name=dc["noise_schedule"],
                          num_steps=dc["steps"], noise=pipe._img2img_noise(image))
    assert start == want_start and torch.equal(x, want_x)
    pipe.base_seed = 99
    x99, _ = pipe._img2img_start(image, diffusion, steps, strength, sampler)
    pipe.base_seed = 1234
    assert torch.equal(pipe._img2img_start(image, diffusion, steps, strength, sampler, base_seed=99)[0], x99)
    assert not torch.equal(x99, x)


def _bare_batcher(version="2.2", task_type="text2img", sampler=None, grid=(8, 8), max_steps=60):
    """A batcher with its host state only (no plan or graph) over a bare pipeline: enough for submit's checks."""
    from kandinsky2.batching import Batcher, Batcher21, _SlotBatcher
    cls = Batcher21 if version == "2.1" else Batcher
    b = cls.__new__(cls)
    b.pipe = _bare_pipe(version, task_type, grid)
    b.sampler = sampler or ("p_sampler" if version == "2.1" else "ddpm_sampler")
    b.max_steps, b._emb_dim, b.h, b.w, b._latent_hw = max_steps, 16, 64, 64, (8, 8)
    b.hinted = task_type == "controlnet"
    b._loras = {}
    _SlotBatcher.__init__(b, 2)
    return b


HINT = torch.zeros(1, 3, 64, 64)
IMAGE = torch.zeros(1, 4, 8, 8)
SUBMIT_22 = [
    ("text2img", {}, dict(strength=0.5), "strength without image"),
    ("text2img", {}, dict(image=IMAGE, strength=1.5), "strength must be"),
    ("text2img", {}, dict(image=IMAGE, strength=-0.1), "strength must be"),
    ("text2img", {}, dict(image=IMAGE, strength=True), "strength must be"),
    ("text2img", {}, dict(image=IMAGE, strength="0.5"), "strength must be"),
    ("text2img", dict(grid=(8, 7)), dict(image=IMAGE, strength=0.5), "latent grid"),
    ("text2img", {}, dict(hint=HINT), "hint is taken"),
    ("text2img", {}, dict(image=IMAGE, strength=0.5, prior_strength=0.8), "prior_strength"),
    ("controlnet", {}, {}, "needs hint"),
    ("controlnet", {}, dict(image=IMAGE, strength=0.5), "needs hint"),
    ("controlnet", {}, dict(hint=HINT, prior_strength=0.8), "prior_strength"),
    ("controlnet", {}, dict(hint=HINT[0, :2]), "one depth map"),
    ("controlnet", {}, dict(hint=HINT.repeat(2, 1, 1, 1)), "one depth map"),
    ("controlnet", {}, dict(hint=HINT, image=IMAGE, strength=0.5, prior_strength=0.8), "prior_strength needs an embedder"),
    ("controlnet", dict(grid=(9, 8)), dict(hint=HINT, image=IMAGE), "latent grid"),
]


@pytest.mark.parametrize("task,bkw,kw,what", SUBMIT_22, ids=[f"{t}-{w}-{i}" for i, (t, _, _, w) in enumerate(SUBMIT_22)])
def test_submit_refuses_bad_img2img_and_controlnet_requests(task, bkw, kw, what):
    """Each bad request is refused at submit with a ValueError naming what is wrong, and leaves nothing queued."""
    b = _bare_batcher("2.2", task, **bkw)
    b.pipe.embedder = object()   # runs no prior: prior_strength has nothing to run
    with pytest.raises(ValueError, match=what):
        b.submit("a cat", decoder_steps=10, **kw)
    assert not b.queue.waiting and not b._requests


@pytest.mark.parametrize("sampler,strength", [("p_sampler", 1.0), ("p_sampler", 0.99), ("ddim_sampler", 1.0),
                                              ("ddim_sampler", 0.9999)])
def test_submit21_refuses_a_strength_that_keeps_no_step(sampler, strength):
    """The 2.1 rule start_step = int(T * (1 - strength)) keeps no step near strength 1: refused at submit, nothing queued."""
    b = _bare_batcher("2.1", sampler=sampler)
    with pytest.raises(ValueError, match="keeps no denoising step"):
        b.submit("a cat", num_steps=50, image=IMAGE, strength=strength)
    assert not b.queue.waiting and not b._requests


@pytest.mark.parametrize("kw,what", [(dict(strength=0.5), "strength without image"),
                                     (dict(image=IMAGE, strength=2), "strength must be"),
                                     (dict(image=torch.zeros(1, 4, 8, 16), strength=0.5), "latent grid")])
def test_submit21_refuses_bad_img2img_requests(kw, what):
    b = _bare_batcher("2.1", grid=tuple(kw["image"].shape[2:]) if "image" in kw else (8, 8))
    with pytest.raises(ValueError, match=what):
        b.submit("a cat", num_steps=50, **kw)
    assert not b.queue.waiting and not b._requests


@pytest.mark.parametrize("version,task,default", [("2.2", "text2img", 0.4), ("2.2", "controlnet", 0.5), ("2.1", "text2img", 0.7)])
def test_strength_defaults_to_the_methods_default(version, task, default):
    """An image without strength takes the strength of the method the request stands for: generate_img2img's (2.2: 0.4, 2.1:
    0.7) or generate_controlnet_img2img's (0.5)."""
    b = _bare_batcher(version, task)
    seen = []
    orig = b.pipe._img2img_start
    b.pipe._img2img_start = lambda lat, d, steps, strength, sampler, base_seed=None: (
        seen.append(strength), orig(lat, d, steps, strength, sampler, base_seed))[1]
    r = b._img2img_start(IMAGE, None, 10, 5)
    assert seen == [default] and r[0].shape == (1, 4, 8, 8)


@pytest.mark.parametrize("sampler", ["unipc_sampler", "euler_sampler", "heun_sampler", "dpmpp_2m_sde_sampler", "p_sampler"])
def test_controlnet_batcher_refuses_unserved_samplers(sampler):
    from kandinsky2.pipelines import Kandinsky2_2
    pipe = Kandinsky2_2.__new__(Kandinsky2_2)
    pipe.task_type = "controlnet"
    with pytest.raises(ValueError, match=sampler):
        pipe.batcher(2, 512, 512, sampler=sampler)


def test_bind_slot_takes_a_hint_on_controlnet_unets_only():
    """bind_slot refuses a hint on a text2img UNet and its absence on a ControlNet UNet, before any device work."""
    from kandinsky2._native import K2Error
    from kandinsky2.model.unet import Text2ImUNet
    for channels, kw in ((0, dict(hint=HINT)), (4, {})):
        unet = Text2ImUNet.__new__(Text2ImUNet)
        unet.hint_channels, unet.cond_version = channels, "2.2"
        with pytest.raises(K2Error, match="hint"):
            unet.bind_slot(None, 0, torch.zeros(16), torch.zeros(16), **kw)
