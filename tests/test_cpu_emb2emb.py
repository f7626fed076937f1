"""CPU: truncated UnCLIP sampling (UnCLIPSchedule(keep=...)), the host side of PriorEmbedder22.emb2emb, and the argument
rules of Kandinsky2_2.generate_controlnet_img2img -- against the restated emb2emb loop of tests/emb2emb_oracle.py."""
import types

import numpy as np
import pytest
import torch

from tests import emb2emb_oracle as eo
from tests import prior22_oracle as p22
from tests.test_cpu_prior22 import _apply_rows


def test_kept_rows_are_the_tail_of_the_full_schedule():
    from kandinsky2.model.prior import UnCLIPSchedule
    for N in range(2, 51):
        full = UnCLIPSchedule(N)
        rows, ts = full.rows(), full.timesteps
        for k in range(1, N + 1):
            s = UnCLIPSchedule(N, keep=k)
            assert s.keep == k and s.num_steps == N
            assert np.array_equal(s.rows(), rows[N - k:]), (N, k)
            assert np.array_equal(s.timesteps, ts[N - k:]), (N, k)
            assert np.array_equal(s.coef_table(), full.coef_table()[N - k:]), (N, k)
        for same in (UnCLIPSchedule(N, keep=None), UnCLIPSchedule(N, keep=N)):
            assert np.array_equal(same.rows(), rows) and np.array_equal(same.timesteps, ts) and same.keep == N
        assert np.array_equal(ts, p22.unclip_timesteps(N))


def test_keep_out_of_range_and_too_few_steps():
    from kandinsky2.model.prior import UnCLIPSchedule
    for N, k in ((5, 0), (5, 6), (5, -1), (2, 3)):
        with pytest.raises(ValueError):
            UnCLIPSchedule(N, keep=k)
    with pytest.raises(ValueError):
        UnCLIPSchedule(1, keep=1)


def test_start_latent_is_add_noise_at_the_first_kept_timestep():
    from kandinsky2.model.prior import UnCLIPSchedule
    g = torch.Generator().manual_seed(0)
    emb, z = torch.randn(3, 16, generator=g, dtype=torch.float64), torch.randn(3, 16, generator=g, dtype=torch.float64)
    for N, k in ((25, 21), (25, 25), (10, 1), (2, 1)):
        s = UnCLIPSchedule(N, keep=k)
        a = s.alphas_cumprod[int(s.timesteps[0])]
        assert torch.equal(s.start_latent(emb, z), float(np.sqrt(a)) * emb + float(np.sqrt(1 - a)) * z)
    full = UnCLIPSchedule(25)
    assert full.timesteps[0] == 999 and UnCLIPSchedule(25, keep=21).timesteps[0] == full.timesteps[4]


@pytest.mark.parametrize("N", [2, 3, 10, 25, 50])
@pytest.mark.parametrize("strength", [0.3, 0.5, 0.85, 1.0])
@pytest.mark.parametrize("guidance", [1.0, 4.0])
def test_kept_rows_reproduce_the_emb2emb_loop(N, strength, guidance):
    """The kept rows through k2_sampler_step's formula, started from start_latent, against the restated
    KandinskyV22PriorEmb2EmbPipeline loop (float64, injected noise, a closed-form stand-in model)."""
    from kandinsky2.model.prior import UnCLIPSchedule
    keep = eo.keep_of(N, strength)
    if keep == 0:   # N = 2, 3 at strength 0.3: the schedule refuses, as emb2emb does
        with pytest.raises(ValueError):
            UnCLIPSchedule(N, keep=keep)
        return
    g = torch.Generator().manual_seed(N)
    B, D = 3, 16
    emb = torch.randn(B, D, generator=g, dtype=torch.float64) * 0.5
    z = torch.randn(B, D, generator=g, dtype=torch.float64)
    noise = torch.randn(keep, B, D, generator=g, dtype=torch.float64)
    mean, std = 0.1 * torch.randn(D, generator=g, dtype=torch.float64), 0.5 + torch.rand(D, generator=g, dtype=torch.float64)
    w = torch.randn(D, D, generator=g, dtype=torch.float64)
    # depends on the sample and reaches past the +-10 clamp; the CFG halves differ (a 2B-row input) or not (B rows)
    fn = lambda xx, tt: (8 * torch.tanh(xx.double() @ w) + torch.linspace(-6, 6, xx.shape[0], dtype=torch.float64)[:, None])  # noqa: E731
    sched = UnCLIPSchedule(N, keep=keep)
    assert sched.rows().shape == (keep, 8)
    if guidance > 1.0:
        got = _apply_rows(sched.rows(), fn, sched.start_latent(emb, z), noise, guidance, mean, std)
    else:   # unguided: the product runs the conditional rows twice, so its CFG combination is the conditional prediction
        cond = lambda xx, tt: fn(xx[xx.shape[0] // 2:], tt).repeat(2, 1)  # noqa: E731
        got = _apply_rows(sched.rows(), cond, sched.start_latent(emb, z), noise, guidance, mean, std)
    ref = eo.emb2emb_sample(fn, emb, z, noise, N, strength, guidance, mean, std)
    assert ((got - ref).abs().max() / ref.abs().max()).item() <= 1e-12


def test_strength_to_keep():
    assert [eo.keep_of(25, s) for s in (0.85, 1.0, 0.3, 0.04, 0.0)] == [21, 25, 7, 1, 0]
    assert eo.keep_of(10, 0.3) == 3 and eo.keep_of(2, 0.3) == 0


# ---------------------------------------------------------------------------------------------------------------------------
# PriorEmbedder22.emb2emb, host side (sample_prior22 replaced by a recorder)
# ---------------------------------------------------------------------------------------------------------------------------
D = 8


def _clip_text(prompts):
    outs = []
    for p in prompts:
        g = torch.Generator().manual_seed(len(p) + 17 * sum(map(ord, p)))
        outs.append((torch.randn(D, generator=g), torch.randn(4, D, generator=g), torch.arange(4) < 2 + len(p) % 3))
    return tuple(torch.stack(t) for t in zip(*outs))


@pytest.fixture
def recorded(monkeypatch):
    from kandinsky2.model import prior as prior_mod
    seen = []

    def fake(model, te, tenc, mask, num_steps, guidance, mean, std, x_T, noise, use_graph=True, keep=None):
        seen.append(dict(te=te, steps=num_steps, guidance=guidance, x_T=x_T, noise=noise, keep=keep))
        return x_T * std + mean

    monkeypatch.setattr(prior_mod, "sample_prior22", fake)
    emb = prior_mod.PriorEmbedder22(prior=types.SimpleNamespace(clip_dim=D), clip_text=_clip_text, clip_mean=torch.zeros(D),
                                    clip_std=torch.ones(D), clip_image=lambda img: torch.full((1, D), 0.25), prior_steps=25)
    return emb, seen


def test_emb2emb_keep_start_and_noise_order(recorded):
    from kandinsky2.model.prior import UnCLIPSchedule
    emb, seen = recorded
    img = torch.randn(1, D, generator=torch.Generator().manual_seed(1))
    emb.emb2emb("a capybara", img, 2, strength=0.85, negative_prior_prompt="ugly")
    r = seen[-1]
    assert r["keep"] == 21 and r["steps"] == 25 and r["noise"].shape == (21, 2, D) and r["guidance"] == 4.0
    assert torch.equal(r["te"], _clip_text(["ugly", "ugly", "a capybara", "a capybara"])[0])
    # the generator of image_emb (seed and prompt), drawing z [B, D] first, then the step noise [keep, B, D]
    x_T_gen = emb._call_args("a capybara", 2, None, None, None)[3]
    z = torch.randn(2, D, generator=x_T_gen)
    assert torch.equal(r["noise"], torch.randn(21, 2, D, generator=x_T_gen))
    assert torch.equal(r["x_T"], UnCLIPSchedule(25, keep=21).start_latent(img.expand(2, D), z))
    # a [B, D] embedding is used as it is, a PIL image goes through clip_image
    emb.emb2emb("a capybara", img.repeat(2, 1), 2, strength=0.85, negative_prior_prompt="ugly")
    assert torch.equal(seen[-1]["x_T"], r["x_T"])
    from PIL import Image
    emb.emb2emb("a capybara", Image.new("RGB", (8, 8)), 2, strength=0.85, negative_prior_prompt="ugly")
    assert torch.equal(seen[-1]["x_T"], UnCLIPSchedule(25, keep=21).start_latent(torch.full((2, D), 0.25), z))
    # strength 1 keeps every step; guidance <= 1 runs the prompt's rows twice
    emb.emb2emb("a capybara", img, 1, strength=1.0, prior_steps=10, prior_guidance_scale=1.0)
    assert seen[-1]["keep"] == 10 and torch.equal(seen[-1]["te"], _clip_text(["a capybara"] * 2)[0])
    emb.emb2emb("a capybara", img, 1, strength=0.3, prior_steps=10)
    assert seen[-1]["keep"] == 3 and seen[-1]["noise"].shape == (3, 1, D)


def test_emb2emb_refusals(recorded):
    from kandinsky2._native import K2Error
    emb, seen = recorded
    img = torch.zeros(1, D)
    for s in (-0.1, 1.5, float("nan")):
        with pytest.raises(ValueError, match="strength"):
            emb.emb2emb("x", img, 1, strength=s)
    with pytest.raises(ValueError, match="keeps no step"):
        emb.emb2emb("x", img, 1, strength=0.03)             # int(25 * 0.03) = 0
    with pytest.raises(ValueError):
        emb.emb2emb("x", img, 1, strength=1.0, prior_steps=1)
    with pytest.raises(ValueError, match="image embedding"):
        emb.emb2emb("x", torch.zeros(3, D), 2, strength=0.5)
    with pytest.raises(ValueError, match="image embedding"):
        emb.emb2emb("x", torch.zeros(1, D + 1), 1, strength=0.5)
    emb.clip_image = None
    with pytest.raises(K2Error, match="clip_image"):
        emb.emb2emb("x", object(), 1, strength=0.5)
    assert seen == []


# ---------------------------------------------------------------------------------------------------------------------------
# Kandinsky2_2.generate_controlnet_img2img, host side (encoder and decoder replaced)
# ---------------------------------------------------------------------------------------------------------------------------
def _pipe(task_type, embedder):
    from kandinsky2.pipelines import Kandinsky2_2
    p = Kandinsky2_2.__new__(Kandinsky2_2)
    p.task_type, p.embedder, p.device, p.base_seed = task_type, embedder, torch.device("cpu"), 1234
    return p


def test_controlnet_img2img_refusals():
    from kandinsky2.pipelines import SyntheticEmbedder
    syn = SyntheticEmbedder(D)
    with pytest.raises(ValueError, match="task_type='controlnet'"):
        _pipe("img2img", syn).generate_controlnet_img2img("x", None, None)
    with pytest.raises(ValueError, match="unknown sampler"):
        _pipe("controlnet", syn).generate_controlnet_img2img("x", None, None, sampler="euler")
    with pytest.raises(ValueError, match="prior_strength"):
        _pipe("controlnet", syn).generate_controlnet_img2img("x", None, None, prior_strength=0.85)

    class RunsPriorOnly(SyntheticEmbedder):   # runs the prior but has no emb2emb
        runs_prior = True
    with pytest.raises(ValueError, match="prior_strength"):
        _pipe("controlnet", RunsPriorOnly(D)).generate_controlnet_img2img("x", None, None, prior_strength=0.85)


def test_controlnet_img2img_prior_calls(monkeypatch):
    """Which embedder calls the method makes: emb2emb(prompt, image, strength=prior_strength, ...) and the decoder negative
    rule with a number; image_emb exactly as generate_controlnet without."""
    calls = []

    class Spy:
        runs_prior = True

        def image_emb(self, prompt, batch_size, **kw):
            calls.append(("image_emb", prompt, batch_size, kw))
            return torch.ones(batch_size, D)

        def emb2emb(self, prompt, image, batch_size, **kw):
            calls.append(("emb2emb", prompt, image, batch_size, kw))
            return torch.ones(batch_size, D)

        def zero_image_emb(self, batch_size):
            calls.append(("zero", batch_size))
            return torch.zeros(batch_size, D)

    p = _pipe("controlnet", Spy())
    decoded = []
    monkeypatch.setattr(p, "_encode_image", lambda image, h, w: torch.zeros(1, 4, h // 8, w // 8), raising=False)
    monkeypatch.setattr(p, "_decode_loop", lambda *a, **kw: decoded.append((a, kw)) or ["img"], raising=False)
    img = "<photo>"
    pk = dict(prior_steps=25, prior_guidance_scale=4, negative_prior_prompt="")
    p.generate_controlnet_img2img("a capybara", img, torch.zeros(1, 3, 64, 64), prior_strength=0.85, batch_size=2, h=64, w=64)
    assert calls == [("emb2emb", "a capybara", img, 2, dict(strength=0.85, **pk)), ("zero", 2)]
    calls.clear()
    p.generate_controlnet_img2img("a capybara", img, torch.zeros(1, 3, 64, 64), prior_strength=0.85, batch_size=2, h=64, w=64,
                                  negative_prior_prompt="bad", negative_decoder_prompt="lowres")
    assert calls == [("emb2emb", "a capybara", img, 2, dict(strength=0.85, prior_steps=25, prior_guidance_scale=4,
                                                             negative_prior_prompt="bad")),
                     ("emb2emb", "lowres", img, 2, dict(strength=1.0, **pk))]
    calls.clear()
    p.generate_controlnet_img2img("a capybara", img, torch.zeros(1, 3, 64, 64), batch_size=2, h=64, w=64)
    assert calls == [("image_emb", "a capybara", 2, pk), ("zero", 2)]
    # the decoder sees the hint, init_step = int(50 * 0.5) and the start latent for both CFG halves
    a, kw = decoded[-1]
    assert kw["init_step"] == 25 and kw["latents"].shape == (4, 4, 8, 8) and kw["hint"].shape == (1, 3, 64, 64)
