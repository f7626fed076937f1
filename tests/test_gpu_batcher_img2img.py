"""GPU: img2img and ControlNet-depth requests on the continuously refilled batch (kandinsky2/batching.py) -- bit for bit against
generate_img2img, generate_controlnet and generate_controlnet_img2img at max_batch = 1, the same bits in any slot next to
requests of other kinds, and one graph replay per step whatever the mix."""
import numpy as np
import pytest
import torch

from tests.sampler_cases import _pipe
from tests.test_gpu_batcher import _run, _step
from tests.test_gpu_batcher_lora import _lora

pytestmark = pytest.mark.gpu

SAMPLERS_22 = ("ddpm_sampler", "dpmpp_2m_sampler", "dpmpp_2m_karras_sampler")
SAMPLERS_21 = ("p_sampler", "ddim_sampler", "dpmpp_2m_sampler", "dpmpp_2m_karras_sampler")
STRENGTHS = (0.3, 0.7)


def _photo(w, h, seed):
    from PIL import Image
    return Image.fromarray((np.random.default_rng(seed).random((h, w, 3)) * 255).astype("uint8"))


def _hint(h, w, seed):
    return torch.rand(1, 3, h, w, generator=torch.Generator().manual_seed(seed))


def _one(b, *args, **req):
    """-> (image, the latent handed to the decoder) of one request run alone on batcher b."""
    lats = {}
    h = b.submit(*args, **req)
    return _run(b, lats)[h], lats[h]


@pytest.mark.parametrize("strength", STRENGTHS)
@pytest.mark.parametrize("sampler", SAMPLERS_22)
def test_22_img2img_request_equals_generate_img2img(sampler, strength):
    """max_batch = 1: a prompt request with an image equals generate_img2img(batch_size=1) with base_seed = its seed, image and
    latent bit for bit; with image_embeds it equals generate_img2img's start and loop on those embeddings."""
    pipe = _pipe("2.2", "text2img")
    photo = _photo(80, 60, 1)
    kw = dict(decoder_steps=7, decoder_guidance_scale=4)
    b = pipe.batcher(1, 64, 64, sampler=sampler, max_steps=8)
    img, lat = _one(b, "a red cat", image=photo, strength=strength, seed=77, **kw)
    pipe.base_seed = 77
    want = pipe.generate_img2img("a red cat", photo, strength=strength, batch_size=1, h=64, w=64, sampler=sampler, **kw)
    assert img.tobytes() == want[0].tobytes() and torch.equal(lat, pipe.seen[-1])
    pos, neg = pipe.embedder.image_emb("a blue dog", 1), pipe.embedder.zero_image_emb(1)
    img2, lat2 = _one(b, image_embeds=pos, negative_image_embeds=neg, image=photo, strength=strength, seed=78, **kw)
    pipe.base_seed = 78
    x, start = pipe._img2img_start(pipe._encode_image(photo, 64, 64), pipe._diffusion(sampler, 7), 7, strength, sampler)
    want2 = pipe._decode_loop(pos, neg, 1, 7, 4, 64, 64, latents=x.repeat(2, 1, 1, 1), init_step=start, sampler=sampler)
    assert img2.tobytes() == want2[0].tobytes() and torch.equal(lat2, pipe.seen[-1])
    assert not torch.equal(lat, lat2)


@pytest.mark.parametrize("strength", STRENGTHS)
@pytest.mark.parametrize("sampler", SAMPLERS_21)
def test_21_img2img_request_equals_generate_img2img(sampler, strength):
    """max_batch = 1: a 2.1 request with an image equals Kandinsky2_1.generate_img2img(batch_size=1), and one with an
    interpolated embedding equals generate_img2img's start and generate_img call on that embedding, bit for bit."""
    pipe = _pipe("2.1", "text2img")
    photo = _photo(80, 60, 2)
    kw = dict(num_steps=7, guidance_scale=5)
    b = pipe.batcher(1, 64, 64, sampler=sampler, max_steps=10)
    img, lat = _one(b, "a red cat", image=photo, strength=strength, seed=55, **kw)
    pipe.base_seed = 55
    want = pipe.generate_img2img("a red cat", photo, strength=strength, batch_size=1, h=64, w=64, sampler=sampler, **kw)
    assert img.tobytes() == want[0].tobytes() and torch.equal(lat, pipe.seen[-1])
    mix = pipe.embedder.interpolate(["a red cat", photo], [0.3, 0.7], 1)
    img2, lat2 = _one(b, "", image_embeds=mix, image=photo, strength=strength, seed=56, **kw)
    pipe.base_seed = 56
    diffusion = pipe._diffusion(sampler, 7)
    x, start = pipe._img2img_start(pipe._encode_image(photo, 64, 64) * pipe.scale, diffusion, 7, strength, sampler)
    want2 = pipe.generate_img("", torch.cat([mix, pipe.embedder.zero_image_emb(1)]), batch_size=1, guidance_scale=5, h=64,
                              w=64, sampler=sampler, num_steps=7, diffusion=diffusion, noise=x.repeat(2, 1, 1, 1),
                              init_step=start)
    assert img2.tobytes() == want2[0].tobytes() and torch.equal(lat2, pipe.seen[-1])


@pytest.mark.parametrize("strength", (None,) + STRENGTHS)
@pytest.mark.parametrize("sampler", SAMPLERS_22)
def test_controlnet_request_equals_generate_controlnet(sampler, strength):
    """max_batch = 1 on a ControlNet pipeline: a request with a hint equals generate_controlnet(batch_size=1), and with an image
    too generate_controlnet_img2img(batch_size=1), bit for bit (a [3, h, w] hint and a hint of another size as those take them)."""
    pipe = _pipe("2.2", "controlnet")
    photo, hint = _photo(80, 60, 3), _hint(64, 64, 4)
    kw = dict(decoder_steps=7, decoder_guidance_scale=4)
    b = pipe.batcher(1, 64, 64, sampler=sampler, max_steps=8)
    if strength is None:
        img, lat = _one(b, "a red cat", hint=hint[0], seed=33, **kw)
        pipe.base_seed = 33
        want = pipe.generate_controlnet("a red cat", hint[0], batch_size=1, h=64, w=64, sampler=sampler, **kw)
    else:
        small = _hint(40, 48, 5)
        img, lat = _one(b, "a red cat", hint=small, image=photo, strength=strength, seed=33, **kw)
        pipe.base_seed = 33
        want = pipe.generate_controlnet_img2img("a red cat", photo, small, strength=strength, batch_size=1, h=64, w=64,
                                                sampler=sampler, **kw)
    assert img.tobytes() == want[0].tobytes() and torch.equal(lat, pipe.seen[-1])


def test_controlnet_prior_strength_equals_generate_controlnet_img2img():
    """prior_strength runs the image-guided prior as generate_controlnet_img2img does (the tiny emb2emb embedder of the
    ControlNet img2img tests): the same bits, with the zero negative and with the notebook's second prior call."""
    from kandinsky2.model.prior import PriorEmbedder22
    from oracle import synth
    from tests import prior22_oracle as p22
    from tests.test_gpu_zz_controlnet_img2img import _pipe as _cn_pipe
    cfg = dict(text_ctx=8, xf_width=128, xf_layers=2, xf_heads=2, xf_final_ln=True, xf_padding=False, clip_dim=1280,
               clip_xf_width=1280)
    dsd = synth.synth_state_dict(p22.diffusers_prior_spec(cfg), seed=13)

    def clip_text(prompts):
        outs = []
        for p in prompts:
            g = torch.Generator().manual_seed(len(p) + 17 * sum(map(ord, p)))
            outs.append((torch.randn(1280, generator=g), torch.randn(8, 1280, generator=g), torch.arange(8) < 2 + len(p) % 6))
        return tuple(torch.stack(t) for t in zip(*outs))

    clip_image = lambda img: torch.full((1, 1280), 0.25 + img.size[0] / 1000)  # noqa: E731
    emb = PriorEmbedder22.from_diffusers(dsd, clip_text, clip_image=clip_image, zero_image_emb=torch.full((1280,), -0.5))
    pipe = _cn_pipe(embedder=emb)
    pipe.seen, finish = [], pipe._finish
    pipe._finish = lambda lat, h, w: (pipe.seen.append(lat.clone()), finish(lat, h, w))[1]
    photo, hint = _photo(64, 64, 9), _hint(64, 64, 10)
    kw = dict(decoder_steps=4, prior_steps=5, negative_prior_prompt="ugly")
    b = pipe.batcher(1, 64, 64, max_steps=4)
    imgs = []
    for ndp in ("", "lowres"):
        img, lat = _one(b, "a capybara", image=photo, hint=hint, strength=0.5, prior_strength=0.85, seed=5,
                        negative_decoder_prompt=ndp, **kw)
        pipe.base_seed = 5
        want = pipe.generate_controlnet_img2img("a capybara", photo, hint, strength=0.5, prior_strength=0.85, batch_size=1,
                                                h=64, w=64, negative_decoder_prompt=ndp, **kw)
        assert img.tobytes() == want[0].tobytes() and torch.equal(lat, pipe.seen[-1]), ndp
        imgs.append(img.tobytes())
    assert imgs[0] != imgs[1]


def _controlnet_isolation(pipe, size, steps, req):
    """(latent of req alone in slot 0, latent of req in slot 2 of a batch whose other slots run a text2img request with
    another hint, img2img requests at other strengths and a LoRA adapter)."""
    la, lb = {}, {}
    alone = pipe.batcher(3, size, size, max_steps=steps, max_loras=1)
    h = alone.submit(**req)
    _run(alone, la)
    del alone
    mixed = pipe.batcher(3, size, size, max_steps=steps, max_loras=1)
    mixed.add_lora("A", _lora(pipe.model, 4, 41), 0.8)
    hint2, photo2 = _hint(size, size, 8), _photo(size, size, 6)
    mixed.submit("a blue dog", hint=hint2, decoder_steps=steps, seed=5)
    _step(mixed, lb)
    mixed.submit("a green bird", image=photo2, hint=hint2, strength=0.6, decoder_steps=steps, seed=6, lora="A")
    _step(mixed, lb)
    h2 = mixed.submit(**req)
    _step(mixed, lb)
    assert mixed.queue.holder[2] == h2
    mixed.submit("a grey owl", image=photo2, hint=req["hint"], strength=1.0, decoder_steps=steps, seed=7, lora="A")
    _run(mixed, lb)
    assert len(lb) == 4 and mixed.queue.holder == [None] * 3
    return la[h], lb[h2]


def test_controlnet_img2img_request_is_isolated_from_the_other_slots():
    pipe = _pipe("2.2", "controlnet")
    req = dict(prompt="a red cat", image=_photo(64, 64, 5), hint=_hint(64, 64, 7), strength=0.5, decoder_steps=8, seed=11)
    a, b = _controlnet_isolation(pipe, 64, 8, req)
    assert torch.isfinite(a).all() and torch.equal(a, b)


def test_21_img2img_request_is_isolated_from_the_other_slots():
    """2.1 p_sampler (each slot's own dynamic threshold): an img2img request has the same bits alone in slot 0 and in slot 2
    next to a text2img request and an img2img request at another strength."""
    pipe = _pipe("2.1", "text2img")
    req = dict(prompt="a red cat", image=_photo(64, 64, 1), strength=0.6, num_steps=10, seed=3)
    la, lb = {}, {}
    alone = pipe.batcher(3, 64, 64, sampler="p_sampler", max_steps=10)
    h = alone.submit(**req)
    _run(alone, la)
    mixed = pipe.batcher(3, 64, 64, sampler="p_sampler", max_steps=10)
    mixed.submit("a blue dog", num_steps=10, seed=4, guidance_scale=3)
    _step(mixed, lb)
    mixed.submit("a green bird", image=_photo(64, 64, 2), strength=0.2, num_steps=10, seed=5)
    _step(mixed, lb)
    h2 = mixed.submit(**req)
    _step(mixed, lb)
    assert mixed.queue.holder[2] == h2
    _run(mixed, lb)
    assert torch.isfinite(la[h]).all() and torch.equal(la[h], lb[h2])


def test_full_size_controlnet_img2img_isolation():
    """The isolation at the full Kandinsky 2.2 ControlNet UNet, 768 x 768 (96 x 96 latents): one ControlNet img2img request has
    the same bits alone in slot 0 and in slot 2 next to requests of the other kinds."""
    from kandinsky2 import get_kandinsky2
    pipe = get_kandinsky2("cuda", task_type="controlnet", model_version="2.2", cache_dir="/nonexistent")
    seen = []
    orig = pipe._finish
    pipe._finish = lambda lat, h, w: (seen.append(lat.clone()), orig(lat, h, w))[1]
    pipe.seen = seen
    req = dict(prompt="a red cat", image=_photo(768, 768, 5), hint=_hint(768, 768, 7), strength=0.5, decoder_steps=4, seed=3)
    a, b = _controlnet_isolation(pipe, 768, 4, req)
    assert a.shape == (1, 4, 96, 96) and torch.isfinite(a).all() and torch.equal(a, b)


def test_one_step_is_one_graph_replay_whatever_the_mix():
    """On a ControlNet batcher with adapters, step() replays the one captured graph once per step while text2img, img2img and
    adapter requests come and go, and every buffer it was captured on (the hint features among them) keeps its address."""
    pipe = _pipe("2.2", "controlnet")
    b = pipe.batcher(2, 64, 64, max_steps=8, max_loras=1)
    b.add_lora("A", _lora(pipe.model, 4, 51))
    g0 = b.graph
    sl = b.slots
    bufs = [sl.x, sl.state, sl.ts_tab, sl.coef_tab, sl.coef, sl.guidance, sl.noise_tab, sl.noise, sl.work, b.w_map, b.plan.x_in,
            b.plan.hint_in, b.plan.t_in, b.plan.out, b.plan.xf_proj] + list(b.plan.enc_kv.values())
    ptrs = [t.data_ptr() for t in bufs]
    calls = []
    orig = g0.replay
    g0.replay = lambda: (calls.append(1), orig())[1]
    photo = _photo(64, 64, 1)
    b.submit("prompt 0", hint=_hint(64, 64, 1), decoder_steps=3, seed=0)
    b.submit("prompt 1", hint=_hint(64, 64, 2), image=photo, strength=0.5, decoder_steps=8, seed=1, lora="A")
    b.submit("prompt 2", hint=_hint(64, 64, 3), image=photo, strength=0.3, decoder_steps=8, seed=2)
    steps = finished = 0
    while b.pending():
        before = len(calls)
        finished += len(b.step())
        steps += 1
        assert len(calls) == before + 1
    assert finished == 3 and steps == len(calls) == 5
    assert b.graph is g0 and [t.data_ptr() for t in bufs] == ptrs
