"""GPU: Kandinsky2_2.generate_controlnet_img2img -- the ControlNet-depth image-to-image of the reference's ControlNet notebook
(diffusers' KandinskyV22ControlnetImg2ImgPipeline, restated in tests/emb2emb_oracle.py), with and without the image-guided
prior (PriorEmbedder22.emb2emb)."""
import os
import sys

import numpy as np
import pytest
import torch

from tests import emb2emb_oracle as eo
from tests import prior22_oracle as p22
from tests.test_gpu_movq_sampler import _tiny_overrides

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _pipe(task_type="controlnet", embedder=None, unet_state_dict=None):
    from kandinsky2 import get_kandinsky2
    from kandinsky2.configs import CONFIG_2_2
    from kandinsky2.pipelines import Kandinsky2_2
    if unet_state_dict is None:
        return get_kandinsky2("cuda", task_type=task_type, model_version="2.2", cache_dir="/nonexistent", embedder=embedder,
                              config_overrides=_tiny_overrides())
    import copy
    config = copy.deepcopy(CONFIG_2_2)
    for k, v in _tiny_overrides().items():
        config[k].update(v)
    return Kandinsky2_2(config, "cuda", task_type=task_type, embedder=embedder, unet_state_dict=unet_state_dict)


def _photo(w, h, seed):
    from PIL import Image
    return Image.fromarray((np.random.default_rng(seed).random((h, w, 3)) * 255).astype("uint8"))


def _bytes(imgs):
    return [im.tobytes() for im in imgs]


@pytest.mark.parametrize("strength", [0.5, 1.0])
def test_ddpm_loop_vs_restated_controlnet_img2img(strength):
    """The method's DDPM decode (uint8 conversion bypassed) against the restated KandinskyV22ControlnetImg2ImgPipeline loop:
    ddpm_v22_loop's arithmetic over timesteps[t_start:] from DDPMScheduler.add_noise of the encoded image, the restated
    ControlNet UNet (oracle/controlnet_oracle.py) on the same synthetic weights, the step noise the pipeline draws."""
    from oracle import controlnet_oracle as co, synth
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = dict(co.CONFIG_2_2_HINT, model_channels=64, num_res_blocks=1, model_dim=128, channel_mult=(1, 2), attention_ds=(2,))
    sd = synth.synth_state_dict(co.param_spec(cfg), seed=21)
    pipe = _pipe(unet_state_dict=sd)
    pipe._finish = lambda latents, h, w: latents.clone()      # the final latents instead of the images
    B, N, h, w, gd = 2, 6, 128, 128, 4.0     # the 6 steps of test_ddpm_v22_loop_vs_restated_diffusers, whose bounds apply
    photo = _photo(150, 110, seed=1)
    hint = torch.rand(1, 3, h, w, generator=torch.Generator().manual_seed(2))
    out = pipe.generate_controlnet_img2img("a capybara", photo, hint, strength=strength, batch_size=B, decoder_steps=N, h=h,
                                           w=w, decoder_guidance_scale=gd)
    keep = eo.keep_of(N, strength)
    lat = pipe._encode_image(photo, h, w)
    noise0 = pipe._img2img_noise(lat)
    step_noise = torch.stack([torch.randn(keep, 4, h // 8, w // 8, device="cuda", generator=gen)
                              for gen in pipe._generators(0, B)], 1)
    emb = torch.cat([pipe.embedder.zero_image_emb(B), pipe.embedder.image_emb("a capybara", B)]).float()
    with torch.no_grad():
        ref = eo.controlnet_img2img_loop(lambda xx, tt: co.unet_forward(sd, cfg, xx, tt, emb, hint.expand(2 * B, -1, -1, -1)),
                                         lat.cpu().expand(B, -1, -1, -1), noise0.cpu().expand(B, -1, -1, -1), N, strength,
                                         gd, step_noise.cpu())
    err = (out.cpu() - ref).abs().max().item()
    rel = ((out.cpu() - ref).norm() / ref.norm()).item()
    print(f"ControlNet img2img DDPM, {keep} of {N} steps: max-abs {err:.3e} rel-L2 {rel:.3e}")
    assert err < 2e-1 and rel < 1e-2, (err, rel)   # test_ddpm_v22_loop_vs_restated_diffusers's bounds


@pytest.mark.parametrize("sampler", ["ddpm_sampler", "dpmpp_2m_sampler", "unipc_sampler"])
def test_equals_the_manual_composition(sampler):
    """encode -> the start shared with generate_img2img -> _decode_loop with the hint: the same images, bit for bit."""
    from kandinsky2.model.gaussian_diffusion import create_ddpm_v22
    pipe = _pipe()
    B, N, h, w, strength = 2, 6, 64, 128, 0.5
    photo, hint = _photo(100, 70, seed=3), torch.rand(1, 3, 40, 60, generator=torch.Generator().manual_seed(4))
    got = pipe.generate_controlnet_img2img("a capybara", photo, hint, strength=strength, batch_size=B, decoder_steps=N, h=h,
                                           w=w, sampler=sampler)
    pos, neg = pipe._embeds("a capybara", B, "", None)
    x, start = pipe._img2img_start(pipe._encode_image(photo, h, w), create_ddpm_v22(N), N, strength, sampler)
    want = pipe._decode_loop(pos, neg, B, N, 4, h, w, latents=x.repeat(2 * B, 1, 1, 1), init_step=start,
                             hint=pipe._hint(hint, h, w), sampler=sampler)
    assert start == 3 and _bytes(got) == _bytes(want)


def test_surface_determinism_and_refusals():
    from kandinsky2.pipelines import SAMPLERS_22
    pipe = _pipe()
    photo, hint = _photo(90, 70, seed=5), torch.rand(1, 3, 64, 128, generator=torch.Generator().manual_seed(6))
    kw = dict(batch_size=2, decoder_steps=6, h=64, w=128)
    a = pipe.generate_controlnet_img2img("a capybara", photo, hint, **kw)
    assert len(a) == 2 and all(im.size == (128, 64) and im.mode == "RGB" for im in a)
    assert _bytes(a) == _bytes(pipe.generate_controlnet_img2img("a capybara", photo, hint, **kw))
    assert a[0].tobytes() != a[1].tobytes()
    for other in (dict(strength=0.9), dict(hint=1.0 - hint), dict(image=_photo(90, 70, seed=7))):
        args = dict(dict(prompt="a capybara", image=photo, hint=hint, **kw), **other)
        assert _bytes(pipe.generate_controlnet_img2img(**args)) != _bytes(a), other
    # a [3, H, W] hint and a latent-tensor image are taken as generate_controlnet / generate_img2img take them
    lat = torch.randn(1, 4, 8, 16, generator=torch.Generator().manual_seed(8))
    assert len(pipe.generate_controlnet_img2img("a capybara", lat, hint[0], **kw)) == 2
    for name in SAMPLERS_22:
        imgs = pipe.generate_controlnet_img2img("a capybara", photo, hint, sampler=name, **kw)
        assert len(imgs) == 2 and _bytes(imgs) == _bytes(pipe.generate_controlnet_img2img("a capybara", photo, hint,
                                                                                         sampler=name, **kw)), name
    with pytest.raises(ValueError, match="unknown sampler"):
        pipe.generate_controlnet_img2img("a capybara", photo, hint, sampler="euler", **kw)
    with pytest.raises(ValueError, match="prior_strength"):    # the synthetic embedder runs no prior
        pipe.generate_controlnet_img2img("a capybara", photo, hint, prior_strength=0.85, **kw)
    with pytest.raises(ValueError, match="task_type='controlnet'"):
        _pipe("img2img").generate_controlnet_img2img("a capybara", photo, hint, **kw)


def test_prior_strength_runs_emb2emb():
    """A PriorEmbedder22 spy: prior_strength=s calls emb2emb(prompt, image, strength=s, ...) for the positive embedding and
    the notebook's second call -- emb2emb(negative_decoder_prompt, image, strength=1, guided against "") -- for the decoder
    negative (zero_image_emb when negative_decoder_prompt is "")."""
    from kandinsky2.model.prior import PriorEmbedder22
    from oracle import synth
    cfg = dict(text_ctx=8, xf_width=128, xf_layers=2, xf_heads=2, xf_final_ln=True, xf_padding=False, clip_dim=1280,
               clip_xf_width=1280)
    dsd = synth.synth_state_dict(p22.diffusers_prior_spec(cfg), seed=13)

    def clip_text(prompts):
        outs = []
        for p in prompts:
            g = torch.Generator().manual_seed(len(p) + 17 * sum(map(ord, p)))
            outs.append((torch.randn(1280, generator=g), torch.randn(8, 1280, generator=g), torch.arange(8) < 2 + len(p) % 6))
        return tuple(torch.stack(t) for t in zip(*outs))

    seen = []

    class Spy(PriorEmbedder22):
        def emb2emb(self, prompt, image, batch_size, **kw):
            seen.append(("emb2emb", prompt, image, batch_size, kw))
            return super().emb2emb(prompt, image, batch_size, **kw)

        def image_emb(self, prompt, batch_size, **kw):
            seen.append(("image_emb", prompt, batch_size, kw))
            return super().image_emb(prompt, batch_size, **kw)

        def zero_image_emb(self, batch_size):
            seen.append(("zero", batch_size))
            return super().zero_image_emb(batch_size)

    clip_image = lambda img: torch.full((1, 1280), 0.25 + img.size[0] / 1000)  # noqa: E731
    spy = Spy.from_diffusers(dsd, clip_text, clip_image=clip_image, zero_image_emb=torch.full((1280,), -0.5))
    pipe = _pipe(embedder=spy)
    photo, hint = _photo(64, 64, seed=9), torch.rand(1, 3, 64, 64, generator=torch.Generator().manual_seed(10))
    kw = dict(batch_size=2, decoder_steps=4, h=64, w=64, prior_steps=5, negative_prior_prompt="ugly")
    a = pipe.generate_controlnet_img2img("a capybara", photo, hint, prior_strength=0.85, **kw)
    pk = dict(prior_steps=5, prior_guidance_scale=4, negative_prior_prompt="ugly")
    assert seen == [("emb2emb", "a capybara", photo, 2, dict(strength=0.85, **pk)), ("zero", 2)]
    seen.clear()
    b = pipe.generate_controlnet_img2img("a capybara", photo, hint, prior_strength=0.85, negative_decoder_prompt="lowres", **kw)
    assert seen == [("emb2emb", "a capybara", photo, 2, dict(strength=0.85, **pk)),
                    ("emb2emb", "lowres", photo, 2, dict(strength=1.0, **dict(pk, negative_prior_prompt="")))]
    assert _bytes(a) != _bytes(b)
    assert _bytes(a) == _bytes(pipe.generate_controlnet_img2img("a capybara", photo, hint, prior_strength=0.85, **kw))
    assert _bytes(a) != _bytes(pipe.generate_controlnet_img2img("a capybara", photo, hint, prior_strength=0.5, **kw))
    seen.clear()
    c = pipe.generate_controlnet_img2img("a capybara", photo, hint, **kw)     # no prior_strength: as generate_controlnet
    assert seen == [("image_emb", "a capybara", 2, pk), ("zero", 2)] and _bytes(c) != _bytes(a)


# ---------------------------------------------------------------------------------------------------------------------------
# two GPUs (skipped on a one-GPU machine), checked as tests/test_gpu_multi.py checks the text-to-image pipelines
# ---------------------------------------------------------------------------------------------------------------------------
def _generate(batch):
    pipe = _pipe()
    photo, hint = _photo(128, 128, seed=11), torch.rand(1, 3, 128, 128, generator=torch.Generator().manual_seed(12))
    imgs = pipe.generate_controlnet_img2img("a capybara", photo, hint, strength=0.5, batch_size=batch, decoder_steps=4,
                                            h=128, w=128)
    return np.stack([np.asarray(im) for im in imgs])


def _worker(rank, world, port, batch, q):
    for p in (ROOT, os.path.join(ROOT, "kandinsky-2_b200")):
        sys.path.insert(0, p)
    import torch.distributed as dist
    os.environ["MASTER_ADDR"] = "127.0.0.1"
    os.environ["MASTER_PORT"] = str(port)
    torch.cuda.set_device(rank)
    dist.init_process_group("nccl", rank=rank, world_size=world, device_id=torch.device("cuda", rank))
    q.put((rank, _generate(batch).copy()))
    dist.barrier()
    dist.destroy_process_group()


def test_two_gpus_reproduce_one_gpu():
    if torch.cuda.device_count() < 2:
        pytest.skip("needs 2 GPUs")
    import torch.multiprocessing as mp
    batch = 4
    ctx = mp.get_context("spawn")
    q = ctx.Queue()
    port = 31600 + (os.getpid() % 2000)
    procs = [ctx.Process(target=_worker, args=(r, 2, port, batch, q)) for r in range(2)]
    for p in procs:
        p.start()
    try:
        got = dict(q.get(timeout=150) for _ in procs)
    finally:
        for p in procs:
            p.join(timeout=30)
            if p.is_alive():
                p.kill()
    assert all(p.exitcode == 0 for p in procs)
    single = _generate(batch)
    multi = np.concatenate([got[0], got[1]])
    assert multi.shape == single.shape == (batch, 128, 128, 3)
    diff = np.abs(multi.astype(np.int16) - single.astype(np.int16))
    psnr = [10 * np.log10(255.0 ** 2 / max(float((diff[i].astype(np.float64) ** 2).mean()), 1e-12)) for i in range(batch)]
    other = single[[1, 0, 3, 2]].astype(np.int16)
    cross = 10 * np.log10(255.0 ** 2 / float(((multi.astype(np.int16) - other).astype(np.float64) ** 2).mean()))
    print(f"ControlNet img2img, 2 GPUs: max uint8 difference {diff.max()}, PSNR per image {[round(v, 1) for v in psnr]} dB "
          f"(different samples: {cross:.1f} dB)")
    assert min(psnr) > 30.0 and cross < 25.0, (psnr, cross)
