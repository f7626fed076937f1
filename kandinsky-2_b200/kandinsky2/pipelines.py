"""Task pipelines with the reference's call surface, decoder side computed by libk2b200.so.

Mirrors Kandinsky2_1 (kandinsky2/kandinsky2_1_model.py:21-548) and Kandinsky2_2 (kandinsky2/kandinsky2_2_model.py:15-173):
same method names, keyword arguments, defaults and return type (list of PIL images).  What runs here is the
hot path: latent init -> `num_steps` x [CFG-doubled UNet + scheduler update] -> MoVQ decode -> uint8.

The stages BEFORE the path (CLIP text/image towers, the diffusion prior, the XLM-R text encoder) are outside the
scope of this build (SURVEY.md section 2 rows 15-16, 8f rank 3): they enter through an `embedder` object.  The
default SyntheticEmbedder draws deterministic N(0,1) embeddings keyed by the prompt text, which is what the
benchmark configurations specify (BASELINE.json: "synthetic CLIP embeds"); a real deployment passes an embedder
wrapping its prior / encoders.  img2img / inpainting take a PIL image (encoded by the MoVQ encoder) or an already-encoded latent tensor.
"""
import hashlib
import math

import torch

from . import ops, parallel
from ._native import K2Error
from .model.gaussian_diffusion import (DDIMSampler, DPMSolverSchedule, PLMSSampler, UniPCSchedule, create_ddpm_v22,
                                       create_gaussian_diffusion)
from .model.model_creation import create_model
from .utils import prepare_image, prepare_mask, q_sample, uint8_to_pil
from .vqgan import MOVQ


class SyntheticEmbedder:
    """Deterministic stand-in for prior + encoders: N(0,1) tensors seeded by sha256(prompt)."""

    def __init__(self, image_dim, text_dim=1024, pooled_dim=768, text_len=77, seed=0):
        self.image_dim, self.text_dim, self.pooled_dim, self.text_len, self.seed = image_dim, text_dim, pooled_dim, text_len, seed

    def _gen(self, key):
        h = int.from_bytes(hashlib.sha256(f"{self.seed}:{key}".encode()).digest()[:7], "little")
        return torch.Generator().manual_seed(h)

    def image_emb(self, prompt, batch_size):
        """[batch_size, image_dim]: what generate_clip_emb / the prior pipeline returns for `prompt`."""
        return torch.randn(1, self.image_dim, generator=self._gen(("img", prompt))).repeat(batch_size, 1)

    def zero_image_emb(self, batch_size):
        """CLIP embedding of a black image (create_zero_img_emb, kandinsky2_1_model.py:295-297) / negative embeds."""
        return torch.randn(1, self.image_dim, generator=self._gen(("img", "<zero>"))).repeat(batch_size, 1)

    def text_emb(self, prompt, batch_size):
        """(full_emb [2B, text_len, text_dim], pooled_emb [2B, pooled_dim]): cond rows then uncond rows
        (encode_text, kandinsky2_1_model.py:115-157)."""
        def one(p):
            g = self._gen(("txt", p))
            return torch.randn(1, self.text_len, self.text_dim, generator=g), torch.randn(1, self.pooled_dim, generator=g)
        fc, pc = one(prompt)
        fu, pu = one("")
        return (torch.cat([fc.repeat(batch_size, 1, 1), fu.repeat(batch_size, 1, 1)]),
                torch.cat([pc.repeat(batch_size, 1), pu.repeat(batch_size, 1)]))

    def interpolate(self, items, weights, batch_size):
        """Weighted mix of the embeddings of prompts / images (mix_images)."""
        acc = None
        for it, w in zip(items, weights):
            key = it if isinstance(it, str) else ("pil", getattr(it, "size", None), hashlib.sha256(
                it.tobytes() if hasattr(it, "tobytes") else repr(it).encode()).hexdigest())
            e = torch.randn(1, self.image_dim, generator=self._gen(("img", key))) * w
            acc = e if acc is None else acc + e
        return acc.repeat(batch_size, 1)


def _new_h_w_latent_21(h, w):  # kandinsky2_1_model.py:106-113 (latent side, /8)
    return math.ceil(h / 64) * 8, math.ceil(w / 64) * 8


# DPM-Solver++(2M) sampler name -> (timestep spacing, SDE variant) of its DPMSolverSchedule
DPM_SAMPLERS = {"dpmpp_2m_sampler": ("linspace", False), "dpmpp_2m_karras_sampler": ("karras", False),
                "dpmpp_2m_sde_sampler": ("linspace", True), "dpmpp_2m_sde_karras_sampler": ("karras", True)}
# UniPC sampler name -> timestep spacing of its UniPCSchedule
UNIPC_SAMPLERS = {"unipc_sampler": "linspace", "unipc_karras_sampler": "karras"}
# every multistep-solver sampler name -> (schedule class, its keyword arguments): the one table _decode and the img2img start use
SOLVER_SAMPLERS = {**{name: (DPMSolverSchedule, dict(spacing=sp, sde=sde)) for name, (sp, sde) in DPM_SAMPLERS.items()},
                   **{name: (UniPCSchedule, dict(spacing=sp)) for name, sp in UNIPC_SAMPLERS.items()}}
SAMPLERS_21 = ("p_sampler", "ddim_sampler", "plms_sampler") + tuple(SOLVER_SAMPLERS)
SAMPLERS_22 = ("ddpm_sampler",) + tuple(SOLVER_SAMPLERS)


def _check_sampler(sampler, allowed):
    if sampler not in allowed:
        raise ValueError(f"unknown sampler {sampler!r}: use one of {', '.join(allowed)}")


def _dpm_keep(num_steps, strength):
    """img2img with DPM-Solver++ or UniPC (and the 2.2 DDPM sampler, as diffusers): the last int(N * strength) evaluations run
    (at least 1)."""
    return max(min(int(num_steps * strength), num_steps), 1)


def _solver_schedule(sampler, diffusion, num_steps, keep=None):
    """The DPMSolverSchedule / UniPCSchedule of a SOLVER_SAMPLERS name over diffusion's base table."""
    cls, kw = SOLVER_SAMPLERS[sampler]
    return cls(diffusion.base_alphas_cumprod, num_steps, keep=keep, **kw)


class _DecoderBase:
    version = None
    # how the versions' decoder steps differ: the order of the CFG-doubled rows, the reference's per-step dynamic threshold
    # (the +-2 clamp alone when False), and the inpainting rule (False: the known region replaces x0; True: it is re-noised
    # to the next timestep)
    cond_first = dynamic_threshold = inpaint_renoise = None

    def __init__(self, config, device, task_type="text2img", embedder=None, unet_state_dict=None, movq_state_dict=None,
                 seed=0):
        if not str(device).startswith("cuda"):
            raise K2Error("k2b200 pipelines run on a CUDA sm_90 device only (no CPU fallback)")
        self.config = config
        self.device = torch.device(device)
        self.task_type = task_type
        self.use_fp16 = True
        mc = dict(config["model_config"])
        if task_type == "controlnet":  # Kandinsky 2.2 ControlNet-depth (BASELINE configs[4]): 4 latent + 4 hint-feature channels
            mc.update(in_channels=mc["in_channels"] + 4, hint_channels=4)
        self.model = create_model(**mc, up=False, inpainting=(task_type == "inpainting"), device=self.device,
                                  param_dtype=torch.float16)
        if unet_state_dict is not None:
            self.model.load_state_dict(unet_state_dict)
        else:
            self.model.init_synthetic_(seed)  # no checkpoint offline: random weights of the architecture
        self.model.convert_to_fp16()
        ie = config["image_enc_params"]
        self.scale = ie["scale"]
        self.image_encoder = MOVQ(**ie["params"], device=self.device, param_dtype=torch.float16)
        if movq_state_dict is not None:
            self.image_encoder.load_state_dict(movq_state_dict)
        else:
            self.image_encoder.init_synthetic_(seed + 1)
        self.embedder = embedder or SyntheticEmbedder(mc["image_encoder_in_dim"], mc["text_encoder_in_dim1"],
                                                      mc["text_encoder_in_dim2"])
        self.base_seed = 1234

    # shared tail: decode + crop + uint8 + PIL (kandinsky2_1_model.py:286-292)
    def _finish(self, latents, h, w):
        u8 = self.image_encoder.decode_to_uint8(latents / self.scale, crop_h=h, crop_w=w)
        return uint8_to_pil(u8)

    def _encode_image(self, image, h, w):
        """PIL image (resized to (w, h), utils.py:33-39) or image tensor [1,3,H,W] in [-1,1] -> latent via the MoVQ
        encoder (kandinsky2_1_model.py:458-461); a [1,4,h/8,w/8] tensor is taken as an already-encoded latent."""
        if torch.is_tensor(image):
            if image.shape[1] == self.image_encoder.embed_dim:
                return image.float().to(self.device)
            return self.image_encoder.encode(image.to(self.device))
        return self.image_encoder.encode(prepare_image(image, w=w, h=h).to(self.device))

    def _generators(self, lo, hi):
        """One device RNG stream per GLOBAL sample index (step noise independent of world size / batch position)."""
        return [torch.Generator(device=self.device).manual_seed(self.base_seed * 7919 + gi) for gi in range(lo, hi)]

    def _img2img_noise(self, latent):
        """Seeded by base_seed alone: every img2img call on one image starts from the same noisy latent."""
        return torch.randn(latent.shape, generator=torch.Generator().manual_seed(self.base_seed)).to(self.device)

    def _dpm_img2img_start(self, latent, diffusion, num_steps, strength, sampler):
        """DPM-Solver++ / UniPC img2img -> (start latent, evaluations kept): the image latent noised to the first kept
        evaluation."""
        keep = _dpm_keep(num_steps, strength)
        sched = _solver_schedule(sampler, diffusion, num_steps, keep)
        return sched.start_latent(latent, self._img2img_noise(latent)), keep

    @torch.no_grad()
    def _decode(self, cond, batch_size, latent_hw, image_hw, sampler, diffusion, num_steps, guidance_scale, *, noise=None,
                init_step=None, inpaint=None, hint=None):
        """The decoder call of both versions.  cond: the conditioning of the GLOBAL batch, [2 * batch_size, ...] per key, in
        the version's row order; rank 0's copy is broadcast and this rank keeps its rows.  noise: the start latents
        [2 * batch_size, 4, H, W], or None to draw them per global sample index.  inpaint: (clean latent [1, 4, H, W], mask
        [1, 1, H, W]) for every sample, on the device.  hint: the ControlNet depth map [1, 3, h, w] for every row.  Runs
        `sampler` over `diffusion` (`num_steps` evaluations for the DDIM, PLMS, DPM-Solver++ and UniPC samplers) and decodes this
        rank's samples to image_hw."""
        rank, ws = parallel.world()
        lo, hi = parallel.shard_range(batch_size, rank, ws)
        B = hi - lo
        H, W = latent_hw
        parallel.broadcast_conditioning(cond, src=0)   # the path's only collective
        rows = list(range(lo, hi)) + list(range(batch_size + lo, batch_size + hi))
        kw = {k: v[rows].contiguous() for k, v in cond.items()}
        if hint is not None:  # one depth map for the whole batch (cond and uncond rows alike, as the diffusers pipeline does)
            kw["hint"] = hint.to(self.device).float().expand(2 * B, -1, -1, -1).contiguous()
        blend = {}
        if inpaint is not None:
            init, mask = inpaint
            kw["inpaint_image"] = (init * mask).repeat(2 * B, 1, 1, 1)
            kw["inpaint_mask"] = mask.repeat(2 * B, 1, 1, 1)
            blend = dict(inpaint_init=init.repeat(B, 1, 1, 1), inpaint_mask=mask.repeat(B, 1, 1, 1),
                         inpaint_renoise=self.inpaint_renoise)
        if noise is None:
            x = parallel.sample_noise(range(lo, hi), (4, H, W), base_seed=self.base_seed, device=self.device)
            noise = torch.cat([x, x], 0)
        elif noise.shape[0] == 2 * batch_size and ws > 1:
            noise = noise[rows].contiguous()   # a caller-supplied start latent covers the GLOBAL batch: keep this rank's rows
        shape = (2 * B, 4, H, W)
        self.model.del_cache()
        if sampler in SOLVER_SAMPLERS:
            sched = _solver_schedule(sampler, diffusion, num_steps, init_step)
            samples = sched.sample(self.model, shape, noise=noise, model_kwargs=kw, device=self.device,
                                   guidance_scale=guidance_scale, cond_first=self.cond_first,
                                   sample_generators=self._generators(lo, hi) if sched.draws_noise else None, **blend)
        elif sampler in ("ddim_sampler", "plms_sampler"):  # kandinsky2_1_model.py:259-284: un-respaced schedule, eta 0
            cls = DDIMSampler if sampler == "ddim_sampler" else PLMSSampler
            samples, _ = cls(self.model, diffusion).sample(num_steps, 2 * B, (4, H, W), conditioning=kw, x_T=noise,
                                                           init_step=init_step, guidance_scale=guidance_scale,
                                                           cond_first=self.cond_first)
        else:  # "p_sampler" (2.1), "ddpm_sampler" (2.2)
            samples = diffusion.p_sample_loop(self.model, shape, device=self.device, noise=noise, model_kwargs=kw,
                                              init_step=init_step, guidance_scale=guidance_scale, cond_first=self.cond_first,
                                              clip_denoised=self.dynamic_threshold,
                                              sample_generators=self._generators(lo, hi), **blend)
        self.model.del_cache()
        return self._finish(samples[:B], *image_hw)


class Kandinsky2_1(_DecoderBase):
    version = "2.1"
    cond_first = dynamic_threshold = True
    inpaint_renoise = False

    def get_new_h_w(self, h, w):
        return _new_h_w_latent_21(h, w)

    @torch.no_grad()
    def generate_img(self, prompt, img_prompt, batch_size=1, diffusion=None, guidance_scale=7, init_step=None,
                     noise=None, init_img=None, img_mask=None, h=512, w=512, sampler="ddim_sampler", num_steps=50):
        """kandinsky2_1_model.py:184-292. img_prompt = cat([cond image emb, zero image emb]) [2B, 768].
        sampler="dpmpp_2m_sampler" runs DPM-Solver++(2M) over `num_steps` evaluations of diffusion's base schedule; with
        init_step = s only the last s of them run (img2img), starting from `noise`.  "dpmpp_2m_karras_sampler" places the
        evaluations with Karras sigma spacing, "dpmpp_2m_sde_sampler" / "dpmpp_2m_sde_karras_sampler" run the SDE variant
        (fresh noise every step, drawn per global sample index like p_sampler's).  "unipc_sampler" / "unipc_karras_sampler" run
        UniPC (DPM-Solver++(2M) plus the UniC corrector, UniPCSchedule) over the same evaluations.  Inpainting: the known region
        replaces x0 inside the step (p_sampler and the solver samplers; the reference's DDIM / PLMS paths have no such blend)."""
        _check_sampler(sampler, SAMPLERS_21)
        full_emb, pooled_emb = self.embedder.text_emb(prompt, batch_size)
        cond = {"full_emb": full_emb.to(self.device), "pooled_emb": pooled_emb.to(self.device),
                "image_emb": img_prompt.to(self.device).float()}
        inpaint = None
        if self.task_type == "inpainting":
            # the reference repeats ONE image / mask for the cond and uncond rows (:536-537); same image for every sample here
            inpaint = (init_img.to(self.device).float()[:1], img_mask.to(self.device).float()[:1])
        return self._decode(cond, batch_size, self.get_new_h_w(h, w), (h, w), sampler, diffusion, num_steps, guidance_scale,
                            noise=noise, init_step=init_step, inpaint=inpaint)

    def _diffusion(self, sampler, num_steps):
        dc = dict(self.config["diffusion_config"])
        if sampler == "p_sampler":
            dc["timestep_respacing"] = str(num_steps)
        return create_gaussian_diffusion(**dc)

    def _image_embs(self, prompt, batch_size, negative_decoder_prompt=""):
        pos = self.embedder.image_emb(prompt, batch_size)
        neg = (self.embedder.zero_image_emb(batch_size) if negative_decoder_prompt == ""
               else self.embedder.image_emb(negative_decoder_prompt, batch_size))
        return torch.cat([pos, neg], 0)

    def generate_text2img(self, prompt, num_steps=100, batch_size=1, guidance_scale=7, h=512, w=512,
                          sampler="ddim_sampler", prior_cf_scale=4, prior_steps="25", negative_prior_prompt="",
                          negative_decoder_prompt=""):
        _check_sampler(sampler, SAMPLERS_21)
        image_emb = self._image_embs(prompt, batch_size, negative_decoder_prompt)
        return self.generate_img(prompt=prompt, img_prompt=image_emb, batch_size=batch_size,
                                 guidance_scale=guidance_scale, h=h, w=w, sampler=sampler, num_steps=num_steps,
                                 diffusion=self._diffusion(sampler, num_steps))

    def mix_images(self, images_texts, weights, num_steps=100, batch_size=1, guidance_scale=7, h=512, w=512,
                   sampler="ddim_sampler", prior_cf_scale=4, prior_steps="25", negative_prior_prompt="",
                   negative_decoder_prompt=""):
        _check_sampler(sampler, SAMPLERS_21)
        assert len(images_texts) == len(weights) and len(images_texts) > 0
        pos = self.embedder.interpolate(images_texts, weights, batch_size)
        image_emb = torch.cat([pos, self.embedder.zero_image_emb(batch_size)], 0)
        return self.generate_img(prompt="", img_prompt=image_emb, batch_size=batch_size, guidance_scale=guidance_scale,
                                 h=h, w=w, sampler=sampler, num_steps=num_steps,
                                 diffusion=self._diffusion(sampler, num_steps))


    def generate_img2img(self, prompt, pil_img, strength=0.7, num_steps=100, batch_size=1, guidance_scale=7, h=512,
                         w=512, sampler="ddim_sampler", prior_cf_scale=4, prior_steps="25"):
        """kandinsky2_1_model.py:428-484: encode the image, noise it to step int(T*(1-strength)) and run the remaining steps.
        With a dpmpp_2m or unipc sampler the last int(num_steps*strength) solver evaluations run (at least 1), from the image
        noised to the first of them."""
        _check_sampler(sampler, SAMPLERS_21)
        diffusion = self._diffusion(sampler, num_steps)
        image = self._encode_image(pil_img, h, w) * self.scale
        if sampler in SOLVER_SAMPLERS:
            x, start_step = self._dpm_img2img_start(image, diffusion, num_steps, strength, sampler)
        else:
            start_step = int(diffusion.num_timesteps * (1 - strength))
            dc = self.config["diffusion_config"]
            x = q_sample(image, diffusion.timestep_map[start_step - 1], schedule_name=dc["noise_schedule"],
                         num_steps=dc["steps"], noise=self._img2img_noise(image))
        x = x.repeat(2 * batch_size, 1, 1, 1)
        image_emb = self._image_embs(prompt, batch_size)
        return self.generate_img(prompt=prompt, img_prompt=image_emb, batch_size=batch_size,
                                 guidance_scale=guidance_scale, h=h, w=w, sampler=sampler, num_steps=num_steps,
                                 diffusion=diffusion, noise=x, init_step=start_step)

    def generate_inpainting(self, prompt, pil_img, img_mask, num_steps=100, batch_size=1, guidance_scale=7, h=512,
                            w=512, sampler="ddim_sampler", prior_cf_scale=4, prior_steps="25",
                            negative_prior_prompt="", negative_decoder_prompt=""):
        """kandinsky2_1_model.py:487-548 (mask: 1 = keep, nearest-resized to the latent grid, then prepare_mask)."""
        _check_sampler(sampler, SAMPLERS_21)
        image = self._encode_image(pil_img, h, w) * self.scale
        m = torch.as_tensor(img_mask).float()[None, None]
        m = torch.nn.functional.interpolate(m, tuple(image.shape[-2:]), mode="nearest")
        m = prepare_mask(m)
        image_emb = torch.cat([self.embedder.image_emb(prompt, batch_size), self.embedder.zero_image_emb(batch_size)], 0)
        return self.generate_img(prompt=prompt, img_prompt=image_emb, batch_size=batch_size,
                                 guidance_scale=guidance_scale, h=h, w=w, sampler=sampler, num_steps=num_steps,
                                 diffusion=self._diffusion(sampler, num_steps),
                                 init_img=image.repeat(2, 1, 1, 1), img_mask=m.repeat(2, 1, 1, 1))


class Kandinsky2_2(_DecoderBase):
    version = "2.2"
    cond_first = dynamic_threshold = False
    # diffusers KandinskyV22InpaintPipeline (the reference delegates to it, kandinsky2_2_model.py:143-173): after every
    # scheduler step the known region (mask = 1) is the clean latent noised to the next timestep with the run's initial noise,
    # and the result is blended with the clean latent at the end -- the step kernels' inpaint_noise mode
    inpaint_renoise = True

    def get_new_h_w(self, h, w):  # kandinsky2_2_model.py:46-53 (pixels)
        return math.ceil(h / 64) * 64, math.ceil(w / 64) * 64

    def _decode_loop(self, image_embeds, negative_embeds, batch_size, steps, guidance, h, w, latents=None, inpaint=None,
                     init_step=None, hint=None, sampler="ddpm_sampler"):
        """The body of diffusers KandinskyV22Pipeline.__call__ (reference call sites kandinsky2_2_model.py:78-80,
        106-111,138-141,168-172): uncond rows first, DDPM learned-range step, +-2 clip, no dynamic threshold.
        sampler="dpmpp_2m_sampler" (or its Karras / SDE variants, DPM_SAMPLERS): DPM-Solver++(2M) over `steps` evaluations of
        the same base schedule instead, "unipc_sampler" / "unipc_karras_sampler" UniPC (init_step = the number of evaluations
        kept for img2img); inpainting re-noises the known region to the next timestep."""
        _check_sampler(sampler, SAMPLERS_22)
        cond = {"image_emb": torch.cat([negative_embeds, image_embeds], 0).to(self.device).float()}
        return self._decode(cond, batch_size, (h // 8, w // 8), (h, w), sampler, create_ddpm_v22(steps), steps, guidance,
                            noise=latents, init_step=init_step, inpaint=inpaint, hint=hint)

    def _prior_kwargs(self, prior_steps, prior_guidance_scale, negative_prior_prompt):
        """The call's prior keywords for an embedder that runs the prior (`runs_prior`, e.g. model.prior.PriorEmbedder22); None
        for every other embedder, which sees exactly the calls it always saw."""
        if not getattr(self.embedder, "runs_prior", False):
            return None
        return dict(prior_steps=prior_steps, prior_guidance_scale=prior_guidance_scale,
                    negative_prior_prompt=negative_prior_prompt)

    def _embeds(self, prompt, batch_size, negative_decoder_prompt, prior_kw=None):
        """(image embedding of prompt, decoder negative): the negative is zero_image_emb when negative_decoder_prompt is "",
        else the prior's embedding of negative_decoder_prompt guided against "" (kandinsky2_2_model.py:72-76)."""
        pos = self.embedder.image_emb(prompt, batch_size, **(prior_kw or {}))
        return pos, self._negative(batch_size, negative_decoder_prompt, prior_kw)

    def _negative(self, batch_size, negative_decoder_prompt, prior_kw):
        if negative_decoder_prompt == "":
            return self.embedder.zero_image_emb(batch_size)
        if prior_kw is None:
            return self.embedder.image_emb(negative_decoder_prompt, batch_size)
        return self.embedder.image_emb(negative_decoder_prompt, batch_size, **{**prior_kw, "negative_prior_prompt": ""})

    def generate_text2img(self, prompt, batch_size=1, decoder_steps=50, prior_steps=25, decoder_guidance_scale=4,
                          prior_guidance_scale=4, h=512, w=512, negative_prior_prompt="", negative_decoder_prompt="",
                          sampler="ddpm_sampler"):
        _check_sampler(sampler, SAMPLERS_22)
        h, w = self.get_new_h_w(h, w)
        pk = self._prior_kwargs(prior_steps, prior_guidance_scale, negative_prior_prompt)
        pos, neg = self._embeds(prompt, batch_size, negative_decoder_prompt, pk)
        return self._decode_loop(pos, neg, batch_size, decoder_steps, decoder_guidance_scale, h, w, sampler=sampler)

    def mix_images(self, images_texts, weights, batch_size=1, decoder_steps=50, prior_steps=25,
                   decoder_guidance_scale=4, prior_guidance_scale=4, h=512, w=512, negative_prior_prompt="",
                   negative_decoder_prompt="", sampler="ddpm_sampler"):
        _check_sampler(sampler, SAMPLERS_22)
        assert len(images_texts) == len(weights) and len(images_texts) > 0
        pk = self._prior_kwargs(prior_steps, prior_guidance_scale, negative_prior_prompt)
        if pk is None:
            pos = self.embedder.interpolate(images_texts, weights, batch_size)
            _, neg = self._embeds("", batch_size, negative_decoder_prompt)
        else:  # no prior run for the unused embedding of ""
            pos = self.embedder.interpolate(images_texts, weights, batch_size, **pk)
            neg = self._negative(batch_size, negative_decoder_prompt, pk)
        return self._decode_loop(pos, neg, batch_size, decoder_steps, decoder_guidance_scale, h, w, sampler=sampler)

    def generate_img2img(self, prompt, image, strength=0.4, batch_size=1, decoder_steps=100, prior_steps=25,
                         decoder_guidance_scale=4, prior_guidance_scale=4, h=512, w=512, negative_prior_prompt="",
                         negative_decoder_prompt="", sampler="ddpm_sampler"):
        _check_sampler(sampler, SAMPLERS_22)
        h, w = self.get_new_h_w(h, w)
        pk = self._prior_kwargs(prior_steps, prior_guidance_scale, negative_prior_prompt)
        pos, neg = self._embeds(prompt, batch_size, negative_decoder_prompt, pk)
        lat = self._encode_image(image, h, w)
        diffusion = create_ddpm_v22(decoder_steps)
        x, start = self._img2img_start(lat, diffusion, decoder_steps, strength, sampler)
        return self._decode_loop(pos, neg, batch_size, decoder_steps, decoder_guidance_scale, h, w,
                                 latents=x.repeat(2 * batch_size, 1, 1, 1), init_step=start, sampler=sampler)

    def _img2img_start(self, lat, diffusion, steps, strength, sampler):
        """img2img of the 2.2 methods -> (start latent [1, 4, h, w], the init_step of _decode_loop): the solver samplers'
        _dpm_img2img_start, else diffusers' KandinskyV22Img2ImgPipeline rule -- the last int(steps * strength) DDPM timesteps
        (at least 1) run, from scheduler.add_noise of the image latent at the first of them."""
        if sampler in SOLVER_SAMPLERS:
            return self._dpm_img2img_start(lat, diffusion, steps, strength, sampler)
        start = _dpm_keep(steps, strength)
        ac = float(diffusion.alphas_cumprod[start - 1])
        return ac ** 0.5 * lat + (1.0 - ac) ** 0.5 * self._img2img_noise(lat), start

    @staticmethod
    def _hint(hint, h, w):
        """The ControlNet depth map as a float tensor [1, 3, h, w] (a [3, H, W] map gains the batch axis; another size is
        resized bilinearly)."""
        hint = torch.as_tensor(hint).float()
        if hint.dim() == 3:
            hint = hint[None]
        if tuple(hint.shape[-2:]) != (h, w):
            hint = torch.nn.functional.interpolate(hint, (h, w), mode="bilinear", align_corners=False)
        return hint

    def generate_controlnet(self, prompt, hint, batch_size=1, decoder_steps=50, prior_steps=25, decoder_guidance_scale=4,
                            prior_guidance_scale=4, h=512, w=512, negative_prior_prompt="", negative_decoder_prompt="",
                            sampler="ddpm_sampler"):
        """Kandinsky 2.2 ControlNet-depth (BASELINE configs[4]).  The reference package has no method for it -- its
        notebooks/kandinsky2_2_controlnet.ipynb calls diffusers' KandinskyV22ControlnetPipeline(image_embeds=...,
        negative_image_embeds=..., hint=hint, height=h, width=w) directly -- so this follows the sibling methods' signature.
        hint: depth map tensor [1, 3, h, w] in [0, 1] (the pipeline object must be built with task_type="controlnet")."""
        _check_sampler(sampler, SAMPLERS_22)
        if self.task_type != "controlnet":
            raise ValueError("generate_controlnet needs a pipeline built with task_type='controlnet'")
        h, w = self.get_new_h_w(h, w)
        pk = self._prior_kwargs(prior_steps, prior_guidance_scale, negative_prior_prompt)
        pos, neg = self._embeds(prompt, batch_size, negative_decoder_prompt, pk)
        hint = self._hint(hint, h, w)
        return self._decode_loop(pos, neg, batch_size, decoder_steps, decoder_guidance_scale, h, w, hint=hint, sampler=sampler)

    def generate_controlnet_img2img(self, prompt, image, hint, strength=0.5, batch_size=1, decoder_steps=50, prior_steps=25,
                                    decoder_guidance_scale=4, prior_guidance_scale=4, h=512, w=512, negative_prior_prompt="",
                                    negative_decoder_prompt="", sampler="ddpm_sampler", prior_strength=None):
        """Kandinsky 2.2 ControlNet-depth image-to-image: what notebooks/kandinsky2_2_controlnet.ipynb, the reference's one use
        of the ControlNet model, runs with diffusers' KandinskyV22ControlnetImg2ImgPipeline (the reference package has no
        method for it; the signature follows generate_controlnet's, the defaults are the notebook's).  image (PIL image, image
        tensor or encoded latent, as generate_img2img takes it) is encoded by the MoVQ encoder and noised to the first of the
        last int(decoder_steps * strength) evaluations (generate_img2img's start, for every sampler name), and those run with
        the depth hint (as generate_controlnet takes it).

        prior_strength=None: the image embeddings come from the prompt alone, as in generate_controlnet.  A number runs the
        prior from the image's CLIP embedding instead (KandinskyV22PriorEmb2EmbPipeline, PriorEmbedder22.emb2emb; image must
        then be a PIL image, which the embedder's clip_image embeds): the positive embedding is emb2emb(prompt, image,
        strength=prior_strength), the decoder negative is zero_image_emb for negative_decoder_prompt == "", else
        emb2emb(negative_decoder_prompt, image, strength=1, guided against "") -- the notebook's second prior call.  That
        needs an embedder with `runs_prior` and `emb2emb`."""
        _check_sampler(sampler, SAMPLERS_22)
        if self.task_type != "controlnet":
            raise ValueError("generate_controlnet_img2img needs a pipeline built with task_type='controlnet'")
        pk = self._prior_kwargs(prior_steps, prior_guidance_scale, negative_prior_prompt)
        if prior_strength is not None and (pk is None or not hasattr(self.embedder, "emb2emb")):
            raise ValueError("prior_strength needs an embedder that runs the prior from an image embedding "
                             "(runs_prior and emb2emb, e.g. model.prior.PriorEmbedder22)")
        h, w = self.get_new_h_w(h, w)
        if prior_strength is None:
            pos, neg = self._embeds(prompt, batch_size, negative_decoder_prompt, pk)
        else:
            pos = self.embedder.emb2emb(prompt, image, batch_size, strength=prior_strength, **pk)
            neg = (self.embedder.zero_image_emb(batch_size) if negative_decoder_prompt == "" else
                   self.embedder.emb2emb(negative_decoder_prompt, image, batch_size, strength=1.0,
                                         **{**pk, "negative_prior_prompt": ""}))
        lat = self._encode_image(image, h, w)
        x, start = self._img2img_start(lat, create_ddpm_v22(decoder_steps), decoder_steps, strength, sampler)
        return self._decode_loop(pos, neg, batch_size, decoder_steps, decoder_guidance_scale, h, w,
                                 latents=x.repeat(2 * batch_size, 1, 1, 1), init_step=start, hint=self._hint(hint, h, w),
                                 sampler=sampler)

    def generate_inpainting(self, prompt, pil_img, img_mask, batch_size=1, decoder_steps=50, prior_steps=25,
                            decoder_guidance_scale=4, prior_guidance_scale=4, h=512, w=512, negative_prior_prompt="",
                            negative_decoder_prompt="", sampler="ddpm_sampler"):
        _check_sampler(sampler, SAMPLERS_22)
        h, w = self.get_new_h_w(h, w)
        pk = self._prior_kwargs(prior_steps, prior_guidance_scale, negative_prior_prompt)
        pos, neg = self._embeds(prompt, batch_size, negative_decoder_prompt, pk)
        lat = self._encode_image(pil_img, h, w)
        m = torch.as_tensor(img_mask).float()[None, None]
        m = torch.nn.functional.interpolate(m, (h // 8, w // 8), mode="nearest").to(self.device)
        return self._decode_loop(pos, neg, batch_size, decoder_steps, decoder_guidance_scale, h, w, inpaint=(lat, m),
                                 sampler=sampler)
