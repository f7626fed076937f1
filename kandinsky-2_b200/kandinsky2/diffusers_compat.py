"""A diffusers-`UNet2DConditionModel`-shaped front for the H100 UNet (SURVEY.md 8b, boundary B2).

The reference's Kandinsky 2.2 builds its decoder pipelines with `unet = UNet2DConditionModel.from_pretrained(..., subfolder='unet')`
and hands that object to `KandinskyV22Pipeline(unet=...)` (kandinsky2/kandinsky2_2_model.py:26-42).  A user who keeps the
diffusers pipelines and only wants the denoiser replaced passes an instance of `K2UNet2DConditionModel` instead: it answers the
calls the Kandinsky 2.2 pipelines make on `self.unet` --

    self.unet.config.in_channels / .out_channels / .sample_size,  self.unet.dtype / .device,
    self.unet(sample=latent_model_input, timestep=t, encoder_hidden_states=None,
              added_cond_kwargs={"image_embeds": image_embeds}, return_dict=False)[0]

-- with `sample` [N, 4 (or 9 for inpainting), h, w] (CFG-doubled by the pipeline, unconditional rows first), a scalar or [N]
timestep and image embeddings [N, 1280]; the result is [N, 8, h, w] in the dtype of `sample`.  The diffusers side of this
contract is restated from the published pipelines (diffusers is not part of /root/reference: parity unpinned); the compute
behind it is the parity-tested Text2ImUNet launch plan.
"""
from types import SimpleNamespace

import torch

from .checkpoints import diffusers_unet_to_k2
from .model.unet import InpaintText2ImUNet, Text2ImUNet


class _Output(SimpleNamespace):
    """diffusers' UNet2DConditionOutput: `.sample`, also indexable like the tuple returned for return_dict=False."""

    def __getitem__(self, i):
        return (self.sample,)[i]


class K2UNet2DConditionModel(torch.nn.Module):
    def __init__(self, unet):
        super().__init__()
        self.unet = unet
        lat = unet._latent_channels if unet._inpainting else unet.in_channels - unet.hint_channels
        self.config = SimpleNamespace(in_channels=unet.in_channels, out_channels=unet.out_channels, sample_size=64,
                                      latent_channels=lat, encoder_hid_dim=unet.image_encoder_in_dim,
                                      addition_embed_type="image", encoder_hid_dim_type="image_proj")
        self._cond_key = None

    @classmethod
    def from_state_dict(cls, state_dict, device="cuda", inpainting=False, **unet_kwargs):
        """Build from a diffusers UNet2DConditionModel state dict (kandinsky-2-2-decoder[/-inpaint], subfolder `unet`) or from
        a state dict that already has this package's key names."""
        kw = dict(model_dim=768, image_encoder_in_dim=1280, num_image_embs=32, pooling_type="from_model", in_channels=4,
                  model_channels=384, out_channels=8, num_res_blocks=3, attention_resolutions=(2, 4, 8),
                  channel_mult=(1, 2, 3, 4), use_fp16=True, num_head_channels=64, use_scale_shift_norm=True,
                  resblock_updown=True, cond_version="2.2", device=device, param_dtype=torch.float16)
        kw.update(unet_kwargs)
        unet = (InpaintText2ImUNet if inpainting else Text2ImUNet)(**kw)
        if any(k.startswith(("down_blocks.", "mid_block.", "up_blocks.")) for k in state_dict):
            state_dict = diffusers_unet_to_k2(state_dict, in_channels=unet.in_channels, model_channels=kw["model_channels"],
                                              channel_mult=kw["channel_mult"], num_res_blocks=kw["num_res_blocks"],
                                              attention_ds=kw["attention_resolutions"])
        unet.load_state_dict(state_dict)
        return cls(unet)

    @property
    def dtype(self):
        return torch.float16

    @property
    def device(self):
        return next(self.unet.parameters()).device

    def half(self):
        return self

    def load_attn_procs(self, pretrained_model_name_or_path_or_dict):
        """diffusers' loader for a LoRA of the attention processors (`save_attn_procs` / `AttnProcsLayers` keys, e.g. the
        `pytorch_model.bin` of a decoder LoRA fine-tune), merged into the weights at scale 1.0 (Text2ImUNet.load_lora).  It
        replaces diffusers' two steps `set_attn_processor(LoRAAttnAddedKVProcessor ...)` + `load_state_dict(..., strict=False)`.
        A path is read with torch.load(map_location="cpu", weights_only=True)."""
        sd = pretrained_model_name_or_path_or_dict
        if not isinstance(sd, dict):
            sd = torch.load(sd, map_location="cpu", weights_only=True)
        self.unet.load_lora(sd)

    def to(self, *args, **kwargs):
        dev = [a for a in args if isinstance(a, (str, torch.device))]
        if dev or "device" in kwargs:
            self.unet.to(kwargs.get("device", dev[0] if dev else None))
        return self

    @torch.no_grad()
    def forward(self, sample, timestep, encoder_hidden_states=None, added_cond_kwargs=None, return_dict=True, **unused):
        emb = (added_cond_kwargs or {}).get("image_embeds")
        if emb is None:
            raise ValueError("K2UNet2DConditionModel needs added_cond_kwargs={'image_embeds': ...} (Kandinsky 2.2 decoder)")
        N = sample.shape[0]
        t = torch.as_tensor(timestep, device=sample.device, dtype=torch.float32).reshape(-1)
        t = t.expand(N) if t.numel() == 1 else t
        # the UNet caches its conditioning per generation (like the reference, text2im_model2_1.py:58-59): drop the cache when
        # the pipeline hands over different embeddings
        hint = (added_cond_kwargs or {}).get("hint")
        key = (emb.data_ptr(), tuple(emb.shape), emb._version) + ((hint.data_ptr(), hint._version) if hint is not None else ())
        if key != self._cond_key:
            self.unet.del_cache()
            self._cond_key = key
        kw = {}
        x = sample
        if self.unet._inpainting:  # the inpaint pipeline concatenates [latents, masked_image, mask] along channels
            lat = self.unet._latent_channels
            x, img, msk = sample[:, :lat], sample[:, lat:2 * lat], sample[:, 2 * lat:]
            # the stem multiplies image by mask itself (text2im_model2_1.py:146-155); the pipeline's masked_image is already
            # image * mask and the mask is binary, so the second product changes nothing
            kw = dict(inpaint_image=img.contiguous(), inpaint_mask=msk.contiguous())
        if self.unet.hint_channels:  # ControlNet-depth: added_cond_kwargs carries the depth hint [N, 3, 8h, 8w]
            kw["hint"] = (added_cond_kwargs or {}).get("hint")
        out = self.unet(x.contiguous(), t, image_emb=emb, **kw)
        out = out.to(sample.dtype)
        return _Output(sample=out) if return_dict else (out,)
