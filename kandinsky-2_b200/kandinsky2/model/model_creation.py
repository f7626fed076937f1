"""create_model / create_gaussian_diffusion with the reference's signatures (kandinsky2/model/model_creation.py:9-128).

create_model(**CONFIG_2_1['model_config'], up=False, inpainting=...) returns the H100-native Text2ImUNet /
InpaintText2ImUNet; channel_mult / attention_resolutions strings are resolved exactly as the reference does
(:33-48: attention 'resolutions' are image_size // res downsample rates).
"""
import torch

from .unet import InpaintText2ImUNet, Text2ImUNet


def create_model(image_size, num_channels, num_res_blocks, channel_mult, attention_resolutions, num_heads,
                 num_head_channels, num_heads_upsample, use_scale_shift_norm, dropout, model_dim, resblock_updown,
                 use_fp16, cache_text_emb, text_encoder_in_dim1, text_encoder_in_dim2, pooling_type, in_channels,
                 out_channels, up=False, inpainting=False, version="2.1", **kwargs):
    if channel_mult == "":
        table = {256: (1, 1, 2, 2, 4, 4), 128: (1, 1, 2, 3, 4), 64: (1, 2, 3, 4)}
        if image_size not in table:
            raise ValueError(f"unsupported image size: {image_size}")
        channel_mult = table[image_size]
    elif isinstance(channel_mult, str):
        channel_mult = tuple(int(c) for c in channel_mult.split(","))
    attention_ds = tuple(image_size // int(res) for res in attention_resolutions.split(","))
    if version not in ("2.1", "2.2"):
        raise ValueError("k2b200 implements the 2.1 / 2.2 decoder UNet (2.0 is out of scope, SURVEY.md section 2 #17)")
    if up:
        raise NotImplementedError("super-resolution UNet (SuperResText2ImUNet) is not on the hot path")
    cls = InpaintText2ImUNet if inpainting else Text2ImUNet
    kwargs.pop("use_flash_attention", None)  # attention is always the fused flash-attention kernel
    return cls(in_channels=in_channels, model_channels=num_channels, out_channels=out_channels,
               num_res_blocks=num_res_blocks, attention_resolutions=attention_ds, dropout=dropout,
               model_dim=model_dim, channel_mult=channel_mult, use_fp16=use_fp16, num_heads=num_heads,
               num_head_channels=num_head_channels, num_heads_upsample=num_heads_upsample,
               use_scale_shift_norm=use_scale_shift_norm, resblock_updown=resblock_updown,
               cache_text_emb=cache_text_emb, text_encoder_in_dim1=text_encoder_in_dim1,
               text_encoder_in_dim2=text_encoder_in_dim2, pooling_type=pooling_type,
               cond_version=version, **kwargs)


def create_decoder_unet(model_config, task_type, device, param_dtype=torch.float16):
    """The decoder UNet of a pipeline: create_model(**model_config) for `task_type` -- "inpainting" adds the image and mask
    channels, "controlnet" (Kandinsky 2.2 ControlNet-depth) 4 hint-feature channels beside the 4 latent ones."""
    mc = dict(model_config)
    if task_type == "controlnet":
        mc.update(in_channels=mc["in_channels"] + 4, hint_channels=4)
    return create_model(**mc, up=False, inpainting=(task_type == "inpainting"), device=device, param_dtype=param_dtype)


def create_gaussian_diffusion(*args, **kwargs):
    from .gaussian_diffusion import create_gaussian_diffusion as _c
    return _c(*args, **kwargs)
