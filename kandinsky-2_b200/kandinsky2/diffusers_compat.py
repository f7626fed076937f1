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

The released Kandinsky 2.2 decoder folders (`kandinsky-2-2-decoder`, `-decoder-inpaint`, `-controlnet-depth`: model_index.json,
unet/, movq/, scheduler/) are read here too: `unet_config`, `movq_config` and `check_scheduler_config` turn their config files
into this package's configuration, refusing by name every value the kernels do not compute; `read_decoder_folder` gathers a
whole folder for `Kandinsky2_2.from_pretrained`.  The config keys are restated from diffusers' published classes
(`UNet2DConditionModel`, `VQModel`, `DDPMScheduler`), so unpinned.
"""
import os
from copy import deepcopy
from types import SimpleNamespace

import torch

from ._native import K2Error
from .checkpoints import (_require_keys, diffusers_movq_to_k2, diffusers_unet_to_k2, k2_to_diffusers_unet, load_weights,
                          read_json)
from .configs import CONFIG_2_2
from .model.model_creation import create_decoder_unet
from .model.unet import InpaintText2ImUNet, Text2ImUNet

# a diffusers component's weights, most preferred first
WEIGHT_FILES = ("diffusion_pytorch_model.safetensors", "diffusion_pytorch_model.bin",
                "diffusion_pytorch_model.fp16.safetensors", "diffusion_pytorch_model.fp16.bin")
# keys diffusers writes about the file itself
_BOOKKEEPING = ("_class_name", "_diffusers_version", "_name_or_path", "_use_default_values")


def _check_keys(cfg, fixed, read, ignored, what):
    """K2Error naming, in one message, every fixed key of the config dict `cfg` whose value (diffusers' default when absent)
    is not one of its accepted values, then every key that is neither read, ignored nor fixed.  The values come first: they
    are what would change the arithmetic.  fixed: {key: (accepted values, default)}."""
    bad = []
    for k, (accepted, default) in fixed.items():
        v = cfg.get(k, default)
        if not any(v == a and isinstance(v, bool) == isinstance(a, bool) for a in accepted):   # true is not 1 here
            absent = "" if k in cfg else ", absent: diffusers' default"
            bad.append(f"{k} = {v!r}{absent} (implemented: {', '.join(map(repr, accepted))})")
    unknown = [k for k in cfg if k not in fixed and k not in read and k not in ignored and k not in _BOOKKEEPING]
    if unknown:
        bad.append(f"unknown keys {unknown}")
    if bad:
        raise K2Error(f"{what}: " + "; ".join(bad))


def _int_list(cfg, key, n, default, what):
    """cfg[key] as a list of n ints: an int is repeated, as diffusers does."""
    v = cfg.get(key, default)
    v = [v] * n if isinstance(v, int) else list(v)
    if len(v) != n or not all(isinstance(x, int) for x in v):
        raise K2Error(f"{what}: {key} = {cfg.get(key, default)!r} is not one int or {n} of them")
    return v


# ------------------------------------------------------------------------------------------------ UNet2DConditionModel
_UNET_DOWN = {"ResnetDownsampleBlock2D": False, "SimpleCrossAttnDownBlock2D": True}
_UNET_UP = {"ResnetUpsampleBlock2D": False, "SimpleCrossAttnUpBlock2D": True}
# (in_channels, addition_embed_type) -> the pipeline task
_UNET_TASKS = {(4, "image"): "text2img", (9, "image"): "inpainting", (8, "image_hint"): "controlnet"}
_UNET_READ = ("in_channels", "out_channels", "block_out_channels", "layers_per_block", "attention_head_dim",
              "cross_attention_dim", "encoder_hid_dim", "down_block_types", "up_block_types", "addition_embed_type")
# keys that only configure blocks this UNet does not have (transformer blocks, text / text_time additions) or training
_UNET_IGNORED = ("sample_size", "dropout", "downsample_padding", "upcast_attention", "use_linear_projection",
                 "transformer_layers_per_block", "reverse_transformer_layers_per_block", "attention_type",
                 "addition_embed_type_num_heads")
_UNET_FIXED = {  # key -> (accepted values, diffusers' default)
    "mid_block_type": (("UNetMidBlock2DSimpleCrossAttn",), "UNetMidBlock2DCrossAttn"),
    "resnet_time_scale_shift": (("scale_shift",), "default"), "encoder_hid_dim_type": (("image_proj",), None),
    "norm_num_groups": ((32,), 32), "norm_eps": ((1e-5,), 1e-5), "act_fn": (("silu",), "silu"),
    "flip_sin_to_cos": ((True,), True), "freq_shift": ((0,), 0), "center_input_sample": ((False,), False),
    "time_embedding_type": (("positional",), "positional"), "time_embedding_dim": ((None,), None),
    "time_embedding_act_fn": ((None,), None), "timestep_post_act": ((None,), None), "time_cond_proj_dim": ((None,), None),
    "conv_in_kernel": ((3,), 3), "conv_out_kernel": ((3,), 3), "class_embed_type": ((None,), None),
    "num_class_embeds": ((None,), None), "projection_class_embeddings_input_dim": ((None,), None),
    "class_embeddings_concat": ((False,), False), "addition_time_embed_dim": ((None,), None),
    "dual_cross_attention": ((False,), False), "only_cross_attention": ((False,), False),
    "mid_block_only_cross_attention": ((None, False), None), "cross_attention_norm": ((None,), None),
    "num_attention_heads": ((None,), None), "mid_block_scale_factor": ((1,), 1), "resnet_out_scale_factor": ((1,), 1.0),
    "resnet_skip_time_act": ((False,), False)}


def unet_config(config):
    """A Kandinsky 2.2 decoder's unet/config.json dict (diffusers `UNet2DConditionModel`) -> (model_config, task_type):
    the `model_config` of create_model (CONFIG_2_2's, with the geometry read from the file) and "text2img" (4 input channels,
    addition_embed_type "image"), "inpainting" (9, "image") or "controlnet" (8, "image_hint").  Read: block_out_channels
    (num_channels, channel_mult), layers_per_block, attention_head_dim (the head width, 64), cross_attention_dim (model_dim),
    encoder_hid_dim (image_encoder_in_dim) and the attention levels, from the SimpleCrossAttn* block types.  Any other block
    type, resnet_time_scale_shift, encoder_hid_dim_type, head width, group count or unknown key raises K2Error naming the key."""
    what = "UNet config.json"
    _check_keys(config, _UNET_FIXED, _UNET_READ, _UNET_IGNORED, what)
    if config.get("_class_name", "UNet2DConditionModel") != "UNet2DConditionModel":
        raise K2Error(f"{what}: _class_name = {config['_class_name']!r}, not UNet2DConditionModel")
    boc = list(config.get("block_out_channels", ()))
    down, up = list(config.get("down_block_types", ())), list(config.get("up_block_types", ()))
    n = len(boc)
    for key, types, table in (("down_block_types", down, _UNET_DOWN), ("up_block_types", up, _UNET_UP)):
        if len(types) != n or any(t not in table for t in types):
            raise K2Error(f"{what}: {key} = {types!r}: {n} of {', '.join(table)} are implemented")
    attn = [k for k, t in enumerate(down) if _UNET_DOWN[t]]
    if [n - 1 - k for k, t in enumerate(up) if _UNET_UP[t]][::-1] != attn:
        raise K2Error(f"{what}: up_block_types = {up!r}: the attention levels must mirror down_block_types'")
    if not attn:
        raise K2Error(f"{what}: down_block_types = {down!r}: no SimpleCrossAttnDownBlock2D level")
    if not boc or boc[0] <= 0 or any(c % boc[0] for c in boc):
        raise K2Error(f"{what}: block_out_channels = {boc!r}: each must be a multiple of the first")
    if set(_int_list(config, "attention_head_dim", n, 8, what)) != {64}:
        raise K2Error(f"{what}: attention_head_dim = {config.get('attention_head_dim', 8)!r}: the attention kernels run "
                      "heads of width 64")
    layers = _int_list(config, "layers_per_block", n, 2, what)
    if len(set(layers)) != 1:
        raise K2Error(f"{what}: layers_per_block = {layers!r}: one count for every level is implemented")
    dims = {key: config.get(key, default) for key, default in (("cross_attention_dim", 1280), ("encoder_hid_dim", None))}
    for key, v in dims.items():
        if not isinstance(v, int) or isinstance(v, bool):
            raise K2Error(f"{what}: {key} = {v!r}: one int is implemented")
    if config.get("out_channels", 4) != 8:
        raise K2Error(f"{what}: out_channels = {config.get('out_channels', 4)!r}: 4 latent channels and their learned "
                      "variance (8) are implemented")
    key = (config.get("in_channels", 4), config.get("addition_embed_type"))
    if key not in _UNET_TASKS:
        raise K2Error(f"{what}: in_channels = {key[0]!r} with addition_embed_type = {key[1]!r}: implemented are "
                      + ", ".join(f"{c} with {a!r} ({t})" for (c, a), t in _UNET_TASKS.items()))
    mc = deepcopy(CONFIG_2_2["model_config"])
    mult = tuple(c // boc[0] for c in boc)
    # CONFIG_2_2 writes channel_mult "", which create_model resolves to (1, 2, 3, 4) at its image_size of 64
    mc.update(num_channels=boc[0], channel_mult="" if mult == (1, 2, 3, 4) else ",".join(map(str, mult)),
              num_res_blocks=layers[0], attention_resolutions=",".join(str(mc["image_size"] >> k) for k in attn),
              model_dim=dims["cross_attention_dim"], image_encoder_in_dim=dims["encoder_hid_dim"], in_channels=4,
              out_channels=8)
    return mc, _UNET_TASKS[key]


def unet_state_dict_to_k2(sd, model):
    """A diffusers UNet2DConditionModel state dict -> this package's names for `model` (a Text2ImUNet of the same geometry,
    any device, meta included).  Keys the model has no parameter for, and keys it needs that sd lacks, raise K2Error naming
    them (diffusers_unet_to_k2 alone reads only the keys it knows)."""
    kw = dict(in_channels=model.in_channels, model_channels=model.model_channels, channel_mult=model.channel_mult,
              num_res_blocks=model.num_res_blocks, attention_ds=model.attention_resolutions)
    meta = {k: torch.empty(v.shape, device="meta") for k, v in model.state_dict().items()}
    _require_keys(sd, list(k2_to_diffusers_unet(meta, **kw)), "diffusers UNet")
    return diffusers_unet_to_k2(sd, **kw)


# ------------------------------------------------------------------------------------------------ VQModel
_MOVQ_DOWN = {"DownEncoderBlock2D": False, "AttnDownEncoderBlock2D": True}
_MOVQ_UP = {"UpDecoderBlock2D": False, "AttnUpDecoderBlock2D": True}
_MOVQ_READ = ("in_channels", "out_channels", "down_block_types", "up_block_types", "block_out_channels", "layers_per_block",
              "latent_channels", "num_vq_embeddings", "vq_embed_dim")
_MOVQ_IGNORED = ("sample_size", "scaling_factor", "force_upcast")   # the decoder pipelines use none of them
_MOVQ_FIXED = {"norm_type": (("spatial",), "group"), "norm_num_groups": ((32,), 32), "act_fn": (("silu",), "silu"),
               "lookup_from_codebook": ((False,), False), "mid_block_add_attention": ((True,), True)}


def movq_config(config):
    """A Kandinsky 2.2 decoder's movq/config.json dict (diffusers `VQModel`, norm_type "spatial") -> (ddconfig, n_embed,
    embed_dim), the arguments of vqgan.autoencoder.MOVQ.  Read: block_out_channels (ch, ch_mult), layers_per_block
    (num_res_blocks), latent_channels (z_channels), in_channels / out_channels, num_vq_embeddings, vq_embed_dim and the
    attention levels, from the Attn* block types (written as attn_resolutions over a resolution whose last level is 32, the
    form of the reference's configs).  norm_type other than "spatial", norm_num_groups other than 32, other block types,
    act_fn other than silu, lookup_from_codebook, mid_block_add_attention false and unknown keys raise K2Error naming the key."""
    what = "MoVQ config.json"
    _check_keys(config, _MOVQ_FIXED, _MOVQ_READ, _MOVQ_IGNORED, what)
    if config.get("_class_name", "VQModel") != "VQModel":
        raise K2Error(f"{what}: _class_name = {config['_class_name']!r}, not VQModel")
    boc = list(config.get("block_out_channels", (64,)))
    down = list(config.get("down_block_types", ("DownEncoderBlock2D",)))
    up = list(config.get("up_block_types", ("UpDecoderBlock2D",)))
    n = len(boc)
    for key, types, table in (("down_block_types", down, _MOVQ_DOWN), ("up_block_types", up, _MOVQ_UP)):
        if len(types) != n or any(t not in table for t in types):
            raise K2Error(f"{what}: {key} = {types!r}: {n} of {', '.join(table)} are implemented")
    attn = [k for k, t in enumerate(down) if _MOVQ_DOWN[t]]
    if [n - 1 - k for k, t in enumerate(up) if _MOVQ_UP[t]][::-1] != attn:
        raise K2Error(f"{what}: up_block_types = {up!r}: the attention levels must mirror down_block_types'")
    if not boc or boc[0] <= 0 or any(c % boc[0] for c in boc):
        raise K2Error(f"{what}: block_out_channels = {boc!r}: each must be a multiple of the first")
    zc = config.get("latent_channels", 3)
    embed_dim = config.get("vq_embed_dim") or zc
    if embed_dim != zc:   # the SpatialNorms take the unquantised latent: vq_embed_dim channels into zc-channel 1x1 convs
        raise K2Error(f"{what}: vq_embed_dim = {embed_dim!r} differs from latent_channels = {zc!r}")
    resolution = 32 << (n - 1)
    dd = {"double_z": False, "z_channels": zc, "resolution": resolution, "in_channels": config.get("in_channels", 3),
          "out_ch": config.get("out_channels", 3), "ch": boc[0], "ch_mult": [c // boc[0] for c in boc],
          "num_res_blocks": config.get("layers_per_block", 1), "attn_resolutions": [resolution >> k for k in attn],
          "dropout": 0.0}
    return dd, config.get("num_vq_embeddings", 256), embed_dim


# ------------------------------------------------------------------------------------------------ DDPMScheduler
_DDPM_FIXED = {  # what create_ddpm_v22 computes: key -> (accepted values, diffusers' default)
    "_class_name": (("DDPMScheduler",), "DDPMScheduler"), "num_train_timesteps": ((1000,), 1000), "beta_start": ((0.00085,), 0.0001),
    "beta_end": ((0.012,), 0.02), "beta_schedule": (("linear",), "linear"), "trained_betas": ((None,), None),
    "variance_type": (("learned_range",), "fixed_small"), "prediction_type": (("epsilon",), "epsilon"),
    "clip_sample": ((True,), True), "clip_sample_range": ((2.0,), 1.0), "thresholding": ((False,), False),
    "timestep_spacing": (("leading",), "leading"), "steps_offset": ((0,), 0), "rescale_betas_zero_snr": ((False,), False)}
_DDPM_IGNORED = ("dynamic_thresholding_ratio", "sample_max_value")   # they act only with thresholding


def check_scheduler_config(config):
    """A Kandinsky 2.2 decoder's scheduler/scheduler_config.json dict against the DDPMScheduler that create_ddpm_v22 computes
    (linear betas 0.00085 .. 0.012 over 1000 steps, learned-range variance, epsilon prediction, clipping at +-2, "leading"
    timesteps 0, r, 2r, ... without offset, no thresholding).  Values that would change that arithmetic (an absent key
    counts as diffusers' default) and unknown keys raise one K2Error naming them.  The released kandinsky-2-2-decoder file
    lacks variance_type and clip_sample_range (DESIGN.md section 7, the scheduler finding), so it is refused here."""
    _check_keys(config, _DDPM_FIXED, (), _DDPM_IGNORED, "scheduler_config.json")


# ------------------------------------------------------------------------------------------------ the decoder folder
_PIPELINE_TASKS = {"KandinskyV22Pipeline": "text2img", "KandinskyV22Img2ImgPipeline": "text2img",
                   "KandinskyV22InpaintPipeline": "inpainting", "KandinskyV22InpaintCombinedPipeline": "inpainting",
                   "KandinskyV22ControlnetPipeline": "controlnet", "KandinskyV22ControlnetImg2ImgPipeline": "controlnet"}
_COMPONENTS = {"unet": "UNet2DConditionModel", "movq": "VQModel", "scheduler": "DDPMScheduler"}


def read_decoder_folder(path, what="Kandinsky2_2.from_pretrained"):
    """A local Kandinsky 2.2 decoder folder (diffusers layout) -> (config, task_type, UNet state dict, MoVQ state dict): config
    is CONFIG_2_2 with the model_config of unet/config.json and the MoVQ parameters of movq/config.json, the state dicts are
    in this package's names on the CPU, as stored (the pipeline's fp16 parameters round them on load).
        model_index.json   _class_name: a KandinskyV22 decoder pipeline, which gives the task ("text2img" for the text2img
                           and img2img pipelines, "inpainting", "controlnet"); a unet/config.json of another task is refused
        unet/              config.json, diffusion_pytorch_model{,.fp16}.{safetensors,bin}
        movq/              config.json, diffusion_pytorch_model{,.fp16}.{safetensors,bin}
        scheduler/         scheduler_config.json (checked against create_ddpm_v22, check_scheduler_config)
    Every config is read before any weights.  A missing file raises K2Error naming it."""
    index = read_json(path, "model_index.json", what)
    name = index.get("_class_name")
    if name not in _PIPELINE_TASKS:
        raise K2Error(f"{what}: {os.path.join(path, 'model_index.json')}: _class_name {name!r} is not a Kandinsky 2.2 "
                      f"decoder pipeline ({', '.join(_PIPELINE_TASKS)})")
    for comp, cls in _COMPONENTS.items():
        entry = index.get(comp)   # diffusers writes [library, class name]
        if entry is not None and not (isinstance(entry, list) and len(entry) == 2 and entry[1] == cls):
            raise K2Error(f"{what}: model_index.json: {comp} = {entry!r}, not [library, {cls!r}]")
    task = _PIPELINE_TASKS[name]
    sub = {comp: os.path.join(path, comp) for comp in _COMPONENTS}
    mc, unet_task = unet_config(read_json(sub["unet"], "config.json", what))
    if unet_task != task:
        raise K2Error(f"{what}: unet/config.json describes a {unet_task} UNet, model_index.json a {name} ({task})")
    dd, n_embed, embed_dim = movq_config(read_json(sub["movq"], "config.json", what))
    check_scheduler_config(read_json(sub["scheduler"], "scheduler_config.json", what))
    unet_sd = unet_state_dict_to_k2(load_weights(sub["unet"], WEIGHT_FILES, what), create_decoder_unet(mc, task, "meta"))
    movq_sd = diffusers_movq_to_k2(load_weights(sub["movq"], WEIGHT_FILES, what), dd)
    config = deepcopy(CONFIG_2_2)
    config["model_config"] = mc
    config["image_enc_params"]["params"] = dict(embed_dim=embed_dim, n_embed=n_embed, ddconfig=dd)
    return config, task, unet_sd, movq_sd


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

    @classmethod
    def from_pretrained(cls, path, device="cuda"):
        """A local diffusers UNet folder (the `unet/` of kandinsky-2-2-decoder, -decoder-inpaint or -controlnet-depth):
        config.json (unet_config gives the geometry and the task) and diffusion_pytorch_model{,.fp16}.{safetensors,bin}, cast
        to fp16 parameters.  A missing file, and a key the geometry has no parameter for or lacks, raise K2Error naming it."""
        what = "K2UNet2DConditionModel.from_pretrained"
        mc, task = unet_config(read_json(path, "config.json", what))
        unet = create_decoder_unet(mc, task, device)
        unet.load_state_dict(unet_state_dict_to_k2(load_weights(path, WEIGHT_FILES, what), unet))
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
