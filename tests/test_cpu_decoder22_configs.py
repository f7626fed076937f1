"""CPU: the config files of the Kandinsky 2.2 decoder folders (kandinsky2.diffusers_compat.unet_config,
check_scheduler_config, read_decoder_folder).

  - unet/config.json of kandinsky-2-2-decoder, as restated here (UNET_22), gives CONFIG_2_2["model_config"] exactly; the
    inpainting (in_channels 9) and ControlNet-depth (8, addition_embed_type "image_hint") variants give their tasks, and for each
    of the three the UNet built from the result has exactly the key set diffusers_unet_to_k2 produces from a diffusers state
    dict of that geometry (oracle/unet_oracle.py's keys, the matching stem and hint stem);
  - every refusal of the UNet and scheduler readers names its key; the scheduler values create_ddpm_v22 computes are accepted;
  - a decoder folder is refused, naming the file or the key, before any weights are read."""
import json
import os

import pytest
import torch

from oracle import unet_oracle as uo

# unet/config.json of kandinsky-community/kandinsky-2-2-decoder, restated from diffusers' UNet2DConditionModel (unpinned)
UNET_22 = {
    "_class_name": "UNet2DConditionModel", "_diffusers_version": "0.18.0.dev0", "act_fn": "silu",
    "addition_embed_type": "image", "addition_embed_type_num_heads": 64, "addition_time_embed_dim": None,
    "attention_head_dim": 64, "block_out_channels": [384, 768, 1152, 1536], "center_input_sample": False,
    "class_embed_type": None, "class_embeddings_concat": False, "conv_in_kernel": 3, "conv_out_kernel": 3,
    "cross_attention_dim": 768, "cross_attention_norm": None,
    "down_block_types": ["ResnetDownsampleBlock2D", "SimpleCrossAttnDownBlock2D", "SimpleCrossAttnDownBlock2D",
                         "SimpleCrossAttnDownBlock2D"],
    "downsample_padding": 1, "dual_cross_attention": False, "encoder_hid_dim": 1280, "encoder_hid_dim_type": "image_proj",
    "flip_sin_to_cos": True, "freq_shift": 0, "in_channels": 4, "layers_per_block": 3, "mid_block_only_cross_attention": None,
    "mid_block_scale_factor": 1, "mid_block_type": "UNetMidBlock2DSimpleCrossAttn", "norm_eps": 1e-05, "norm_num_groups": 32,
    "num_class_embeds": None, "only_cross_attention": False, "out_channels": 8, "projection_class_embeddings_input_dim": None,
    "resnet_out_scale_factor": 1.0, "resnet_skip_time_act": False, "resnet_time_scale_shift": "scale_shift",
    "sample_size": 64, "time_cond_proj_dim": None, "time_embedding_act_fn": None, "time_embedding_dim": None,
    "time_embedding_type": "positional", "timestep_post_act": None,
    "up_block_types": ["SimpleCrossAttnUpBlock2D", "SimpleCrossAttnUpBlock2D", "SimpleCrossAttnUpBlock2D",
                       "ResnetUpsampleBlock2D"],
    "upcast_attention": False, "use_linear_projection": False}
UNET_22_INPAINT = dict(UNET_22, in_channels=9)
UNET_22_CONTROLNET = dict(UNET_22, in_channels=8, addition_embed_type="image_hint")
# the DDPMScheduler create_ddpm_v22 computes
SCHEDULER_22 = {"_class_name": "DDPMScheduler", "_diffusers_version": "0.18.0.dev0", "beta_end": 0.012,
                "beta_schedule": "linear", "beta_start": 0.00085, "clip_sample": True, "clip_sample_range": 2.0,
                "dynamic_thresholding_ratio": 0.995, "num_train_timesteps": 1000, "prediction_type": "epsilon",
                "sample_max_value": 1.0, "steps_offset": 0, "thresholding": False, "timestep_spacing": "leading",
                "trained_betas": None, "variance_type": "learned_range"}
# diffusers ImageHintTimeEmbedding.input_hint_block: its eight 3x3 convolutions (Cin, Cout), SiLU between them
_HINT_CONVS = [(3, 16), (16, 16), (16, 32), (32, 32), (32, 96), (96, 96), (96, 256), (256, 4)]


def test_released_unet_config_is_config_2_2():
    from kandinsky2.configs import CONFIG_2_2
    from kandinsky2.diffusers_compat import unet_config
    assert unet_config(UNET_22) == (CONFIG_2_2["model_config"], "text2img")
    assert unet_config(UNET_22_INPAINT) == (CONFIG_2_2["model_config"], "inpainting")
    assert unet_config(UNET_22_CONTROLNET) == (CONFIG_2_2["model_config"], "controlnet")
    assert unet_config(dict(UNET_22, attention_head_dim=[64] * 4, layers_per_block=[3] * 4))[0] == CONFIG_2_2["model_config"]


def _diffusers_keys(cfg, hint):
    """{diffusers key: meta tensor} of a decoder UNet at the oracle's geometry cfg (k2_to_diffusers_unet of its keys)."""
    from kandinsky2.checkpoints import k2_to_diffusers_unet
    sd = {k: torch.empty(s, device="meta") for k, s in uo.unet_param_spec(cfg)}
    d = k2_to_diffusers_unet(sd, in_channels=2 * cfg["in_channels"] + 1 if cfg["inpainting"] else cfg["in_channels"],
                             model_channels=cfg["model_channels"], channel_mult=tuple(cfg["channel_mult"]),
                             num_res_blocks=cfg["num_res_blocks"], attention_ds=tuple(cfg["attention_ds"]))
    if hint:
        for i, (ci, co) in enumerate(_HINT_CONVS):
            d[f"add_embedding.input_hint_block.{2 * i}.weight"] = torch.empty(co, ci, 3, 3, device="meta")
            d[f"add_embedding.input_hint_block.{2 * i}.bias"] = torch.empty(co, device="meta")
    return d


@pytest.mark.parametrize("config,oracle_cfg,hint", [
    (UNET_22, dict(uo.CONFIG_2_2), False),
    (UNET_22_INPAINT, dict(uo.CONFIG_2_2, inpainting=True), False),
    (UNET_22_CONTROLNET, dict(uo.CONFIG_2_2, in_channels=8), True)], ids=["text2img", "inpainting", "controlnet"])
def test_unet_config_builds_the_key_set_of_the_remap(config, oracle_cfg, hint):
    from kandinsky2.checkpoints import diffusers_unet_to_k2
    from kandinsky2.diffusers_compat import unet_config, unet_state_dict_to_k2
    from kandinsky2.model.model_creation import create_decoder_unet
    mc, task = unet_config(config)
    model = create_decoder_unet(mc, task, "meta")
    have = {k: tuple(v.shape) for k, v in model.state_dict().items()}
    dsd = _diffusers_keys(oracle_cfg, hint)
    remapped = diffusers_unet_to_k2(dsd, in_channels=config["in_channels"], model_channels=384, channel_mult=(1, 2, 3, 4),
                                    num_res_blocks=3, attention_ds=(2, 4, 8))
    assert {k: tuple(v.shape) for k, v in remapped.items()} == have
    assert {k: tuple(v.shape) for k, v in unet_state_dict_to_k2(dsd, model).items()} == have


def test_unet_state_dict_refusals_name_the_key():
    from kandinsky2._native import K2Error
    from kandinsky2.diffusers_compat import unet_config, unet_state_dict_to_k2
    from kandinsky2.model.model_creation import create_decoder_unet
    model = create_decoder_unet(*unet_config(UNET_22_CONTROLNET), "meta")
    dsd = _diffusers_keys(dict(uo.CONFIG_2_2, in_channels=8), True)
    with pytest.raises(K2Error, match=r"unknown keys \['mid_block.attentions.0.norm_cross.weight'\]"):
        unet_state_dict_to_k2(dict(dsd, **{"mid_block.attentions.0.norm_cross.weight": torch.empty(1)}), model)
    gone = {k: v for k, v in dsd.items() if not k.startswith("add_embedding.input_hint_block.14.")}
    with pytest.raises(K2Error, match=r"missing keys \['add_embedding.input_hint_block.14.weight', "):
        unet_state_dict_to_k2(gone, model)


@pytest.mark.parametrize("key,value", [
    ("down_block_types", ["ResnetDownsampleBlock2D", "CrossAttnDownBlock2D", "SimpleCrossAttnDownBlock2D",
                          "SimpleCrossAttnDownBlock2D"]),
    ("up_block_types", ["SimpleCrossAttnUpBlock2D", "SimpleCrossAttnUpBlock2D", "ResnetUpsampleBlock2D",
                        "ResnetUpsampleBlock2D"]),
    ("mid_block_type", "UNetMidBlock2DCrossAttn"), ("resnet_time_scale_shift", "default"),
    ("encoder_hid_dim_type", "text_proj"), ("attention_head_dim", 32), ("attention_head_dim", [64, 64, 64, 32]),
    ("norm_num_groups", 16), ("norm_eps", 1e-6), ("act_fn", "gelu"), ("time_embedding_type", "fourier"),
    ("class_embed_type", "timestep"), ("only_cross_attention", True), ("flip_sin_to_cos", False),
    ("in_channels", 5), ("addition_embed_type", "text"), ("out_channels", 4), ("block_out_channels", [384, 768, 1100, 1536]),
    ("layers_per_block", [3, 3, 2, 3]), ("a_key_from_a_newer_diffusers", 0)])
def test_unet_config_refusals_name_the_key(key, value):
    from kandinsky2._native import K2Error
    from kandinsky2.diffusers_compat import unet_config
    with pytest.raises(K2Error, match=key):
        unet_config(dict(UNET_22, **{key: value}))


def test_unet_config_reads_a_smaller_geometry():
    from kandinsky2.diffusers_compat import unet_config
    mc, task = unet_config(dict(UNET_22, block_out_channels=[64, 128], layers_per_block=1, cross_attention_dim=128,
                                down_block_types=["ResnetDownsampleBlock2D", "SimpleCrossAttnDownBlock2D"],
                                up_block_types=["SimpleCrossAttnUpBlock2D", "ResnetUpsampleBlock2D"]))
    assert task == "text2img"
    assert (mc["num_channels"], mc["channel_mult"], mc["num_res_blocks"], mc["attention_resolutions"], mc["model_dim"]) == \
        (64, "1,2", 1, "32", 128)


def test_scheduler_config_accepts_what_create_ddpm_v22_computes():
    from kandinsky2.diffusers_compat import check_scheduler_config
    check_scheduler_config(SCHEDULER_22)
    check_scheduler_config(dict(SCHEDULER_22, dynamic_thresholding_ratio=0.9, sample_max_value=3.0))   # thresholding is off
    check_scheduler_config({k: v for k, v in SCHEDULER_22.items() if k in ("beta_start", "beta_end", "variance_type",
                                                                            "clip_sample_range")})   # the rest at the defaults


@pytest.mark.parametrize("key,value", [
    ("_class_name", "DDIMScheduler"), ("num_train_timesteps", 2000), ("beta_start", 0.0001), ("beta_end", 0.02),
    ("beta_schedule", "scaled_linear"), ("trained_betas", [0.1] * 1000), ("variance_type", "fixed_small"),
    ("prediction_type", "v_prediction"), ("clip_sample", False), ("clip_sample_range", 1.0), ("thresholding", True),
    ("timestep_spacing", "trailing"), ("steps_offset", 1), ("rescale_betas_zero_snr", True), ("variance_typo", 1)])
def test_scheduler_refusals_name_the_key(key, value):
    from kandinsky2._native import K2Error
    from kandinsky2.diffusers_compat import check_scheduler_config
    with pytest.raises(K2Error, match=key):
        check_scheduler_config(dict(SCHEDULER_22, **{key: value}))


# What the reference's notebooks/lora_decoder.ipynb records of the released kandinsky-2-2-decoder scheduler_config.json
# (317 bytes): DDPMScheduler.from_pretrained reports trained_betas, sample_max_value, dynamic_thresholding_ratio,
# clip_sample_range, variance_type and timestep_spacing "not found in config".  The values of the keys it holds are not
# recorded; here they are the ones create_ddpm_v22 computes, the most favourable case.
RELEASED_ABSENT = ("trained_betas", "sample_max_value", "dynamic_thresholding_ratio", "clip_sample_range", "variance_type",
                   "timestep_spacing")


def test_the_released_scheduler_config_is_refused_on_its_absent_keys():
    from kandinsky2._native import K2Error
    from kandinsky2.diffusers_compat import check_scheduler_config
    released = {k: v for k, v in SCHEDULER_22.items() if k not in RELEASED_ABSENT}
    with pytest.raises(K2Error) as e:
        check_scheduler_config(released)
    msg = str(e.value)
    assert "variance_type = 'fixed_small', absent: diffusers' default" in msg
    assert "clip_sample_range = 1.0, absent: diffusers' default" in msg
    assert "timestep_spacing" not in msg        # diffusers' default, "leading", is what create_ddpm_v22 computes


def test_one_refusal_names_every_offending_key_values_first():
    from kandinsky2._native import K2Error
    from kandinsky2.diffusers_compat import check_scheduler_config
    with pytest.raises(K2Error) as e:
        check_scheduler_config(dict(SCHEDULER_22, steps_offset=1, clip_sample=False, set_alpha_to_one=False))
    msg = str(e.value)
    assert msg.index("clip_sample = False") < msg.index("steps_offset = 1") < msg.index("unknown keys ['set_alpha_to_one']")


def _write_configs(root, pipeline="KandinskyV22Pipeline", unet=UNET_22):
    from tests.movq22_oracle import VQMODEL_22
    files = {"model_index.json": {"_class_name": pipeline, "unet": ["diffusers", "UNet2DConditionModel"],
                                  "movq": ["diffusers", "VQModel"], "scheduler": ["diffusers", "DDPMScheduler"]},
             "unet/config.json": unet, "movq/config.json": VQMODEL_22, "scheduler/scheduler_config.json": SCHEDULER_22}
    for name, content in files.items():
        os.makedirs(os.path.dirname(os.path.join(root, name)), exist_ok=True)
        with open(os.path.join(root, name), "w") as f:
            json.dump(content, f)


def test_decoder_folder_refusals_name_the_file_or_key(tmp_path):
    from kandinsky2._native import K2Error
    from kandinsky2.diffusers_compat import read_decoder_folder
    root = str(tmp_path / "decoder")
    _write_configs(root)
    with pytest.raises(K2Error, match=r"unet/diffusion_pytorch_model.safetensors or .*fp16.bin not found"):
        read_decoder_folder(root)     # every config read, then the weights
    _write_configs(root, pipeline="KandinskyV22InpaintPipeline")
    with pytest.raises(K2Error, match="text2img UNet, model_index.json a KandinskyV22InpaintPipeline"):
        read_decoder_folder(root)
    for entry in ("UNet2DConditionModel", [], ["diffusers", "UNet2DModel"]):
        _write_configs(root)
        with open(os.path.join(root, "model_index.json")) as f:
            index = json.load(f)
        with open(os.path.join(root, "model_index.json"), "w") as f:
            json.dump(dict(index, unet=entry), f)
        with pytest.raises(K2Error, match=r"model_index.json: unet = .*, not \[library, 'UNet2DConditionModel'\]"):
            read_decoder_folder(root)
    _write_configs(root, pipeline="StableDiffusionPipeline")
    with pytest.raises(K2Error, match="_class_name 'StableDiffusionPipeline'"):
        read_decoder_folder(root)
    _write_configs(root, pipeline="KandinskyV22ControlnetPipeline", unet=UNET_22_CONTROLNET)
    with open(os.path.join(root, "scheduler", "scheduler_config.json"), "w") as f:
        json.dump(dict(SCHEDULER_22, steps_offset=1), f)
    with pytest.raises(K2Error, match="steps_offset"):
        read_decoder_folder(root)
    for name in ("scheduler/scheduler_config.json", "movq/config.json", "unet/config.json", "model_index.json"):
        os.remove(os.path.join(root, name))
        with pytest.raises(K2Error, match=name.replace("/", r"[/\\]")):
            read_decoder_folder(root)
