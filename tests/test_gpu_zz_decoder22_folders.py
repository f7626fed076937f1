"""GPU: the Kandinsky 2.2 decoders loaded from their folders in the diffusers layout, on tiny folders written here
(model_index.json, unet/, movq/, scheduler/; text2img, inpainting and ControlNet-depth; safetensors and .bin):

  - MOVQ.from_pretrained decodes and encodes bit for bit like MOVQ.load_state_dict of the same weights under the reference's
    names;
  - Kandinsky2_2.from_pretrained gives the images of a pipeline built by hand from the same state dicts (unet_state_dict= /
    movq_state_dict=), bit for bit, for generate_text2img, generate_img2img, generate_inpainting and generate_controlnet with
    the DDPM sampler and a solver sampler each; K2UNet2DConditionModel.from_pretrained equals the hand-built UNet;
  - prior= a tiny kandinsky-2-2-prior folder equals passing PriorEmbedder22.from_pretrained of it by hand;
  - a folder without movq/ or scheduler/ raises K2Error naming the file."""
import json
import os
import shutil
from copy import deepcopy

import pytest
import torch

from tests import movq22_oracle as m22
from tests.test_cpu_decoder22_configs import SCHEDULER_22, UNET_22

pytestmark = pytest.mark.gpu

PIPELINES = {"text2img": "KandinskyV22Pipeline", "inpainting": "KandinskyV22InpaintPipeline",
             "controlnet": "KandinskyV22ControlnetPipeline"}
# the geometry of tests/test_gpu_movq_sampler.py's tiny pipelines, in diffusers' config form
UNET_TINY = dict(UNET_22, block_out_channels=[64, 128], layers_per_block=1, cross_attention_dim=128,
                 down_block_types=["ResnetDownsampleBlock2D", "SimpleCrossAttnDownBlock2D"],
                 up_block_types=["SimpleCrossAttnUpBlock2D", "ResnetUpsampleBlock2D"])
UNET_IN = {"text2img": dict(in_channels=4), "inpainting": dict(in_channels=9),
           "controlnet": dict(in_channels=8, addition_embed_type="image_hint")}
MOVQ_TINY = dict(m22.VQMODEL_22, block_out_channels=[32, 32, 64, 64], layers_per_block=1, num_vq_embeddings=64)


@pytest.fixture(scope="module", autouse=True)
def bitwise():
    from kandinsky2 import launch_plan
    old = launch_plan.TUNE_SMALL_M
    launch_plan.TUNE_SMALL_M = 0     # bit-identical GEMM configurations only (as bench.py --dump-outputs)
    yield
    launch_plan.TUNE_SMALL_M = old


def _tiny_config():
    from kandinsky2.configs import CONFIG_2_2
    from tests.test_gpu_movq_sampler import _tiny_overrides
    config = deepcopy(CONFIG_2_2)
    for k, v in _tiny_overrides().items():
        config[k].update(v)
    return config


def _save(sd, folder, fmt):
    os.makedirs(folder, exist_ok=True)
    sd = {k: v.detach().contiguous().clone() for k, v in sd.items()}
    if fmt == "bin":
        torch.save(sd, os.path.join(folder, "diffusion_pytorch_model.bin"))
    else:
        from safetensors.torch import save_file
        save_file(sd, os.path.join(folder, "diffusion_pytorch_model.safetensors"))


def _json(path, content):
    os.makedirs(os.path.dirname(path), exist_ok=True)
    with open(path, "w") as f:
        json.dump(content, f)


def _write_decoder(root, task, fmt, seed):
    """A tiny decoder folder of `task` with random fp32 weights -> (config, UNet and MoVQ state dicts in this package's names)."""
    from kandinsky2.checkpoints import k2_to_diffusers_movq, k2_to_diffusers_unet
    from kandinsky2.model.model_creation import create_decoder_unet
    from kandinsky2.vqgan import MOVQ
    config = _tiny_config()
    unet = create_decoder_unet(config["model_config"], task, "cpu", torch.float32).init_synthetic_(seed)
    unet_sd = {k: v.clone() for k, v in unet.state_dict().items()}
    p = config["image_enc_params"]["params"]
    movq_sd = {k: v.clone() for k, v in MOVQ(**p, device="cpu").init_synthetic_(seed + 1).state_dict().items()}
    _save(k2_to_diffusers_unet(unet_sd, in_channels=unet.in_channels, model_channels=64, channel_mult=(1, 2), num_res_blocks=1,
                               attention_ds=(2,)), os.path.join(root, "unet"), fmt)
    _save(k2_to_diffusers_movq(movq_sd, p["ddconfig"]), os.path.join(root, "movq"), fmt)
    _json(os.path.join(root, "model_index.json"),
          {"_class_name": PIPELINES[task], "_diffusers_version": "0.18.0.dev0", "unet": ["diffusers", "UNet2DConditionModel"],
           "movq": ["diffusers", "VQModel"], "scheduler": ["diffusers", "DDPMScheduler"]})
    _json(os.path.join(root, "unet", "config.json"), dict(UNET_TINY, **UNET_IN[task]))
    _json(os.path.join(root, "movq", "config.json"), MOVQ_TINY)
    _json(os.path.join(root, "scheduler", "scheduler_config.json"), SCHEDULER_22)
    return config, unet_sd, movq_sd


def _same(a, b):
    return len(a) == len(b) and all(x.tobytes() == y.tobytes() for x, y in zip(a, b))


@pytest.mark.parametrize("fmt", ["safetensors", "bin"])
def test_movq_from_pretrained_equals_the_reference_names(tmp_path, fmt):
    from kandinsky2.vqgan import MOVQ
    config, _, movq_sd = _write_decoder(str(tmp_path / "dec"), "text2img", fmt, seed=3)
    p = config["image_enc_params"]["params"]
    a = MOVQ.from_pretrained(str(tmp_path / "dec" / "movq"))
    b = MOVQ(**p, device="cuda", param_dtype=torch.float16)
    b.load_state_dict(movq_sd)
    assert a.ddconfig == b.ddconfig and (a.n_embed, a.embed_dim) == (b.n_embed, b.embed_dim)
    assert all(torch.equal(x, y) and x.dtype == torch.float16 for x, y in zip(a.state_dict().values(), b.state_dict().values()))
    g = torch.Generator(device="cuda").manual_seed(0)
    lat = torch.randn(2, 4, 8, 8, device="cuda", generator=g)
    img = torch.rand(2, 3, 64, 64, device="cuda", generator=g) * 2 - 1
    da, db = a.decode(lat), b.decode(lat)
    ea, eb = a.encode(img), b.encode(img)
    assert torch.isfinite(da).all() and torch.equal(da, db)
    assert torch.isfinite(ea).all() and torch.equal(ea, eb)
    assert torch.equal(a.decode_to_uint8(lat), b.decode_to_uint8(lat))


@pytest.fixture(scope="module")
def folders(tmp_path_factory):
    """{task: (folder, config, UNet state dict, MoVQ state dict)}: text2img and ControlNet as safetensors, inpainting as .bin."""
    out = {}
    for i, (task, fmt) in enumerate((("text2img", "safetensors"), ("inpainting", "bin"), ("controlnet", "safetensors"))):
        root = str(tmp_path_factory.mktemp(task) / f"kandinsky-2-2-{task}")
        out[task] = (root, *_write_decoder(root, task, fmt, seed=10 + 2 * i))
    return out


def _pipelines(folders, task, hand_embedder=None, **kw):
    """(Kandinsky2_2.from_pretrained(folder, **kw), the pipeline built by hand from the folder's state dicts)."""
    from kandinsky2.pipelines import Kandinsky2_2
    root, config, unet_sd, movq_sd = folders[task]
    loaded = Kandinsky2_2.from_pretrained(root, **kw)
    hand = Kandinsky2_2(config, "cuda", task_type=task, unet_state_dict=unet_sd, movq_state_dict=movq_sd,
                        embedder=hand_embedder)
    assert loaded.task_type == task and loaded.config == config
    return loaded, hand


KW = dict(batch_size=2, decoder_steps=3, h=64, w=64)


@pytest.mark.parametrize("sampler", ["ddpm_sampler", "dpmpp_2m_sampler"])
def test_text2img_and_img2img_equal_the_hand_built_pipeline(folders, sampler):
    loaded, hand = _pipelines(folders, "text2img")
    a = loaded.generate_text2img("a red cat", sampler=sampler, **KW)
    assert len(a) == 2 and a[0].size == (64, 64)
    assert _same(a, hand.generate_text2img("a red cat", sampler=sampler, **KW))
    from PIL import Image
    img = Image.new("RGB", (64, 64), (200, 40, 90))
    i2i = sampler.replace("dpmpp_2m", "unipc")
    assert _same(loaded.generate_img2img("a hat", img, strength=0.6, sampler=i2i, **KW),
                 hand.generate_img2img("a hat", img, strength=0.6, sampler=i2i, **KW))


@pytest.mark.parametrize("sampler", ["ddpm_sampler", "unipc_sampler"])
def test_inpainting_equals_the_hand_built_pipeline(folders, sampler):
    loaded, hand = _pipelines(folders, "inpainting")
    lat = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(1))
    mask = torch.ones(64, 64)
    mask[:, 40:] = 0
    a = loaded.generate_inpainting("a hat", lat, mask.numpy(), sampler=sampler, **KW)
    assert len(a) == 2 and _same(a, hand.generate_inpainting("a hat", lat, mask.numpy(), sampler=sampler, **KW))


@pytest.mark.parametrize("sampler", ["ddpm_sampler", "dpmpp_2m_sampler"])
def test_controlnet_equals_the_hand_built_pipeline(folders, sampler):
    marker = object()
    loaded, hand = _pipelines(folders, "controlnet", depth_estimator=marker)
    assert loaded.depth_estimator is marker
    hint = torch.rand(1, 3, 64, 64, generator=torch.Generator().manual_seed(3))
    a = loaded.generate_controlnet("a red cat", hint, sampler=sampler, **KW)
    assert len(a) == 2 and _same(a, hand.generate_controlnet("a red cat", hint, sampler=sampler, **KW))


@pytest.mark.parametrize("task", ["text2img", "controlnet"])
def test_unet_from_pretrained_equals_the_hand_built_unet(folders, task):
    from kandinsky2.diffusers_compat import K2UNet2DConditionModel
    from kandinsky2.model.model_creation import create_decoder_unet
    root, config, unet_sd, _ = folders[task]
    a = K2UNet2DConditionModel.from_pretrained(os.path.join(root, "unet"))
    b = create_decoder_unet(config["model_config"], task, "cuda")
    b.load_state_dict(unet_sd)
    assert a.unet.state_dict().keys() == b.state_dict().keys()
    assert all(torch.equal(x, y) for x, y in zip(a.unet.state_dict().values(), b.state_dict().values()))
    g = torch.Generator(device="cuda").manual_seed(4)
    x = torch.randn(2, 4, 8, 8, device="cuda", generator=g)
    emb = torch.randn(2, 1280, device="cuda", generator=g)
    t = torch.tensor([999.0, 10.0], device="cuda")
    kw = {"hint": torch.rand(2, 3, 64, 64, device="cuda", generator=g)} if task == "controlnet" else {}
    y = a(x, t, added_cond_kwargs={"image_embeds": emb, **kw}).sample
    assert torch.isfinite(y).all() and torch.equal(y, K2UNet2DConditionModel(b)(x, t, added_cond_kwargs={"image_embeds": emb,
                                                                                                        **kw}).sample)


def test_prior_folder_equals_the_embedder_passed_by_hand(folders, tmp_path):
    from kandinsky2.model.prior import PriorEmbedder22
    from oracle import synth
    from tests import prior22_oracle as p22
    from tests import test_gpu_zz_clip_text as ct
    fx = torch.load(ct.cto.FIXTURE)
    prior_root = str(tmp_path / "kandinsky-2-2-prior")
    ct._write_folder(prior_root, fx, synth.synth_state_dict(p22.diffusers_prior_spec(ct.PRIOR_CFG), seed=13),
                     ct._tiny_cfg(fx, projection_dim=1280), 9, "safetensors")
    loaded, hand = _pipelines(folders, "text2img", hand_embedder=PriorEmbedder22.from_pretrained(prior_root), prior=prior_root)
    assert isinstance(loaded.embedder, PriorEmbedder22) and loaded.embedder is not hand.embedder
    kw = dict(KW, prior_steps=3, negative_prior_prompt="low quality")
    a = loaded.generate_text2img("a red cat", **kw)
    assert _same(a, hand.generate_text2img("a red cat", **kw))


@pytest.mark.parametrize("missing", ["movq", "scheduler"])
def test_a_missing_component_is_named(folders, tmp_path, missing):
    from kandinsky2._native import K2Error
    from kandinsky2.pipelines import Kandinsky2_2
    root = str(tmp_path / "decoder")
    shutil.copytree(folders["text2img"][0], root)
    shutil.rmtree(os.path.join(root, missing))
    name = "config.json" if missing == "movq" else "scheduler_config.json"
    with pytest.raises(K2Error, match=os.path.join(root, missing, name).replace("\\", "\\\\")):
        Kandinsky2_2.from_pretrained(root)
