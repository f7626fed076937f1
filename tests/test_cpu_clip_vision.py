"""CPU: the CLIP image tower's host side.  The restated forward (tests/clip_vision_oracle.py) against transformers' own outputs
in tests/golden/clip_vision_tiny.pt, the state-dict remap through the network, preprocess against CLIPImageProcessor's crops and
normalised values, the config refusals, and the two new C-ABI entry points' argument checks (no device needed: nothing is
launched).  Where transformers is importable, a second seed runs against it live."""
import copy

import pytest
import torch

from tests import clip_vision_oracle as cvo
from tests.test_cpu_vector_arg_checks import A, P, _refused, _with


@pytest.fixture(scope="module")
def fx():
    return torch.load(cvo.FIXTURE)


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


@pytest.mark.parametrize("i", [0, 1])
def test_oracle_equals_transformers_golden(fx, i):
    t = fx["towers"][i]
    sd = cvo.synth_weights(t["cfg"], t["weight_seed"])
    hid, emb = cvo.forward(sd, t["cfg"], cvo.tower_pixels(t))
    assert _rel(hid, t["last_hidden_state"]) <= 1e-5 and _rel(emb, t["image_embeds"]) <= 1e-5


@pytest.mark.parametrize("i", [0, 1])
def test_remapped_forward_equals_transformers_names(fx, i):
    from kandinsky2.checkpoints import transformers_clip_vision_to_k2
    t = fx["towers"][i]
    sd = cvo.synth_weights(t["cfg"], t["weight_seed"])
    sd_pos = dict(sd, **{"vision_model.embeddings.position_ids": torch.arange(5)[None]})   # a stray buffer is ignored
    k2 = transformers_clip_vision_to_k2(sd_pos)
    pix = cvo.tower_pixels(t)
    a = cvo.forward(sd, t["cfg"], pix)
    b = cvo.forward_k2(k2, t["cfg"], pix)
    for x, y in zip(a, b):
        assert _rel(x, y) <= 1e-6


def test_remap_refuses_missing_and_unexpected_keys(fx):
    from kandinsky2._native import K2Error
    from kandinsky2.checkpoints import transformers_clip_vision_to_k2
    sd = cvo.synth_weights(cvo.CONFIG_TINY, 0)
    gone = "vision_model.encoder.layers.1.mlp.fc2.bias"
    with pytest.raises(K2Error, match=gone.replace(".", r"\.")):
        transformers_clip_vision_to_k2({k: v for k, v in sd.items() if k != gone})
    with pytest.raises(K2Error, match="text_projection"):
        transformers_clip_vision_to_k2(dict(sd, **{"text_projection.weight": torch.zeros(2, 2)}))


def test_preprocess_reproduces_clip_image_processor(fx):
    from kandinsky2.model.clip_vision import DEFAULT_PREPROCESSOR, preprocess_images
    for name, img in cvo.sample_images():
        crop = preprocess_images(img, dict(DEFAULT_PREPROCESSOR, do_rescale=False, do_normalize=False))[0]
        assert torch.equal(crop, crop.to(torch.uint8).float()), name              # whole numbers in [0, 255]
        crop = crop.to(torch.uint8)
        assert torch.equal(crop[:, :1], fx["crop_rows"][name]), name
        assert cvo.sha256(crop) == fx["crop_sha256"][name], name                   # the whole crop, exactly
        pv = preprocess_images(img)[0]
        assert pv.shape == (3, 224, 224) and pv.dtype == torch.float32
        assert (pv[:, :1] - fx["normalised_rows"][name]).abs().max().item() <= 1e-6, name


@pytest.mark.parametrize("change,msg", [
    (dict(hidden_act="quick_gelu"), "hidden_act"),
    (dict(hidden_act=None), "hidden_act"),
    (dict(hidden_size=1280, num_attention_heads=20), "head width 64"),
    (dict(num_attention_heads=4), "head width 52"),
    (dict(image_size=60), "multiple of patch_size"),
])
def test_from_transformers_refuses_unimplemented_configs(change, msg):
    from kandinsky2._native import K2Error
    from kandinsky2.model.clip_vision import CLIPVisionTower
    cfg = dict(cvo.CONFIG_TINY, **change)
    if cfg["hidden_act"] is None:
        del cfg["hidden_act"]              # transformers' default is quick_gelu
    with pytest.raises(K2Error, match=msg):
        CLIPVisionTower.from_transformers(cvo.synth_weights(cvo.CONFIG_TINY, 0), cfg, device="cpu")


def test_tower_refuses_weights_that_do_not_fit_the_config():
    from kandinsky2._native import K2Error
    from kandinsky2.checkpoints import transformers_clip_vision_to_k2
    from kandinsky2.model.clip_vision import CLIPVisionTower
    sd = transformers_clip_vision_to_k2(cvo.synth_weights(cvo.CONFIG_TINY, 0))
    with pytest.raises(K2Error, match="mlp.fc1.weight"):
        CLIPVisionTower(sd, dict(cvo.CONFIG_TINY, intermediate_size=512), device="cpu")


# k2_attention_heads(qkv, ldq, hs, q_off, k_off, v_off, B, heads, T, head_dim, scale, out, ldo, ohs, stream)
HEADS = dict(qkv=P(A), ldq=4992, hs=312, q_off=0, k_off=104, v_off=208, B=2, heads=16, T=257, head_dim=104, scale=0.098,
             out=P(A), ldo=1664, ohs=104, stream=None)


@pytest.mark.parametrize("change,msg", [
    (dict(head_dim=64), "head width 104"),
    (dict(head_dim=112), "head width 104"),
    (dict(qkv=None), "bad arguments"),
    (dict(out=None), "bad arguments"),
    (dict(B=0), "bad arguments"),
    (dict(heads=0), "bad arguments"),
    (dict(T=0), "bad arguments"),
    (dict(ldq=4996), "multiples of 8"),
    (dict(ldo=1660), "multiples of 8"),
    (dict(hs=316), "multiples of 8"),
    (dict(k_off=100), "multiples of 8"),
    (dict(ohs=100), "multiples of 8"),
    (dict(q_off=-8), "non-negative"),
    (dict(ldq=4984), "qkv row narrower"),
    (dict(ldo=1656), "output row narrower"),
    (dict(ohs=96), "output row narrower"),
    (dict(qkv=P(A + 8)), "alignment"),
    (dict(out=P(A + 2)), "alignment"),
])
def test_attention_heads_refuses(change, msg):
    _refused("k2_attention_heads", list(_with(HEADS, **change).values()), msg)


# k2_clip_patchify(x, B, S, P, out, ldo, Kp, stream)
PATCH = dict(x=P(A), B=2, S=224, P=14, out=P(A), ldo=640, Kp=640, stream=None)


@pytest.mark.parametrize("change,msg", [
    (dict(x=None), "bad arguments"),
    (dict(out=None), "bad arguments"),
    (dict(B=0), "bad arguments"),
    (dict(P=0), "bad arguments"),
    (dict(S=230), "multiple of the patch size"),
    (dict(Kp=588), "Kp must hold"),
    (dict(ldo=632), "Kp must hold"),
    (dict(x=P(A + 2)), "alignment"),
    (dict(out=P(A + 1)), "alignment"),
])
def test_clip_patchify_refuses(change, msg):
    _refused("k2_clip_patchify", list(_with(PATCH, **change).values()), msg)


def test_live_transformers_second_seed():
    pytest.importorskip("transformers")
    from kandinsky2.model.clip_vision import preprocess_images
    for cfg in (cvo.CONFIG_TINY, cvo.CONFIG_TINY_26):
        sd = cvo.synth_weights(cfg, 17)
        pix = torch.randn(2, 3, cfg["image_size"], cfg["image_size"], generator=torch.Generator().manual_seed(17))
        ref = cvo.transformers_outputs(copy.deepcopy(sd), cfg, pix)
        got = cvo.forward(sd, cfg, pix)
        assert all(_rel(g, r) <= 1e-5 for g, r in zip(got, ref))
    for name, img in cvo.sample_images():
        crop, pv = cvo.transformers_preprocess(img)
        assert (preprocess_images(img)[0] - pv).abs().max().item() <= 1e-6, name
