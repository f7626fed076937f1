"""CPU: the DPT depth estimator's host side (kandinsky2/model/depth.py, checkpoints.transformers_dpt_to_k2) against
tests/golden/dpt_tiny.pt (written by transformers) and, where transformers is installed, against transformers run live on a
second seed: the oracle (tests/dpt_oracle.py), the preprocessing, the weight remap through the network, every config
refusal, the refusal of unknown and missing keys, and the pipeline's postprocess bit for bit."""
import numpy as np
import pytest
import torch

from tests import dpt_oracle as do


@pytest.fixture(scope="module")
def fx():
    return torch.load(do.FIXTURE)


def _tiny(name):
    return {n: (cfg, proc) for n, cfg, proc in do.TINY}[name]


@pytest.mark.parametrize("name", ["even", "odd"])
def test_oracle_and_preprocess_against_golden(fx, name):
    from kandinsky2.model.depth import preprocess_images, preprocessor_settings
    g = fx["configs"][name]
    cfg, proc = _tiny(name)
    assert g["config"] == cfg and g["preprocessor"] == proc
    images = [img for _, img in do.sample_images(fx["image_seed"])]
    pix = preprocess_images(images, preprocessor_settings(proc, cfg["image_size"]), proc["size"]["height"])
    assert (pix - g["pixel_values"]).abs().max().item() <= 1e-6
    ref = g["predicted_depth"]
    got = do.forward(do.synth_weights(cfg, fx["weight_seed"]), cfg, g["pixel_values"])
    assert got.shape == ref.shape and ((got - ref).norm() / ref.norm()).item() <= 1e-5
    assert (ref > 0).float().mean().item() > 0.5      # the synthetic weights give a map that is not degenerate


@pytest.mark.parametrize("name", ["even", "odd"])
def test_postprocess_bit_equal_to_the_pipeline(fx, name):
    from kandinsky2.model.depth import depth_image
    g = fx["configs"][name]
    for (_, img), pred, u8 in zip(do.sample_images(fx["image_seed"]), g["pipeline_predicted_depth"], g["depth_u8"]):
        got = np.array(depth_image(pred, img.size[1], img.size[0]))
        assert got.dtype == np.uint8 and got.shape == tuple(u8.shape) and np.array_equal(got, u8.numpy())


def test_postprocess_of_a_constant_map_is_zero():
    from kandinsky2.model.depth import depth_image
    assert not np.array(depth_image(torch.full((8, 8), 3.0), 8, 8)).any()     # same size: the resize is a copy


def _back_to_transformers(k2, sd):
    """Inverse of transformers_dpt_to_k2 on the keys the network reads (the dropped ones are taken from sd)."""
    from kandinsky2.checkpoints import _DPT_LAYER, _DPT_TOP, unpack_heads
    out = {d: k2[k] for k, d in _DPT_TOP.items()}
    out["dpt.embeddings.cls_token"] = k2["cls_token"].reshape(1, 1, -1)
    out["dpt.embeddings.position_embeddings"] = k2["position_embedding"][None]
    L = sum(1 for k in k2 if k.endswith("attn.qkv.weight"))
    for i in range(L):
        for d, k in _DPT_LAYER.items():
            for s in ("weight", "bias"):
                out[f"dpt.encoder.layer.{i}.{d}.{s}"] = k2[f"layers.{i}.{k}.{s}"]
        for s in ("weight", "bias"):
            for n, t in zip(("query", "key", "value"), unpack_heads(k2[f"layers.{i}.attn.qkv.{s}"], 3, 64)):
                out[f"dpt.encoder.layer.{i}.attention.attention.{n}.{s}"] = t
    out.update({k: v for k, v in k2.items() if k.startswith(("neck.", "head."))})
    return out


@pytest.mark.parametrize("name", ["even", "odd"])
def test_remap_through_the_network(fx, name):
    from kandinsky2.checkpoints import transformers_dpt_to_k2
    from kandinsky2.model.depth import dpt_config, k2_shapes
    cfg, _ = _tiny(name)
    sd = do.synth_weights(cfg, 5)
    k2 = transformers_dpt_to_k2(sd, cfg)
    shapes = k2_shapes(dpt_config(cfg))
    assert set(k2) == set(shapes) and all(tuple(k2[k].shape) == s for k, s in shapes.items())
    assert not any(k.startswith(("dpt.layernorm", "neck.fusion_stage.layers.0.residual_layer1")) for k in k2)
    back = _back_to_transformers(k2, sd)
    pix = fx["configs"][name]["pixel_values"][:2]
    assert torch.equal(do.forward(back, cfg, pix), do.forward(sd, cfg, pix))


def test_remap_refuses_unknown_and_missing_keys():
    from kandinsky2._native import K2Error
    from kandinsky2.checkpoints import transformers_dpt_to_k2
    cfg, _ = _tiny("even")
    sd = do.synth_weights(cfg, 5)
    with pytest.raises(K2Error, match=r"unknown keys \['dpt.pooler.dense.weight'\]"):
        transformers_dpt_to_k2(dict(sd, **{"dpt.pooler.dense.weight": torch.zeros(1)}), cfg)
    for gone in ("dpt.layernorm.bias", "neck.fusion_stage.layers.0.residual_layer1.convolution1.weight",
                 "dpt.encoder.layer.3.attention.attention.key.bias", "neck.reassemble_stage.layers.1.resize.weight"):
        with pytest.raises(K2Error, match=r"missing keys \['" + gone.replace(".", r"\.") + r"'\]"):
            transformers_dpt_to_k2({k: v for k, v in sd.items() if k != gone}, cfg)


@pytest.mark.parametrize("key,value", [("is_hybrid", True), ("backbone_config", {"model_type": "bit"}),
                                       ("backbone", "vit"), ("readout_type", "add"), ("readout_type", "ignore"),
                                       ("hidden_act", "quick_gelu"), ("num_attention_heads", 4),
                                       ("use_batch_norm_in_fusion_residual", True), ("use_bias_in_fusion_residual", False),
                                       ("add_projection", True), ("head_in_index", 0), ("reassemble_factors", [4, 2, 1, 0.25]),
                                       ("reassemble_factors", [8, 2, 1, 0.5]), ("qkv_bias", False), ("num_channels", 1)])
def test_config_refusals_name_the_key(key, value):
    from kandinsky2._native import K2Error
    from kandinsky2.model.depth import dpt_config
    cfg, _ = _tiny("even")
    dpt_config(cfg)
    with pytest.raises(K2Error, match=key):
        dpt_config(dict(cfg, **{key: value}))


def test_geometry_comes_from_the_config():
    from kandinsky2.model.depth import dpt_config
    c = dpt_config(do.CFG_LARGE)
    assert (c["hidden_size"], c["num_hidden_layers"], c["num_attention_heads"], c["backbone_out_indices"]) == \
        (1024, 24, 16, [5, 11, 17, 23])
    d = dpt_config({})                                   # transformers' DPTConfig defaults
    assert (d["hidden_size"], d["neck_hidden_sizes"], d["layer_norm_eps"]) == (768, [96, 192, 384, 768], 1e-12)


def test_preprocess_refuses_non_square_outputs():
    from PIL import Image

    from kandinsky2._native import K2Error
    from kandinsky2.model.depth import preprocess_images, preprocessor_settings
    img = Image.new("RGB", (90, 60))
    keep = preprocessor_settings(dict(size=384, keep_aspect_ratio=True, ensure_multiple_of=32), 384)
    assert keep["size"] == {"height": 384, "width": 384}
    with pytest.raises(K2Error, match="only the square 384 x 384"):
        preprocess_images([img], keep, 384)
    with pytest.raises(K2Error, match="do_pad"):
        preprocessor_settings(dict(do_pad=True, size_divisor=32), 384)


def test_make_hint_restates_diffusers():
    from PIL import Image

    from kandinsky2.model.depth import make_hint
    a = np.random.default_rng(0).integers(0, 256, (30, 40), dtype=np.uint8)

    class Est:
        def depth(self, images):
            assert len(images) == 1
            return [Image.fromarray(a)]

    hint = make_hint(Image.new("RGB", (40, 30)), Est())
    assert hint.dtype == torch.float32 and hint.shape == (3, 30, 40)
    for c in range(3):
        assert torch.equal(hint[c], torch.from_numpy(a).float() / 255.0)


def test_against_transformers_live_second_seed():
    pytest.importorskip("transformers")
    from kandinsky2.model.depth import depth_image, preprocess_images, preprocessor_settings
    images = [img for _, img in do.sample_images(7)]
    for _, cfg, proc in do.TINY:
        sd = do.synth_weights(cfg, 12)
        model = do.transformers_model(cfg, sd)
        tp = do.transformers_processor(proc)
        pix = torch.cat([tp(img.convert("RGB"), return_tensors="pt")["pixel_values"] for img in images])
        ours = preprocess_images(images, preprocessor_settings(proc, cfg["image_size"]), proc["size"]["height"])
        assert (ours - pix).abs().max().item() <= 1e-6
        with torch.no_grad():
            ref = model(pixel_values=pix).predicted_depth
        assert ((do.forward(sd, cfg, pix) - ref).norm() / ref.norm()).item() <= 1e-5
        u8, pred = do.pipeline_depths(model, proc, images[:2])
        for img, p, a in zip(images, pred, u8):
            assert np.array_equal(np.array(depth_image(p, img.size[1], img.size[0])), a)
