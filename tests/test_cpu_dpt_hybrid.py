"""CPU: the hybrid DPT's host side (kandinsky2/model/depth.py, checkpoints.transformers_dpt_hybrid_to_k2) and the oracle.

  - the oracle (tests/dpt_hybrid_oracle.py) against the golden fixture, and against live transformers where it is installed;
  - the hybrid config parser: Intel/dpt-hybrid-midas's geometry and transformers' BiT defaults accepted, everything else
    refused with K2Error naming the key; dpt_config keeps refusing is_hybrid;
  - the remap: the transformers key set, and unknown / missing keys refused by name;
  - weight standardisation against transformers' batch_norm form;
  - the annotator pieces of midas_hint: HWC3, resize_image's sizes and cv2 call, / 127.5 - 1, the uint8 postprocess."""
import copy

import numpy as np
import pytest
import torch

from kandinsky2._native import K2Error
from kandinsky2.checkpoints import transformers_dpt_hybrid_keys, transformers_dpt_hybrid_to_k2
from kandinsky2.model import depth
from tests import dpt_hybrid_oracle as ho


@pytest.fixture(scope="module")
def fx():
    return torch.load(ho.FIXTURE)


def test_oracle_matches_golden(fx):
    sd = ho.synth_weights(fx["config"], fx["weight_seed"])
    for (h, w), g in fx["sizes"].items():
        got, maps = ho.forward(sd, fx["config"], ho.fixture_pixels(g), with_maps=True)
        ref = g["predicted_depth"]
        assert got.shape == ref.shape
        assert ((got - ref).norm() / ref.norm()).item() <= 1e-5, (h, w)
        for a, b in zip(maps, g["bit_channel_means"]):
            assert (a.mean((0, 2, 3)) - b).abs().max().item() <= 1e-5 * b.abs().max().item(), (h, w)
        for a, b in zip(maps, g.get("bit_maps", [])):   # stored rounded to fp16
            assert ((a - b.float()).norm() / b.float().norm()).item() <= 1e-3, (h, w)
    assert "bit_maps" in fx["sizes"][(64, 64)]


def test_oracle_matches_live_transformers(fx):
    pytest.importorskip("transformers")
    spec = ho.hybrid_spec(fx["config"])
    assert sorted(k for k, _ in spec) == sorted(transformers_dpt_hybrid_keys(fx["config"]))
    assert dict(spec) == dict(ho.spec_from_config(fx["config"]))
    sd = ho.synth_weights(fx["config"], fx["weight_seed"], spec)
    model = ho.transformers_model(fx["config"], sd)
    for (h, w), g in fx["sizes"].items():
        ref, _ = ho.transformers_compose(model, ho.fixture_pixels(g))
        assert torch.equal(ref, g["predicted_depth"]) or ((ref - g["predicted_depth"]).norm() / ref.norm()).item() <= 1e-6


def test_config_accepts_the_real_geometry_and_defaults():
    c = depth.dpt_hybrid_config(ho.CFG_HYBRID)
    assert c["bit"] == dict(stem=64, channels=[256, 512, 1024], mids=[64, 128, 256], depths=[3, 4, 9])
    assert c["kp"] == 1088 and c["backbone_out_indices"] == [2, 5, 8, 11]
    no_bc = {k: v for k, v in ho.CFG_HYBRID.items() if k != "backbone_config"}
    assert depth.dpt_hybrid_config(no_bc)["bit"] == c["bit"]
    with pytest.raises(K2Error, match="is_hybrid"):
        depth.dpt_config(ho.CFG_HYBRID)


@pytest.mark.parametrize("key,value", [("layer_type", "preactivation"), ("global_padding", "valid"), ("num_groups", 16),
                                       ("embedding_dynamic_padding", False), ("width_factor", 2), ("hidden_act", "gelu"),
                                       ("output_stride", 8), ("out_features", ["stage1", "stage2"]),
                                       ("depths", [3, 4])])
def test_config_refuses_other_backbones_naming_the_key(key, value):
    cfg = copy.deepcopy(ho.CFG_HYBRID)
    cfg["backbone_config"][key] = value
    with pytest.raises(K2Error, match=f"backbone_config.{key}"):
        depth.dpt_hybrid_config(cfg)


@pytest.mark.parametrize("key,value", [("readout_type", "ignore"), ("neck_hidden_sizes", [96, 192, 768, 768]),
                                       ("backbone_featmap_shape", [1, 2048, 24, 24]), ("neck_ignore_stages", [0]),
                                       ("hidden_act", "relu"), ("patch_size", 8)])
def test_config_refuses_other_necks_naming_the_key(key, value):
    cfg = dict(ho.CFG_HYBRID, **{key: value})
    with pytest.raises(K2Error, match=key):
        depth.dpt_hybrid_config(cfg)


def test_remap_refuses_unknown_and_missing_keys():
    cfg = ho.CFG_TINY
    sd = ho.synth_weights(cfg, 1)
    out = transformers_dpt_hybrid_to_k2(sd, cfg)
    assert set(out) == set(depth.k2_hybrid_shapes(depth.dpt_hybrid_config(cfg)))
    assert all(tuple(out[k].shape) == s for k, s in depth.k2_hybrid_shapes(depth.dpt_hybrid_config(cfg)).items())
    bad = dict(sd, **{"dpt.embeddings.backbone.bit.encoder.stages.0.layers.5.conv1.weight": torch.zeros(1)})
    with pytest.raises(K2Error, match=r"unknown keys \['dpt.embeddings.backbone.bit.encoder.stages.0.layers.5.conv1.weight'\]"):
        transformers_dpt_hybrid_to_k2(bad, cfg)
    miss = {k: v for k, v in sd.items() if k != "dpt.embeddings.backbone.bit.encoder.stages.1.layers.0.downsample.norm.bias"}
    with pytest.raises(K2Error, match="missing keys.*stages.1.layers.0.downsample.norm.bias"):
        transformers_dpt_hybrid_to_k2(miss, cfg)
    plain = dict(sd, **{"neck.reassemble_stage.readout_projects.0.0.weight": torch.zeros(1)})
    with pytest.raises(K2Error, match="readout_projects.0.0.weight"):
        transformers_dpt_hybrid_to_k2(plain, cfg)


def test_weight_standardisation_matches_transformers_form():
    g = torch.Generator().manual_seed(0)
    for shape in ((64, 3, 7, 7), (256, 64, 1, 1), (128, 128, 3, 3)):
        w = 0.05 * torch.randn(shape, generator=g) + 0.01
        ref = ho.standardized(w.double())
        got = depth.standardize_weight(w)
        assert got.dtype == torch.float64
        assert (got - ref).abs().max().item() < 1e-12
        assert torch.equal(got.half(), ref.half())


def test_hwc3():
    rng = np.random.default_rng(0)
    grey = rng.integers(0, 256, (5, 7), dtype=np.uint8)
    assert np.array_equal(depth.hwc3(grey), np.stack([grey] * 3, 2))
    rgb = rng.integers(0, 256, (5, 7, 3), dtype=np.uint8)
    assert depth.hwc3(rgb) is rgb
    rgba = rng.integers(0, 256, (5, 7, 4), dtype=np.uint8)
    color, alpha = rgba[:, :, :3].astype(np.float32), rgba[:, :, 3:].astype(np.float32) / 255.0
    want = (color * alpha + 255.0 * (1.0 - alpha)).clip(0, 255).astype(np.uint8)
    assert np.array_equal(depth.hwc3(rgba), want)
    with pytest.raises(K2Error, match="uint8"):
        depth.hwc3(rgb.astype(np.float32))


def test_resize_image_sizes_and_cv2_call():
    assert depth.resize_image_size(512, 512, 512)[:2] == (512, 512)
    assert depth.resize_image_size(480, 640, 640)[:2] == (640, 832)   # k = 4 / 3
    assert depth.resize_image_size(300, 200, 200)[:2] == (320, 192)
    same = np.arange(512 * 512 * 3, dtype=np.uint8).reshape(512, 512, 3)
    assert depth.resize_image(same, 512) is same
    cv2 = pytest.importorskip("cv2")
    for interp in (cv2.INTER_AREA, cv2.INTER_LANCZOS4):
        assert np.array_equal(cv2.resize(same, (512, 512), interpolation=interp), same)
    rng = np.random.default_rng(1)
    for h, w in ((300, 200), (700, 500)):
        x = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        H, W, k = depth.resize_image_size(h, w, w)
        want = cv2.resize(x, (W, H), interpolation=cv2.INTER_LANCZOS4 if k > 1 else cv2.INTER_AREA)
        assert np.array_equal(depth.resize_image(x, w), want)


def test_midas_pixels_and_u8_postprocess():
    rng = np.random.default_rng(2)
    img = rng.integers(0, 256, (32, 48, 3), dtype=np.uint8)
    px = depth.midas_pixels(img)
    assert px.shape == (1, 3, 32, 48) and px.dtype == torch.float32
    assert torch.equal(px[0].permute(1, 2, 0), torch.from_numpy(img).float() / 127.5 - 1.0)
    d = (rng.standard_normal((32, 48)) * 3 + 10).astype(np.float32)
    e = d - d.min()
    e = e / e.max()
    assert np.array_equal(depth.midas_depth_u8(d), (e * 255.0).clip(0, 255).astype(np.uint8))
    assert not depth.midas_depth_u8(np.full((4, 4), 2.5, np.float32)).any()
