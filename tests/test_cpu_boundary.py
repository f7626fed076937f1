"""CPU: the drop-in boundary -- every symbol of include/k2b200.h is exported by libk2b200.so, the product modules
expose the reference's state_dict keys / constructor surface, and the product refuses to run without a GPU."""
import os
import re
import sys

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def test_abi_exports_every_declared_symbol():
    from kandinsky2 import _native
    hdr = open(os.path.join(ROOT, "include", "k2b200.h")).read()
    declared = set(re.findall(r"\b(k2_[a-z0-9_]+)\s*\(", hdr))
    lib = _native.load()
    assert not _native.MISSING, _native.MISSING
    for name in declared:
        assert hasattr(lib, name), f"{name} declared in k2b200.h but not exported"
    assert declared == set(_native.SIGNATURES), declared ^ set(_native.SIGNATURES)
    assert lib.k2_version() >= 100


def test_unet_state_dict_keys_match_reference_spec():
    from kandinsky2.configs import CONFIG_2_1
    from kandinsky2.model.model_creation import create_model
    from oracle import unet_oracle as uo
    cfg = dict(CONFIG_2_1["model_config"], num_channels=64, num_res_blocks=1)  # same topology rules, small
    m = create_model(**cfg, up=False, inpainting=False)
    ocfg = dict(uo.CONFIG_2_1, model_channels=64, num_res_blocks=1)
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == [(k, tuple(s)) for k, s in uo.unet_param_spec(ocfg)]
    mi = create_model(**cfg, up=False, inpainting=True)
    assert mi.state_dict()["input_blocks.0.0.weight"].shape[1] == 9
    assert m.dtype == torch.float16 and m.model_channels == 64
    with pytest.raises(NotImplementedError):
        create_model(**dict(cfg, use_scale_shift_norm=False), up=False, inpainting=False)


def test_movq_state_dict_keys_match_reference_spec():
    from kandinsky2.vqgan import MOVQ
    from oracle import movq_oracle as mo
    m = MOVQ(mo.DDCONFIG_TINY, 64, 4)
    assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == \
        [(k, tuple(s)) for k, s in mo.movq_param_spec(dict(mo.DDCONFIG_TINY, double_z=False), 4, 64)]
    # training checkpoints may carry loss.* entries: dropped
    sd = dict(m.state_dict())
    sd["loss.discriminator.main.0.weight"] = torch.zeros(1)
    m.load_state_dict(sd, strict=True)


def test_no_cpu_fallback():
    from kandinsky2._native import K2Error
    from kandinsky2.model.unet import Text2ImUNet
    from oracle import unet_oracle as uo
    if torch.cuda.is_available():
        pytest.skip("checks the CPU-only failure mode")
    cfg = uo.CONFIG_TINY
    m = Text2ImUNet(model_dim=cfg["model_dim"], image_encoder_in_dim=48, text_encoder_in_dim1=96, text_encoder_in_dim2=48,
                    num_image_embs=3, pooling_type="from_model", in_channels=4, model_channels=64, out_channels=8,
                    num_res_blocks=1, attention_resolutions=(2,), channel_mult=(1, 2), use_fp16=True,
                    num_head_channels=64, use_scale_shift_norm=True, resblock_updown=True)
    with pytest.raises(K2Error):
        m(torch.zeros(2, 4, 16, 16), torch.zeros(2), full_emb=torch.zeros(2, 7, 96), pooled_emb=torch.zeros(2, 48),
          image_emb=torch.zeros(2, 48))


def test_product_never_imports_oracle():
    pkg = os.path.join(ROOT, "kandinsky-2_b200", "kandinsky2")
    for dp, _, files in os.walk(pkg):
        for f in files:
            if f.endswith(".py"):
                src = open(os.path.join(dp, f)).read()
                assert not re.search(r"^\s*(from|import)\s+oracle\b", src, re.M), f"{f} imports the oracle"


def test_conv_plan_host_logic():
    """k2_conv_plan = the decisions k2_conv_gemm takes before touching a pointer (tile box, N tile, split-K, GroupNorm-partial
    layout); pure host arithmetic, so the shapes of the 768x768 step are pinned here without a GPU (132 SMs assumed when no
    device is present, as on an H100 SXM)."""
    from kandinsky2 import ops
    # level 0, 384 -> 384 3x3 at 96x96, UNet batch 8: (8 x 16)-pixel tiles, N tile 192 (divides 384), single CTA, no split,
    # one GroupNorm partial per M tile
    pl = ops.conv_plan(8, 96, 96, 9, 9 * 384, 384)
    assert pl == dict(n_tile=192, cta_pair=0, splits=1, m_tiles=576, images_per_tile=1, gn_partial_mode=1, row_groups=576)
    # level 1, 768 -> 768: 144 M tiles x 6 N tiles of 128 = 864 units fill 132 SMs better than 256-wide tiles
    pl = ops.conv_plan(8, 48, 48, 9, 9 * 768, 768)
    assert (pl["n_tile"], pl["splits"], pl["m_tiles"]) == (128, 1, 144)
    # level 2 (24 x 24): unsplit, N tile 192 (1152 = 6 x 192), 5-row tiles inside one image
    pl = ops.conv_plan(8, 24, 24, 9, 9 * 1152, 1152)
    assert (pl["n_tile"], pl["splits"], pl["m_tiles"], pl["images_per_tile"], pl["gn_partial_mode"]) == (192, 1, 40, 1, 1)
    # level 3 (12 x 12): (4 x 4 pixels x 8 images) tiles with every MMA row used, partials per (image, spatial tile)
    pl = ops.conv_plan(8, 12, 12, 9, 9 * 1536, 1536)
    assert (pl["m_tiles"], pl["images_per_tile"], pl["splits"], pl["gn_partial_mode"], pl["row_groups"]) == (9, 8, 1, 1, 72)
    # attention qkv as a flat-row GEMM, and the 4-channel fp32 NCHW output head (N tile 16)
    assert ops.conv_plan(1, 1, 18432, 1, 768, 2304, want_gn_partial=False)["n_tile"] == 256
    pl = ops.conv_plan(8, 96, 96, 9, 9 * 384, 8, out_mode=1, want_gn_partial=False)
    assert (pl["n_tile"], pl["cta_pair"], pl["gn_partial_mode"]) == (16, 0, 0)
    # a forced 2-way split moves the statistics to the second pass (16-row groups); without a workspace it cannot split
    ops.set_tuning(1, 2)
    try:
        pl = ops.conv_plan(8, 12, 12, 9, 9 * 1536, 1536)
        assert (pl["splits"], pl["gn_partial_mode"], pl["row_groups"]) == (2, 2, 8 * 144 // 16)
        assert ops.conv_plan(8, 12, 12, 9, 9 * 1536, 1536, workspace_bytes=0)["splits"] == 1
    finally:
        ops.set_tuning(1, 0)
    # ragged geometry: tiles never exceed 128 pixels and cover the image
    for (nb, h, w) in [(3, 16, 12), (1, 7, 5), (5, 12, 12), (2, 100, 36)]:
        pl = ops.conv_plan(nb, h, w, 9, 9 * 64, 64)
        assert pl["m_tiles"] * 128 >= nb * h * w


def test_diffusers_key_remap_roundtrip_and_head_interleave():
    """kandinsky2/checkpoints.py: the 2.2 (diffusers-layout) <-> package key maps are inverse bijections onto the exact key
    set of Text2ImUNet(cond_version="2.2"), and the head-interleaved qkv packing equals separate q / k / v projections
    under the reference's own split (`unet.py:296-307`)."""
    from kandinsky2 import checkpoints as ck
    from oracle import unet_oracle as uo
    cfg = uo.CONFIG_2_2
    spec = uo.unet_param_spec(cfg)
    g = torch.Generator().manual_seed(3)
    sd = {k: torch.randn(*s, generator=g) for k, s in spec}
    kw = dict(in_channels=cfg["in_channels"], model_channels=cfg["model_channels"], channel_mult=tuple(cfg["channel_mult"]),
              num_res_blocks=cfg["num_res_blocks"], attention_ds=tuple(cfg["attention_ds"]))
    dsd = ck.k2_to_diffusers_unet(sd, **kw)
    assert len(dsd) > len(sd)                      # qkv / encoder_kv split into 5 tensors each
    assert any(k.startswith("down_blocks.0.downsamplers.0.conv1") for k in dsd)
    assert "down_blocks.1.attentions.0.add_k_proj.weight" in dsd and "up_blocks.0.upsamplers.0.norm1.weight" in dsd
    back = ck.diffusers_unet_to_k2(dsd, **kw)
    assert sorted(back) == sorted(sd)
    assert all(torch.equal(back[k], sd[k]) for k in sd)
    # numerics of the interleave: Conv1d(qkv) + the reference's per-head split == three separate Linear projections
    C, heads, T = 128, 2, 5
    wq, wk, wv = (torch.randn(C, C, generator=g) for _ in range(3))
    x = torch.randn(3, C, T, generator=g)
    qkv = torch.nn.functional.conv1d(x, ck.pack_heads([wq, wk, wv]).unsqueeze(-1))          # [B, 3C, T]
    q, k, v = qkv.reshape(3 * heads, 3 * 64, T).split(64, dim=1)                             # unet.py:298-299
    for got, w in ((q, wq), (k, wk), (v, wv)):
        ref = torch.einsum("oc,bct->bot", w, x).reshape(3 * heads, 64, T)
        assert torch.allclose(got, ref, atol=1e-5)


def test_prior_state_dict_keys_match_reference_spec():
    """The prior groundwork module keeps the reference's parameter names and shapes (prior.py:191-228), i.e. the key set the
    oracle spec was checked against when tests/golden/prior_tiny.pt was written from the reference's own classes."""
    from kandinsky2.model.prior import PriorTransformer
    from oracle import prior_oracle as po
    for cfg in (po.CONFIG_PRIOR_TINY, dict(po.CONFIG_PRIOR, xf_layers=2)):
        m = PriorTransformer(**cfg)
        assert [(k, tuple(v.shape)) for k, v in m.state_dict().items()] == [(k, tuple(s)) for k, s in po.prior_param_spec(cfg)]
