"""CPU: the Kandinsky 2.2 MoVQ in diffusers' `VQModel` layout (kandinsky2.checkpoints.diffusers_movq_to_k2 /
k2_to_diffusers_movq, kandinsky2.diffusers_compat.movq_config).

  - both remaps are inverse bijections between the restated diffusers key set (tests/movq22_oracle.py) and the key set MOVQ
    registers (oracle/movq_oracle.movq_param_spec), at the tiny geometry on random weights and at the real one by shape;
  - through the network: the pinned oracle decode / encode (the reference's MOVQ) on the remapped weights equals the restated
    diffusers forward (decode with force_not_quantize, encode's latents) to 1e-5 relative in fp32;
  - the attention names older diffusers conversions wrote load to the same tensors; unknown and missing keys, and every config
    value MOVQ does not implement, are refused by name."""
import pytest
import torch

from oracle import movq_oracle as mo
from tests import movq22_oracle as m22


def _spec_shapes(spec):
    return {k: tuple(s) for k, s in spec}


def _random(cfg, seed):
    from oracle import synth
    return synth.synth_state_dict(m22.vqmodel_spec(cfg), seed=seed)


@pytest.mark.parametrize("which", ["tiny", "kandinsky22"])
def test_remaps_are_inverse_bijections_onto_the_movq_key_set(which):
    from kandinsky2.checkpoints import diffusers_movq_to_k2, k2_to_diffusers_movq
    from kandinsky2.diffusers_compat import movq_config
    cfg = m22.VQMODEL_TINY if which == "tiny" else m22.VQMODEL_22
    dd, n_embed, embed_dim = movq_config(cfg)
    if which == "tiny":
        dsd = _random(cfg, seed=3)
    else:   # the real geometry by shape alone
        dsd = {k: torch.empty(s, device="meta") for k, s in m22.vqmodel_spec(cfg)}
    k2 = diffusers_movq_to_k2(dsd, dd)
    want = _spec_shapes(mo.movq_param_spec(mo.DDCONFIG_TINY if which == "tiny" else mo.DDCONFIG_2_1, embed_dim, n_embed))
    assert {k: tuple(v.shape) for k, v in k2.items()} == want
    back = k2_to_diffusers_movq(k2, dd)
    assert {k: tuple(v.shape) for k, v in back.items()} == _spec_shapes(m22.vqmodel_spec(cfg))
    if which == "tiny":
        assert all(torch.equal(back[k], dsd[k]) for k in dsd)
        again = diffusers_movq_to_k2(back, dd)
        assert all(torch.equal(again[k], k2[k]) for k in k2)


def test_movq_config_of_the_released_layout_is_the_reference_config():
    from kandinsky2.configs import CONFIG_2_2
    from kandinsky2.diffusers_compat import movq_config
    p = CONFIG_2_2["image_enc_params"]["params"]
    assert movq_config(m22.VQMODEL_22) == (p["ddconfig"], p["n_embed"], p["embed_dim"])
    dd, n_embed, embed_dim = movq_config(m22.VQMODEL_TINY)
    assert (n_embed, embed_dim) == (64, 4)
    assert mo.encoder_topology(dd) == mo.encoder_topology(mo.DDCONFIG_TINY)
    assert mo.decoder_topology(dd) == mo.decoder_topology(mo.DDCONFIG_TINY)


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def test_oracle_forward_on_remapped_weights_equals_the_diffusers_form():
    from kandinsky2.checkpoints import diffusers_movq_to_k2
    from kandinsky2.diffusers_compat import movq_config
    cfg = m22.VQMODEL_TINY
    dd, _, _ = movq_config(cfg)
    dsd = _random(cfg, seed=11)
    k2 = diffusers_movq_to_k2(dsd, dd)
    g = torch.Generator().manual_seed(0)
    lat = torch.randn(2, 4, 8, 8, generator=g)
    img = torch.rand(2, 3, 32, 32, generator=g) * 2 - 1
    with torch.no_grad():
        dec, ref_dec = mo.movq_decode(k2, dd, lat), m22.vqmodel_decode(dsd, cfg, lat)
        enc, ref_enc = mo.movq_encode(k2, dd, img), m22.vqmodel_encode(dsd, cfg, img)
    assert dec.shape == (2, 3, 16, 16) and enc.shape == (2, 4, 16, 16)
    print(f"MoVQ oracle vs diffusers form: decode rel-L2 {_rel(dec, ref_dec):.2e}, encode rel-L2 {_rel(enc, ref_enc):.2e}")
    assert _rel(dec, ref_dec) <= 1e-5 and _rel(enc, ref_enc) <= 1e-5
    # and not trivially: the up-block order matters
    swapped = dict(dsd)
    for a, b in (("decoder.up_blocks.0.resnets.0.conv1.weight", "decoder.up_blocks.0.resnets.1.conv1.weight"),):
        swapped[a], swapped[b] = dsd[b], dsd[a]
    with torch.no_grad():
        assert _rel(mo.movq_decode(diffusers_movq_to_k2(swapped, dd), dd, lat), ref_dec) > 1e-3


def test_legacy_attention_names_load_to_the_same_tensors():
    from kandinsky2.checkpoints import diffusers_movq_to_k2
    from kandinsky2.diffusers_compat import movq_config
    from kandinsky2._native import K2Error
    cfg = m22.VQMODEL_TINY
    dd, _, _ = movq_config(cfg)
    dsd = _random(cfg, seed=5)
    old = {"to_q": "query", "to_k": "key", "to_v": "value", "to_out.0": "proj_attn"}
    legacy = {}
    for k, v in dsd.items():
        for new, name in old.items():
            if ".attentions." in k and f".{new}." in k:
                k = k.replace(f".{new}.", f".{name}.")
        legacy[k] = v
    assert any(".proj_attn." in k for k in legacy) and not any(".to_q." in k for k in legacy)
    a, b = diffusers_movq_to_k2(dsd, dd), diffusers_movq_to_k2(legacy, dd)
    assert a.keys() == b.keys() and all(torch.equal(a[k], b[k]) for k in a)
    both = dict(dsd, **{"encoder.mid_block.attentions.0.query.weight": dsd["encoder.mid_block.attentions.0.to_q.weight"]})
    with pytest.raises(K2Error, match="to_q.weight"):
        diffusers_movq_to_k2(both, dd)


def test_unknown_and_missing_keys_are_named():
    from kandinsky2.checkpoints import diffusers_movq_to_k2, k2_to_diffusers_movq
    from kandinsky2.diffusers_compat import movq_config
    from kandinsky2._native import K2Error
    dd, _, _ = movq_config(m22.VQMODEL_TINY)
    dsd = _random(m22.VQMODEL_TINY, seed=1)
    with pytest.raises(K2Error, match=r"unknown keys \['decoder.up_blocks.0.extra.weight'\]"):
        diffusers_movq_to_k2(dict(dsd, **{"decoder.up_blocks.0.extra.weight": torch.zeros(1)}), dd)
    gone = {k: v for k, v in dsd.items() if k != "decoder.conv_norm_out.conv_y.bias"}
    with pytest.raises(K2Error, match=r"missing keys \['decoder.conv_norm_out.conv_y.bias'\]"):
        diffusers_movq_to_k2(gone, dd)
    k2 = diffusers_movq_to_k2(dsd, dd)
    with pytest.raises(K2Error, match="decoder.up.1.attn.0.q.weight"):
        k2_to_diffusers_movq({k: v for k, v in k2.items() if k != "decoder.up.1.attn.0.q.weight"}, dd)


@pytest.mark.parametrize("key,value", [("norm_type", "group"), ("norm_num_groups", 16), ("act_fn", "gelu"),
                                       ("lookup_from_codebook", True), ("mid_block_add_attention", False),
                                       ("down_block_types", ["DownEncoderBlock2D", "SomeDownBlock2D"]),
                                       ("up_block_types", ["UpDecoderBlock2D", "AttnUpDecoderBlock2D"]),
                                       ("vq_embed_dim", 8), ("block_out_channels", [32, 48]), ("some_new_key", 1)])
def test_movq_config_refusals_name_the_key(key, value):
    from kandinsky2.diffusers_compat import movq_config
    from kandinsky2._native import K2Error
    with pytest.raises(K2Error, match=key):
        movq_config(dict(m22.VQMODEL_TINY, **{key: value}))
    if key == "norm_type":   # absent means diffusers' default, "group"
        with pytest.raises(K2Error, match="norm_type"):
            movq_config({k: v for k, v in m22.VQMODEL_TINY.items() if k != "norm_type"})
