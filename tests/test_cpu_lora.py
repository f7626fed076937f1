"""CPU: LoRA adapters of the decoder UNet in diffusers' attention-processor format -> (up', down') factors of the packed
weights (kandinsky2/checkpoints.py: lora_to_k2), their rejections, and the argument checks of k2_lora_merge."""
import ctypes

import pytest
import torch

from tests import lora_oracle as lo


def _mid_cfg():
    from oracle import unet_oracle as uo
    return dict(uo.CONFIG_2_2, model_channels=128, num_res_blocks=2, model_dim=256)


def _geom(cfg):
    return dict(in_channels=cfg["in_channels"], model_channels=cfg["model_channels"], channel_mult=tuple(cfg["channel_mult"]),
                num_res_blocks=cfg["num_res_blocks"], attention_ds=tuple(cfg["attention_ds"]))


def test_full_size_adapter_fully_consumed():
    """The notebook's adapter on the full 2.2 decoder: 22 attention blocks x 6 projections x (down, up) = 264 tensors, every
    block gets all three packed targets, and the targets cover the 168.7 M attention weight elements."""
    from kandinsky2.checkpoints import lora_to_k2
    from oracle import unet_oracle as uo
    lora = lo.synth_lora(uo.CONFIG_2_2, rank=4, dtype=torch.float16)
    assert len(lora) == 264
    packed = lora_to_k2(lora)   # the defaults are the full-size 2.2 decoder
    assert len(packed) == 66
    elems = 0
    for key, (up, down) in packed.items():
        assert up.dtype == down.dtype == torch.float32 and up.is_contiguous() and down.is_contiguous()
        C = down.shape[1] if key.endswith(("qkv.weight", "proj_out.weight")) else up.shape[0] // 2
        n, r = {"qkv": (3, 12), "encoder_kv": (2, 8), "proj_out": (1, 4)}[key.split(".")[-2]]
        assert up.shape == (n * C, r) and down.shape == (r, 768 if n == 2 else C)
        elems += up.shape[0] * down.shape[1]
    assert abs(elems - 168.7e6) < 0.05e6, elems


@pytest.mark.parametrize("dtype", [torch.float32, torch.float16, torch.bfloat16])
def test_packed_factors_equal_diffusers_layout_delta(dtype):
    """Per packed target, up' @ down' (float64) equals diffusers_unet_to_k2 applied to the diffusers-layout delta W = up @ down
    of every projection (zero for a missing one), to 1e-12 relative.  Some blocks carry only a subset of the projections."""
    from kandinsky2.checkpoints import diffusers_unet_to_k2, lora_to_k2
    cfg = _mid_cfg()
    lora = lo.synth_lora(cfg, rank=3, seed=5, dtype=dtype)
    dropped = {("mid_block.attentions.0", "to_k"), ("mid_block.attentions.0", "add_v_proj"),
               ("up_blocks.0.attentions.1", "to_out")}
    dropped |= {("down_blocks.1.attentions.0", p) for p in ("add_k_proj", "add_v_proj")}
    lora = {k: v for k, v in lora.items() if (k.split(".processor.")[0], k.split(".processor.")[1].split("_lora.")[0])
            not in dropped}
    packed = lora_to_k2(lora, model_dim=cfg["model_dim"], **_geom(cfg))
    dsd = {}
    for dp, C in lo.attention_blocks(cfg):
        dsd[f"{dp}.group_norm.weight"] = dsd[f"{dp}.group_norm.bias"] = torch.zeros(C, dtype=torch.float64)
        for proj in lo.PROJECTIONS:
            fan_in = cfg["model_dim"] if proj.startswith("add_") else C
            wk = f"{dp}.{lo._WEIGHT[proj]}"
            key = f"{dp}.processor.{proj}_lora."
            if key + "down.weight" in lora:
                dsd[wk + ".weight"] = lora[key + "up.weight"].double() @ lora[key + "down.weight"].double()
            else:
                dsd[wk + ".weight"] = torch.zeros(C, fan_in, dtype=torch.float64)
            dsd[wk + ".bias"] = torch.zeros(C, dtype=torch.float64)
    k2sd = diffusers_unet_to_k2(dsd, **_geom(cfg))
    n_targets = 0
    for key, w in k2sd.items():
        if not key.endswith(("qkv.weight", "encoder_kv.weight", "proj_out.weight")):
            continue
        want = w.squeeze(-1)
        if key not in packed:
            assert not want.any(), key
            continue
        n_targets += 1
        up, down = packed[key]
        got = up.double() @ down.double()
        assert got.shape == want.shape
        assert ((got - want).norm() / want.norm()).item() < 1e-12, key
    assert n_targets == 3 * len(lo.attention_blocks(cfg)) - 2   # mid encoder_kv keeps add_k; down_blocks.1.attentions.0 has none


def _rejects(lora, match):
    from kandinsky2._native import K2Error
    from kandinsky2.checkpoints import lora_to_k2
    cfg = _mid_cfg()
    with pytest.raises(K2Error, match=match):
        lora_to_k2(lora, model_dim=cfg["model_dim"], **_geom(cfg))


def test_rejections_name_the_offending_key():
    cfg = _mid_cfg()
    base = lo.synth_lora(cfg, rank=2, seed=1)
    mid = "mid_block.attentions.0.processor."
    C = 512  # mid block channels at 128 base channels x 4

    # unknown projection, unknown attention prefix (level 0 has no attention here), a stray key
    _rejects(dict(base, **{mid + "to_z_lora.down.weight": torch.zeros(2, C)}), "to_z_lora")
    _rejects(dict(base, **{"down_blocks.0.attentions.0.processor.to_q_lora.down.weight": torch.zeros(2, 128)}),
             r"down_blocks\.0\.attentions\.0")
    _rejects(dict(base, **{"mid_block.attentions.0.to_q.weight": torch.zeros(C, C)}), r"attentions\.0\.to_q\.weight")
    # a down without its up (and the reverse)
    d = dict(base)
    del d[mid + "to_k_lora.up.weight"]
    _rejects(d, r"to_k_lora\.down\.weight.*no matching up")
    d = dict(base)
    del d[mid + "add_v_proj_lora.down.weight"]
    _rejects(d, r"add_v_proj_lora\.up\.weight.*no matching down")
    # rank mismatch within a pair
    _rejects(dict(base, **{mid + "to_v_lora.up.weight": torch.zeros(C, 3)}), r"to_v_lora.*rank mismatch")
    # wrong in / out dimensions (in = C for to_*, model_dim for add_k / add_v)
    _rejects(dict(base, **{mid + "add_k_proj_lora.down.weight": torch.zeros(2, C)}), r"add_k_proj_lora.*down \[rank, 256\]")
    _rejects(dict(base, **{mid + "to_q_lora.down.weight": torch.zeros(2, 256)}), r"to_q_lora.*down \[rank, 512\]")
    _rejects(dict(base, **{mid + "to_out_lora.up.weight": torch.zeros(C + 64, 2)}), r"to_out_lora.*up \[512, rank\]")
    # PEFT keys and alpha entries
    _rejects(dict(base, **{"mid_block.attentions.0.to_q.lora_A.weight": torch.zeros(2, C)}), r"lora_A.*PEFT")
    _rejects(dict(base, **{mid + "to_q_lora.network_alpha": torch.tensor(4.0)}), r"to_q_lora\.network_alpha.*alpha")
    _rejects(dict(base, **{mid + "to_q_lora.alpha": torch.tensor(4.0)}), r"to_q_lora\.alpha.*alpha")
    # not a floating 2-D tensor
    _rejects(dict(base, **{mid + "to_q_lora.down.weight": torch.zeros(2, C, dtype=torch.int32)}), r"to_q_lora\.down")


def test_lora_merge_argument_errors_without_gpu():
    """k2_lora_merge checks its arguments before any CUDA call: < 0 and a message, also on a machine without a GPU."""
    from kandinsky2 import _native
    lib = _native.load()
    p = ctypes.c_void_p(256)   # never dereferenced: every call below fails its checks first
    cases = [((None, 8, p, p, 4, 8, 2, 1.0, p, 8), "null pointer"),
             ((p, 8, None, p, 4, 8, 2, 1.0, p, 8), "null pointer"),
             ((p, 8, p, p, 4, 8, 2, 1.0, None, 8), "null pointer"),
             ((p, 8, p, p, 0, 8, 2, 1.0, p, 8), "rank must be >= 1"),
             ((p, 8, p, p, 4, 0, 2, 1.0, p, 8), "rank must be >= 1"),
             ((p, 8, p, p, 4, 8, 0, 1.0, p, 8), "rank must be >= 1"),
             ((p, 7, p, p, 4, 8, 2, 1.0, p, 8), "strides must be >= cols"),
             ((p, 8, p, p, 4, 8, 2, 1.0, p, 5), "strides must be >= cols")]
    for args, msg in cases:
        assert lib.k2_lora_merge(*args, None) < 0, args
        assert msg in lib.k2_last_error().decode(), (args, lib.k2_last_error())


def _tiny_unet(**kw):
    from kandinsky2.model.unet import Text2ImUNet
    return Text2ImUNet(model_dim=128, image_encoder_in_dim=48, num_image_embs=3, pooling_type="from_model", in_channels=4,
                       model_channels=64, out_channels=8, num_res_blocks=1, attention_resolutions=(2,), channel_mult=(1, 2),
                       use_fp16=True, num_head_channels=64, use_scale_shift_norm=True, resblock_updown=True, cond_version="2.2",
                       **kw)


def test_load_lora_without_gpu_raises(tmp_path):
    """Like every op, merging needs the GPU: load_lora (and the diffusers-named load_attn_procs, from a file) raise K2Error on
    a CPU module and leave it without an adapter.  A malformed adapter is refused before that."""
    from kandinsky2._native import K2Error
    from kandinsky2.diffusers_compat import K2UNet2DConditionModel
    if torch.cuda.is_available():
        pytest.skip("checks the CPU-only failure mode")
    cfg = dict(in_channels=4, model_channels=64, channel_mult=(1, 2), num_res_blocks=1, attention_ds=(2,), model_dim=128)
    lora = lo.synth_lora(cfg, rank=2)
    m = _tiny_unet()
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}
    with pytest.raises(K2Error):
        m.load_lora(lora)
    assert m.lora_scale is None
    with pytest.raises(K2Error, match="to_x_lora"):
        m.load_lora(dict(lora, **{"mid_block.attentions.0.processor.to_x_lora.up.weight": torch.zeros(128, 2)}))
    path = tmp_path / "pytorch_model.bin"
    torch.save(lora, path)
    with pytest.raises(K2Error):
        K2UNet2DConditionModel(m).load_attn_procs(str(path))
    assert m.lora_scale is None
    assert all(torch.equal(v, sd0[k]) for k, v in m.state_dict().items())
