"""LoRA oracle (TEST INFRASTRUCTURE): synthetic decoder-UNet adapters in diffusers' attention-processor format and their fp32
fold into a diffusers-layout state dict.

Parity unpinned: LoRA is not part of the reference package (its notebooks/lora_decoder.ipynb trains and loads one through
diffusers, which is not installed), so this restates diffusers' LoRALinearLayer (delta W = up @ down, no network_alpha) and the
key names `AttnProcsLayers` / `save_attn_procs` write for LoRAAttnAddedKVProcessor.  It lives next to the tests rather than in
oracle/, whose modules restate the reference itself.  fold_lora works in the DIFFUSERS layout (separate to_q / to_k / to_v /
add_k_proj / add_v_proj / to_out.0 Linears), before checkpoints.diffusers_unet_to_k2, so it shares nothing with the product's
packed-layout path (checkpoints.lora_to_k2 + k2_lora_merge).
"""
import torch

PROJECTIONS = ("to_q", "to_k", "to_v", "to_out", "add_k_proj", "add_v_proj")
_WEIGHT = {"to_q": "to_q", "to_k": "to_k", "to_v": "to_v", "to_out": "to_out.0", "add_k_proj": "add_k_proj",
           "add_v_proj": "add_v_proj"}


def attention_blocks(cfg):
    """[(diffusers attention prefix, channels)] of a UNet config of oracle/unet_oracle.py."""
    from kandinsky2.checkpoints import unet_block_map
    from oracle import unet_oracle as uo
    inp, mid, out = uo.unet_topology(dict(cfg, inpainting=False))
    chans = [layer[1] for blk in inp + [mid] + out for layer in blk if layer[0] == "attn"]
    prefixes = [dp for dp, _, kind in unet_block_map(cfg["in_channels"], cfg["model_channels"], tuple(cfg["channel_mult"]),
                                                     cfg["num_res_blocks"], tuple(cfg["attention_ds"])) if kind == "attn"]
    assert len(prefixes) == len(chans)
    return list(zip(prefixes, chans))


def synth_lora(cfg, rank, seed=0, gain=0.3, projections=PROJECTIONS, dtype=torch.float32):
    """A notebook-format adapter with BOTH factors random (diffusers initialises `up` to zero, which would test nothing):
    down ~ N(0, 1/fan_in), up ~ N(0, gain^2/rank), so each delta W is about `gain` times a fan-in-scaled weight."""
    g = torch.Generator().manual_seed(seed)
    out = {}
    for dp, C in attention_blocks(cfg):
        for proj in projections:
            fan_in = cfg["model_dim"] if proj.startswith("add_") else C
            out[f"{dp}.processor.{proj}_lora.down.weight"] = (torch.randn(rank, fan_in, generator=g) / fan_in ** 0.5).to(dtype)
            out[f"{dp}.processor.{proj}_lora.up.weight"] = (torch.randn(C, rank, generator=g) * (gain / rank ** 0.5)).to(dtype)
    return out


def fold_lora(sd_diffusers, lora, scale=1.0):
    """W + scale * up @ down in fp32 on the state dict's device, for every LoRA pair, in the diffusers layout."""
    out = dict(sd_diffusers)
    for key, down in lora.items():
        if not key.endswith("_lora.down.weight"):
            continue
        prefix, rest = key.split(".processor.")
        wk = f"{prefix}.{_WEIGHT[rest[:-len('_lora.down.weight')]]}.weight"
        w = sd_diffusers[wk]
        up = lora[key[:-len("down.weight")] + "up.weight"]
        out[wk] = w.float() + scale * (up.to(w.device).float() @ down.to(w.device).float())
    return out
