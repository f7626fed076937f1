"""Checkpoint / wire formats (SURVEY.md section 8f, rank 4) -- pure host code.

* Kandinsky 2.1 files (`decoder_fp16.ckpt`, `movq_final.ckpt`; `kandinsky2_1_model.py:82-91`) are plain state dicts with
  the key names this package's modules already use: `Text2ImUNet.load_state_dict` / `MOVQ.load_state_dict` take them as
  they are.
* Kandinsky 2.2 ships the decoder as a diffusers `UNet2DConditionModel` (`kandinsky2_2_model.py:26-28`,
  `kandinsky-community/kandinsky-2-2-decoder`, subfolder `unet`).  It is the same backbone (SURVEY.md section 8c) with a
  different parameter naming and separate q / k / v (and added k / v) Linear layers where the reference has one
  head-interleaved `qkv` (and `encoder_kv`) Conv1d.  `diffusers_unet_to_k2` renames and re-packs such a state dict into
  the key layout of `Text2ImUNet(cond_version="2.2")`; `k2_to_diffusers_unet` is its inverse.

* Kandinsky 2.2 ships its prior as a diffusers `PriorTransformer` (`kandinsky-community/kandinsky-2-2-prior`, subfolder
  `prior`): the 2.1 prior network with separate q / k / v.  `diffusers_prior_to_k2` renames and re-packs it into
  `model.prior.PriorTransformer` names and returns clip_mean / clip_std beside it (tests/test_cpu_prior22.py pins it through the
  network: the reference's forward on the remapped weights equals the diffusers-form forward).

* Kandinsky 2.2's prior pipeline carries a CLIP image tower, a transformers `CLIPVisionModelWithProjection`
  (`kandinsky2_2_model.py:24`, subfolder `image_encoder`).  `transformers_clip_vision_to_k2` renames it into
  `model.clip_vision.CLIPVisionTower` names and packs q / k / v per head (tests/test_cpu_clip_vision.py pins it through the
  network against the transformers-name forward and transformers' own outputs).  Its text tower, a transformers
  `CLIPTextModelWithProjection` (subfolder `text_encoder`), goes the same way through `transformers_clip_text_to_k2` into
  `model.clip_text.CLIPTextTower` names (tests/test_cpu_clip_text.py).

* Kandinsky 2.1's text encoder (`2_1/text_encoder/pytorch_model.bin`, the reference's `MultilingualCLIP`:
  XLM-RoBERTa-large and a Linear, `model/text_encoders.py:108-122`) goes through `mclip_to_k2` into
  `model.text_encoders.MultilingualCLIP` names (tests/test_cpu_text_encoder.py).

* Kandinsky 2.1's CLIP ViT-L/14 (`ViT-L-14.pt`, an OpenAI `clip` checkpoint) goes through `openai_clip_to_k2` into the
  text and image tower names above, with the geometry read from the shapes (tests/test_cpu_clip_vitl14.py).

* The depth estimator of the Kandinsky 2.2 ControlNet-depth hint, a transformers `DPTForDepthEstimation` with a plain ViT
  backbone (`Intel/dpt-large`), goes through `transformers_dpt_to_k2` into `model.depth.DPTDepthEstimator` names
  (tests/test_cpu_dpt.py).

* The transformer remaps above (diffusers prior, both transformers CLIP towers, M-CLIP, OpenAI CLIP, DPT) are tables over one
  recipe: `_stack_keys` lists a checkpoint's keys, `_require_keys` refuses unknown and missing ones, `_stack_to_k2` renames
  the top-level and per-layer names and packs q / k / v per head.  Each format's own cases (dropped keys, reshapes,
  transposes) stay at its call site.  `read_json` and `load_weights` read the component folders the towers load from.

* `lora_to_k2` maps a decoder LoRA in diffusers' attention-processor format onto low-rank factors of the packed
  qkv / encoder_kv / proj_out weights (merged on the GPU by `Text2ImUNet.load_lora`); `prior_lora_to_k2` does the same for
  an adapter of the 2.2 prior's self-attention, onto its c_qkv / c_proj (merged by `PriorTransformer.load_lora`).

* Kandinsky 2.2 ships its MoVQ as a diffusers `VQModel` with `norm_type="spatial"` (the decoder folders' `movq/`).  It is the
  reference's MOVQ under other names: `diffusers_movq_to_k2` renames it into `vqgan.autoencoder.MOVQ` names and turns the
  attention's Linear q / k / v / out into the 1x1 convolutions MOVQ registers; `k2_to_diffusers_movq` is its inverse
  (tests/test_cpu_movq22.py pins both through the network against a diffusers-form forward, tests/movq22_oracle.py).

**Parity unpinned:** diffusers is not part of /root/reference (`setup.py:27` lists it unpinned) and is not installed in the
build container, so the diffusers-side key names below are restated from the published `UNet2DConditionModel` layout
(`ResnetDownsampleBlock2D` / `SimpleCrossAttnDownBlock2D` / `UNetMidBlock2DSimpleCrossAttn` / `SimpleCrossAttnUpBlock2D` /
`ResnetUpsampleBlock2D`, attention with `added_kv_proj_dim`).  What IS tested (tests/test_cpu_boundary.py): the two maps
are inverse bijections onto the package's exact key set, and the head-interleaved packing reproduces separate
q / k / v projections numerically.
"""
import json
import math
import os
import re

import torch

from ._native import K2Error
from .model.unet import _topology

_RES = {"norm1": "in_layers.0", "conv1": "in_layers.2", "time_emb_proj": "emb_layers.1", "norm2": "out_layers.0",
        "conv2": "out_layers.3", "conv_shortcut": "skip_connection"}
_TOP = {"time_embedding.linear_1": "time_embed.0", "time_embedding.linear_2": "time_embed.2", "conv_in": "input_blocks.0.0",
        "conv_norm_out": "out.0", "conv_out": "out.2",
        "add_embedding.image_proj": "add_embedding.image_proj", "add_embedding.image_norm": "add_embedding.image_norm",
        "encoder_hid_proj.image_embeds": "encoder_hid_proj.image_embeds", "encoder_hid_proj.norm": "encoder_hid_proj.norm"}


def unet_block_map(in_channels, model_channels, channel_mult, num_res_blocks, attention_ds):
    """[(diffusers prefix, k2 prefix, kind)] for every ResBlock ('res') and attention block ('attn') of the UNet, in the
    reference's block order (`unet.py:421-557`): input_blocks.i.{0,1}, middle_block.{0,1,2}, output_blocks.i.{0,1,2}."""
    inp, mid, out = _topology(in_channels, model_channels, channel_mult, num_res_blocks, attention_ds)
    pairs = []
    level, j = 0, 0
    for i, blk in enumerate(inp[1:], start=1):
        if blk[0][0] == "res" and blk[0][3] == "down":
            pairs.append((f"down_blocks.{level}.downsamplers.0", f"input_blocks.{i}.0", "res"))
            level, j = level + 1, 0
            continue
        pairs.append((f"down_blocks.{level}.resnets.{j}", f"input_blocks.{i}.0", "res"))
        if len(blk) > 1:
            pairs.append((f"down_blocks.{level}.attentions.{j}", f"input_blocks.{i}.1", "attn"))
        j += 1
    pairs += [("mid_block.resnets.0", "middle_block.0", "res"), ("mid_block.attentions.0", "middle_block.1", "attn"),
              ("mid_block.resnets.1", "middle_block.2", "res")]
    level, j = 0, 0
    for i, blk in enumerate(out):
        pairs.append((f"up_blocks.{level}.resnets.{j}", f"output_blocks.{i}.0", "res"))
        pos = 1
        if len(blk) > 1 and blk[1][0] == "attn":
            pairs.append((f"up_blocks.{level}.attentions.{j}", f"output_blocks.{i}.1", "attn"))
            pos = 2
        j += 1
        if blk[-1][0] == "res" and blk[-1][3] == "up":
            pairs.append((f"up_blocks.{level}.upsamplers.0", f"output_blocks.{i}.{pos}", "res"))
            level, j = level + 1, 0
    return pairs


def pack_heads(parts, head_dim=64):
    """[W_a, W_b, ...] each [C, K] (rows = output channels, head-major) -> [len(parts)*C, K] with the reference's per-head
    interleave: head h owns rows [h*n*d, (h+1)*n*d) = [a_h | b_h | ...]  (`unet.py:296-299,304-307`: the Conv1d output is
    viewed as (heads, n*d, T) and split along dim 1)."""
    C = parts[0].shape[0]
    heads = C // head_dim
    stacked = torch.stack([p.reshape(heads, head_dim, *p.shape[1:]) for p in parts], dim=1)  # [heads, n, d, ...]
    return stacked.reshape(len(parts) * C, *parts[0].shape[1:])


def unpack_heads(w, n, head_dim=64):
    """Inverse of pack_heads: [n*C, ...] -> n tensors [C, ...]."""
    C = w.shape[0] // n
    heads = C // head_dim
    v = w.reshape(heads, n, head_dim, *w.shape[1:])
    return [v[:, i].reshape(C, *w.shape[1:]) for i in range(n)]


_WB = ("weight", "bias")


def _stack_keys(top, prefix, layer, qkv, layers):
    """The keys of a transformer checkpoint: `top` (the keys outside the layers), then for each of the `layers` layers,
    under prefix.format(i), the names of `layer` ({source name: this package's name}) and the q / k / v projections, each
    with its weight and bias.  qkv: the three projections' names up to the weight / bias suffix (e.g. "self_attn.q_proj."),
    or one name of a fused [q; k; v] projection (OpenAI's "attn.in_proj_")."""
    keys = list(top)
    for i in range(layers):
        lp = prefix.format(i)
        keys += [f"{lp}{d}.{s}" for d in layer for s in _WB] + [f"{lp}{n}{s}" for n in qkv for s in _WB]
    return keys


def _stack_to_k2(sd, top, prefix, layer, qkv, layers, dst, dst_qkv, head_dim):
    """A transformer checkpoint laid out as _stack_keys describes -> this package's names: top ({this package's name: source
    key}) copied, and layer i's `layer` names renamed under dst.format(i), its q / k / v packed per head_dim head into
    dst.format(i) + dst_qkv (pack_heads; a fused projection is split into thirds first)."""
    out = {k: sd[d] for k, d in top.items()}
    for i in range(layers):
        sp, dp = prefix.format(i), dst.format(i)
        for d, k in layer.items():
            for s in _WB:
                out[f"{dp}{k}.{s}"] = sd[f"{sp}{d}.{s}"]
        for s in _WB:
            parts = [sd[f"{sp}{n}{s}"] for n in qkv]
            out[f"{dp}{dst_qkv}.{s}"] = pack_heads(parts if len(parts) == 3 else list(parts[0].chunk(3)), head_dim)
    return out


def _count_layers(sd, prefix):
    """1 + the largest i with a key starting prefix.format(i), or 0."""
    rx = re.compile(re.escape(prefix).replace(r"\{\}", r"(\d+)"))
    return max((int(m.group(1)) + 1 for m in map(rx.match, sd) if m), default=0)


def _require_keys(sd, expected, what):
    """K2Error naming the keys of sd that are not expected and the expected keys sd lacks."""
    unknown = sorted(set(sd) - set(expected))
    missing = [k for k in expected if k not in sd]
    if unknown or missing:
        raise K2Error(f"{what} state dict: unknown keys {unknown}, missing keys {missing}")


def diffusers_unet_to_k2(sd, in_channels=4, model_channels=384, channel_mult=(1, 2, 3, 4), num_res_blocks=3,
                         attention_ds=(2, 4, 8), head_dim=64):
    """diffusers `UNet2DConditionModel` state dict (Kandinsky 2.2 decoder) -> `Text2ImUNet(cond_version="2.2")` keys.
    Linear q/k/v/out weights [C, C] become k=1 Conv1d weights [.., C, 1]; q|k|v and add_k|add_v are head-interleaved."""
    out = {k: v for k, v in sd.items() if k.startswith("add_embedding.input_hint_block.")}  # ControlNet hint stem: same names
    for d, k in _TOP.items():
        for suffix in ("weight", "bias"):
            if f"{d}.{suffix}" in sd:
                out[f"{k}.{suffix}"] = sd[f"{d}.{suffix}"]
    for dp, kp, kind in unet_block_map(in_channels, model_channels, channel_mult, num_res_blocks, attention_ds):
        if kind == "res":
            for dn, kn in _RES.items():
                for suffix in ("weight", "bias"):
                    key = f"{dp}.{dn}.{suffix}"
                    if key in sd:  # conv_shortcut only where the channel count changes
                        out[f"{kp}.{kn}.{suffix}"] = sd[key]
        else:
            out[f"{kp}.norm.weight"] = sd[f"{dp}.group_norm.weight"]
            out[f"{kp}.norm.bias"] = sd[f"{dp}.group_norm.bias"]
            q, k_, v = (sd[f"{dp}.to_{n}.weight"] for n in "qkv")
            out[f"{kp}.qkv.weight"] = pack_heads([q, k_, v], head_dim).unsqueeze(-1)
            out[f"{kp}.qkv.bias"] = pack_heads([sd[f"{dp}.to_{n}.bias"] for n in "qkv"], head_dim)
            ak, av = sd[f"{dp}.add_k_proj.weight"], sd[f"{dp}.add_v_proj.weight"]
            out[f"{kp}.encoder_kv.weight"] = pack_heads([ak, av], head_dim).unsqueeze(-1)
            out[f"{kp}.encoder_kv.bias"] = pack_heads([sd[f"{dp}.add_k_proj.bias"], sd[f"{dp}.add_v_proj.bias"]], head_dim)
            out[f"{kp}.proj_out.weight"] = sd[f"{dp}.to_out.0.weight"].unsqueeze(-1)
            out[f"{kp}.proj_out.bias"] = sd[f"{dp}.to_out.0.bias"]
    return out


_LORA_KEY = re.compile(r"^(.+)\.processor\.(to_q|to_k|to_v|to_out|add_k_proj|add_v_proj)_lora\.(down|up)\.weight$")
# packed target -> the projections that feed it, in pack_heads order
_LORA_TARGETS = {"qkv": ("to_q", "to_k", "to_v"), "encoder_kv": ("add_k_proj", "add_v_proj"), "proj_out": ("to_out",)}


def _read_lora(lora, rx, dims, what):
    """The factors of an adapter in diffusers' attention-processor form -> {(attention prefix, projection): {"down": fp32 [r, K],
    "up": fp32 [C, r]}} on the CPU.  rx matches a key into (attention prefix, projection, "down" | "up"); dims(prefix,
    projection) is (C, K), the projection's output rows and fan-in, or None for a prefix the model does not have.  Raises
    K2Error naming the first offending key for: PEFT (lora_A / lora_B) or alpha entries, unknown keys, non-floating or non-2-D
    tensors, a factor without its partner, rank or shape mismatches.  `what` names the model in the unknown-key message."""
    found = {}
    for key, t in lora.items():
        if "lora_A" in key or "lora_B" in key:
            raise K2Error(f"LoRA key {key!r}: PEFT-format (lora_A / lora_B) adapters are not supported")
        if "alpha" in key.rsplit(".", 1)[-1]:
            raise K2Error(f"LoRA key {key!r}: alpha / network_alpha scaling is not supported")
        m = rx.match(key)
        if m is None or dims(m.group(1), m.group(2)) is None:
            raise K2Error(f"LoRA key {key!r} is not an attention-processor LoRA weight of {what}")
        if not torch.is_tensor(t) or t.dtype not in (torch.float16, torch.bfloat16, torch.float32) or t.dim() != 2:
            raise K2Error(f"LoRA key {key!r}: expected a 2-D fp16, bf16 or fp32 tensor")
        found.setdefault((m.group(1), m.group(2)), {})[m.group(3)] = t.detach().to("cpu", torch.float32)
    for key in lora:
        dp, proj, which = rx.match(key).groups()
        pair = found[(dp, proj)]
        other = "up" if which == "down" else "down"
        if other not in pair:
            raise K2Error(f"LoRA key {key!r} has no matching {other} weight")
        down, up = pair["down"], pair["up"]
        C, fan_in = dims(dp, proj)
        if up.shape[1] != down.shape[0]:
            raise K2Error(f"LoRA key {key!r}: rank mismatch between down {tuple(down.shape)} and up {tuple(up.shape)}")
        if down.shape[1] != fan_in or up.shape[0] != C:
            raise K2Error(f"LoRA key {key!r}: expected down [rank, {fan_in}] and up [{C}, rank], got down "
                          f"{tuple(down.shape)} and up {tuple(up.shape)}")
    return found


def _lora_factors(pairs, projs, C, head_dim):
    """(up', down') of one packed weight whose rows are the projections `projs` (each C rows; head-interleaved by pack_heads
    when there are several), from pairs {projection: {"down", "up"}} of the present ones, or None when none is present.
    down' stacks the present projections' down matrices and up' is block-diagonal (zeros elsewhere), so up' @ down' packs the
    per-projection deltas up @ down -- the zero terms add exact zeros, so each element's fp32 sum equals that of its own
    projection.  A missing projection has no delta."""
    present = [p for p in projs if p in pairs]
    if not present:
        return None
    downs = [pairs[p]["down"] for p in present]
    R = sum(d.shape[0] for d in downs)
    ups, col = [], 0
    for p in projs:
        u = torch.zeros(C, R)
        if p in pairs:
            r = pairs[p]["down"].shape[0]
            u[:, col:col + r] = pairs[p]["up"]
            col += r
        ups.append(u)
    up = pack_heads(ups, head_dim) if len(projs) > 1 else ups[0]
    return up.contiguous(), torch.cat(downs, 0).contiguous()


def lora_to_k2(lora, in_channels=4, model_channels=384, channel_mult=(1, 2, 3, 4), num_res_blocks=3, attention_ds=(2, 4, 8),
               model_dim=768, head_dim=64):
    """A LoRA adapter of the decoder UNet in diffusers' attention-processor form -- the keys `AttnProcsLayers` /
    `UNet2DConditionModel.save_attn_procs` write for `LoRAAttnAddedKVProcessor`:
        {attention prefix}.processor.{to_q,to_k,to_v,to_out,add_k_proj,add_v_proj}_lora.{down,up}.weight
    with the attention prefixes of unet_block_map (e.g. `mid_block.attentions.0`) -> {packed weight key: (up', down')}, fp32,
    keyed like the output of diffusers_unet_to_k2 (`middle_block.1.qkv.weight`, `.encoder_kv.weight`, `.proj_out.weight`).

    The delta of a projection is up @ down (diffusers' LoRALinearLayer without network_alpha), so
    up' @ down' = diffusers_unet_to_k2 of the per-projection deltas (_lora_factors).  A missing projection has no delta.
    Raises K2Error naming the first offending key for anything else: unknown keys, PEFT (lora_A / lora_B) or alpha entries,
    a factor without its partner, rank or shape mismatches, non-floating tensors."""
    inp, mid, out = _topology(in_channels, model_channels, channel_mult, num_res_blocks, attention_ds)
    chans = [layer[1] for blk in inp + [mid] + out for layer in blk if layer[0] == "attn"]
    prefixes = [(dp, kp) for dp, kp, kind in unet_block_map(in_channels, model_channels, channel_mult, num_res_blocks,
                                                             attention_ds) if kind == "attn"]
    blocks = {dp: (kp, c) for (dp, kp), c in zip(prefixes, chans)}  # both lists are in the reference's block order

    def dims(dp, proj):
        if dp not in blocks:
            return None
        C = blocks[dp][1]
        return C, model_dim if proj.startswith("add_") else C

    found = _read_lora(lora, _LORA_KEY, dims, "this UNet")
    packed = {}
    for dp, (kp, C) in blocks.items():
        for target, projs in _LORA_TARGETS.items():
            f = _lora_factors({p: found[(dp, p)] for p in projs if (dp, p) in found}, projs, C, head_dim)
            if f is not None:
                packed[f"{kp}.{target}.weight"] = f
    return packed


_PRIOR_LORA_KEY = re.compile(r"^(transformer_blocks\.\d+\.attn1)\.processor\.(to_q|to_k|to_v|to_out)_lora\.(down|up)\.weight$")
# packed prior weight -> the projections that feed it, in pack_heads order
_PRIOR_LORA_TARGETS = {"attn.c_qkv": ("to_q", "to_k", "to_v"), "attn.c_proj": ("to_out",)}


def prior_lora_to_k2(lora, width, layers, head_dim=64):
    """A LoRA adapter of the Kandinsky 2.2 diffusion prior in diffusers' attention-processor form -- the keys `AttnProcsLayers`
    writes for `LoRAAttnProcessor` on the prior's self-attention:
        transformer_blocks.{i}.attn1.processor.{to_q,to_k,to_v,to_out}_lora.{down,up}.weight,  down [r, width], up [width, r]
    -> {packed weight key: (up', down')}, fp32, keyed like the output of diffusers_prior_to_k2
    (`transformer.resblocks.{i}.attn.c_qkv.weight`, `.attn.c_proj.weight`).  to_q / to_k / to_v become one pair with rows
    head-interleaved like c_qkv (_lora_factors), to_out the pair of c_proj.  Any subset of the projections may be present; a
    missing one has no delta.  The rank is read from the tensors.  Raises K2Error naming the first offending key as
    lora_to_k2 does, layer indices outside [0, layers) included."""
    blocks = {f"transformer_blocks.{i}.attn1": i for i in range(layers)}
    found = _read_lora(lora, _PRIOR_LORA_KEY, lambda dp, proj: (width, width) if dp in blocks else None, "this prior")
    packed = {}
    for dp, i in blocks.items():
        for target, projs in _PRIOR_LORA_TARGETS.items():
            f = _lora_factors({p: found[(dp, p)] for p in projs if (dp, p) in found}, projs, width, head_dim)
            if f is not None:
                packed[f"transformer.resblocks.{i}.{target}.weight"] = f
    return packed


_PRIOR_TOP = {"time_embedding.linear_1": "time_embed.0", "time_embedding.linear_2": "time_embed.2", "proj_in": "clip_img_proj",
              "embedding_proj": "text_emb_proj", "encoder_hidden_states_proj": "text_enc_proj", "norm_out": "final_ln",
              "proj_to_clip_embeddings": "out_proj"}
_PRIOR_BLOCK = {"norm1": "ln_1", "norm3": "ln_2", "attn1.to_out.0": "attn.c_proj", "ff.net.0.proj": "mlp.c_fc",
                "ff.net.2": "mlp.c_proj"}
_PRIOR_QKV = ("attn1.to_q.", "attn1.to_k.", "attn1.to_v.")


def diffusers_prior_keys(layers):
    """Every key of a diffusers Kandinsky 2.2 `PriorTransformer` state dict with `layers` transformer blocks."""
    top = ["positional_embedding", "prd_embedding", "clip_mean", "clip_std", *(f"{d}.{s}" for d in _PRIOR_TOP for s in _WB)]
    return _stack_keys(top, "transformer_blocks.{}.", _PRIOR_BLOCK, _PRIOR_QKV, layers)


def diffusers_prior_to_k2(sd, head_dim=64):
    """diffusers `PriorTransformer` state dict (Kandinsky 2.2, `kandinsky-community/kandinsky-2-2-prior`, subfolder `prior`) ->
    (state dict in `kandinsky2.model.prior.PriorTransformer` names, clip_mean [clip_dim], clip_std [clip_dim]).

    The network is the 2.1 prior's (token order, causal attention, exact GELU, final LayerNorm); only the names differ, and
    attn1.to_q / to_k / to_v become one c_qkv whose rows are interleaved per head [q_h | k_h | v_h] (pack_heads).  The
    `causal_attention_mask` buffer is dropped: the attention kernel builds the causal mask itself.  Raises K2Error naming
    the unknown and the missing keys.  Restated from diffusers' published layout (diffusers is not a dependency)."""
    sd = {k: v for k, v in sd.items() if k != "causal_attention_mask"}
    layers = _count_layers(sd, "transformer_blocks.{}.")
    _require_keys(sd, diffusers_prior_keys(layers), "diffusers prior")
    top = {"positional_embedding": "positional_embedding", "prd_emb": "prd_embedding",
           **{f"{k}.{s}": f"{d}.{s}" for d, k in _PRIOR_TOP.items() for s in _WB}}
    out = _stack_to_k2(sd, top, "transformer_blocks.{}.", _PRIOR_BLOCK, _PRIOR_QKV, layers, "transformer.resblocks.{}.",
                       "attn.c_qkv", head_dim)
    return out, sd["clip_mean"].reshape(-1), sd["clip_std"].reshape(-1)


def k2_to_diffusers_unet(sd,in_channels=4, model_channels=384, channel_mult=(1, 2, 3, 4), num_res_blocks=3,
                         attention_ds=(2, 4, 8), head_dim=64):
    """Inverse of diffusers_unet_to_k2 (export, and the round-trip test)."""
    out = {k: v for k, v in sd.items() if k.startswith("add_embedding.input_hint_block.")}
    for d, k in _TOP.items():
        for suffix in ("weight", "bias"):
            if f"{k}.{suffix}" in sd:
                out[f"{d}.{suffix}"] = sd[f"{k}.{suffix}"]
    for dp, kp, kind in unet_block_map(in_channels, model_channels, channel_mult, num_res_blocks, attention_ds):
        if kind == "res":
            for dn, kn in _RES.items():
                for suffix in ("weight", "bias"):
                    key = f"{kp}.{kn}.{suffix}"
                    if key in sd:
                        out[f"{dp}.{dn}.{suffix}"] = sd[key]
        else:
            out[f"{dp}.group_norm.weight"] = sd[f"{kp}.norm.weight"]
            out[f"{dp}.group_norm.bias"] = sd[f"{kp}.norm.bias"]
            for n, w, b in zip("qkv", unpack_heads(sd[f"{kp}.qkv.weight"].squeeze(-1), 3, head_dim),
                               unpack_heads(sd[f"{kp}.qkv.bias"], 3, head_dim)):
                out[f"{dp}.to_{n}.weight"], out[f"{dp}.to_{n}.bias"] = w, b
            for n, w, b in zip(("add_k_proj", "add_v_proj"), unpack_heads(sd[f"{kp}.encoder_kv.weight"].squeeze(-1), 2, head_dim),
                               unpack_heads(sd[f"{kp}.encoder_kv.bias"], 2, head_dim)):
                out[f"{dp}.{n}.weight"], out[f"{dp}.{n}.bias"] = w, b
            out[f"{dp}.to_out.0.weight"] = sd[f"{kp}.proj_out.weight"].squeeze(-1)
            out[f"{dp}.to_out.0.bias"] = sd[f"{kp}.proj_out.bias"]
    return out


_CLIP_LAYER = {"layer_norm1": "ln_1", "layer_norm2": "ln_2", "self_attn.out_proj": "attn.proj", "mlp.fc1": "mlp.fc1",
               "mlp.fc2": "mlp.fc2"}
_CLIP_QKV = ("self_attn.q_proj.", "self_attn.k_proj.", "self_attn.v_proj.")
# the keys outside the encoder layers: this package's name -> transformers' name
_CLIP_TOP = {
    "vision": {"class_embedding": "vision_model.embeddings.class_embedding",
               "patch_embedding.weight": "vision_model.embeddings.patch_embedding.weight",
               "position_embedding": "vision_model.embeddings.position_embedding.weight",
               "pre_ln.weight": "vision_model.pre_layrnorm.weight", "pre_ln.bias": "vision_model.pre_layrnorm.bias",
               "post_ln.weight": "vision_model.post_layernorm.weight", "post_ln.bias": "vision_model.post_layernorm.bias",
               "proj.weight": "visual_projection.weight"},
    "text": {"token_embedding": "text_model.embeddings.token_embedding.weight",
             "position_embedding": "text_model.embeddings.position_embedding.weight",
             "final_ln.weight": "text_model.final_layer_norm.weight", "final_ln.bias": "text_model.final_layer_norm.bias",
             "proj.weight": "text_projection.weight"},
}


def _clip_keys(tower, layers):
    return _stack_keys(_CLIP_TOP[tower].values(), f"{tower}_model.encoder.layers.{{}}.", _CLIP_LAYER, _CLIP_QKV, layers)


def _clip_to_k2(sd, tower, head_dim):
    """transformers CLIP `tower` ("text" / "vision") state dict -> this package's names, q / k / v packed per head_dim head."""
    p = f"{tower}_model."
    sd = {k: v for k, v in sd.items() if k != p + "embeddings.position_ids"}
    layers = _count_layers(sd, p + "encoder.layers.{}.")
    _require_keys(sd, _clip_keys(tower, layers), f"transformers CLIP {tower}")
    return _stack_to_k2(sd, _CLIP_TOP[tower], p + "encoder.layers.{}.", _CLIP_LAYER, _CLIP_QKV, layers, "layers.{}.",
                        "attn.qkv", head_dim)


def transformers_clip_vision_keys(layers):
    """Every key of a transformers `CLIPVisionModelWithProjection` state dict with `layers` encoder layers (without the
    non-persistent `position_ids` buffer)."""
    return _clip_keys("vision", layers)


def transformers_clip_vision_to_k2(sd, head_dim=104):
    """transformers `CLIPVisionModelWithProjection` state dict (the Kandinsky 2.2 prior's `image_encoder`) ->
    `model.clip_vision.CLIPVisionTower` names:
        class_embedding [H], patch_embedding.weight [H, 3, P, P], position_embedding [T, H], pre_ln.*, post_ln.*, proj.weight,
        layers.{i}.{ln_1, ln_2, attn.qkv, attn.proj, mlp.fc1, mlp.fc2}.{weight, bias}
    where attn.qkv stacks self_attn.{q,k,v}_proj per head [q_h | k_h | v_h] (pack_heads with the tower's head width).  A
    `position_ids` buffer is ignored; unknown and missing keys raise K2Error naming them."""
    return _clip_to_k2(sd, "vision", head_dim)


def transformers_clip_text_keys(layers):
    """Every key of a transformers `CLIPTextModelWithProjection` state dict with `layers` encoder layers (without the
    `position_ids` buffer)."""
    return _clip_keys("text", layers)


def transformers_clip_text_to_k2(sd):
    """transformers `CLIPTextModelWithProjection` state dict (the Kandinsky 2.2 prior's `text_encoder`) ->
    `model.clip_text.CLIPTextTower` names:
        token_embedding [V, H], position_embedding [T, H], final_ln.*, proj.weight,
        layers.{i}.{ln_1, ln_2, attn.qkv, attn.proj, mlp.fc1, mlp.fc2}.{weight, bias}
    where attn.qkv stacks self_attn.{q,k,v}_proj per head [q_h | k_h | v_h] (pack_heads, head width 64).  A `position_ids`
    buffer (older checkpoints carry it) is ignored; unknown and missing keys raise K2Error naming them."""
    return _clip_to_k2(sd, "text", 64)


# DPTForDepthEstimation: the ViT layer's names -> model/encoder.py's
_DPT_LAYER = {"layernorm_before": "ln_1", "layernorm_after": "ln_2", "attention.output.dense": "attn.proj",
              "intermediate.dense": "mlp.fc1", "output.dense": "mlp.fc2"}
_DPT_TOP = {"cls_token": "dpt.embeddings.cls_token", "position_embedding": "dpt.embeddings.position_embeddings",
            "patch_embedding.weight": "dpt.embeddings.patch_embeddings.projection.weight",
            "patch_embedding.bias": "dpt.embeddings.patch_embeddings.projection.bias"}
_DPT_QKV = ("attention.attention.query.", "attention.attention.key.", "attention.attention.value.")


def transformers_dpt_keys(config):
    """Every key of a transformers `DPTForDepthEstimation` state dict (plain ViT) for a config.json dict, including the
    ones transformers_dpt_to_k2 drops."""
    from .model.depth import dpt_config, k2_shapes
    c = dpt_config(config)
    keys = _stack_keys([*_DPT_TOP.values(), "dpt.layernorm.weight", "dpt.layernorm.bias"], "dpt.encoder.layer.{}.", _DPT_LAYER,
                       _DPT_QKV, c["num_hidden_layers"])
    keys += [k for k in k2_shapes(c) if k.startswith(("neck.", "head."))]
    return keys + [f"neck.fusion_stage.layers.0.residual_layer1.{conv}.{s}" for conv in ("convolution1", "convolution2")
                   for s in _WB]


def transformers_dpt_to_k2(sd, config):
    """transformers `DPTForDepthEstimation` state dict (plain ViT backbone, e.g. Intel/dpt-large) and its config.json dict ->
    `model.depth.DPTDepthEstimator` names:
        cls_token [H], position_embedding [T, H], patch_embedding.{weight, bias},
        layers.{i}.{ln_1, ln_2, attn.qkv, attn.proj, mlp.fc1, mlp.fc2}.{weight, bias},
        neck.* and head.* as transformers names them
    where attn.qkv stacks attention.attention.{query,key,value} per 64-wide head [q_h | k_h | v_h] (pack_heads).  Dropped on
    purpose, because transformers never runs them: dpt.layernorm.* (the neck reads the raw per-layer hidden states) and
    neck.fusion_stage.layers.0.residual_layer1.* (the first fusion layer gets no residual).  Unknown and missing keys raise
    K2Error naming them."""
    from .model.depth import dpt_config
    _require_keys(sd, transformers_dpt_keys(config), "transformers DPT")
    out = _stack_to_k2(sd, _DPT_TOP, "dpt.encoder.layer.{}.", _DPT_LAYER, _DPT_QKV, dpt_config(config)["num_hidden_layers"],
                       "layers.{}.", "attn.qkv", 64)
    out["cls_token"] = out["cls_token"].reshape(-1)                    # [1, 1, H] -> [H]
    out["position_embedding"] = out["position_embedding"][0]           # [1, T, H] -> [T, H]
    out.update({k: v for k, v in sd.items() if k.startswith(("neck.", "head."))
                and not k.startswith("neck.fusion_stage.layers.0.residual_layer1.")})
    return out


# the M-CLIP text encoder (Kandinsky 2.1's text_encoder/pytorch_model.bin): this package's name -> the checkpoint's name
_MCLIP_TOP = {"word_embedding": "transformer.embeddings.word_embeddings.weight",
              "position_embedding": "transformer.embeddings.position_embeddings.weight",
              "token_type_embedding": "transformer.embeddings.token_type_embeddings.weight",
              "emb_ln.weight": "transformer.embeddings.LayerNorm.weight", "emb_ln.bias": "transformer.embeddings.LayerNorm.bias",
              "proj.weight": "LinearTransformation.weight", "proj.bias": "LinearTransformation.bias"}
_MCLIP_LAYER = {"attention.output.dense": "attn.proj", "attention.output.LayerNorm": "ln_1", "intermediate.dense": "mlp.fc1",
                "output.dense": "mlp.fc2", "output.LayerNorm": "ln_2"}
_MCLIP_QKV = ("attention.self.query.", "attention.self.key.", "attention.self.value.")


def mclip_keys(layers):
    """Every key of the reference's MultilingualCLIP state dict with `layers` XLM-R layers, without the ones mclip_to_k2
    ignores (transformer.pooler.*, transformer.embeddings.position_ids)."""
    return _stack_keys(_MCLIP_TOP.values(), "transformer.encoder.layer.{}.", _MCLIP_LAYER, _MCLIP_QKV, layers)


def mclip_to_k2(sd, layers, head_dim=64):
    """The reference's MultilingualCLIP state dict (text_encoders.py:108-122: `transformer` an XLMRobertaModel,
    `LinearTransformation` the 1024 -> 768 Linear) -> `model.text_encoders.MultilingualCLIP` names:
        word_embedding [V, H], position_embedding [P, H], token_type_embedding [types, H], emb_ln.*, proj.{weight, bias},
        layers.{i}.{ln_1, ln_2, attn.qkv, attn.proj, mlp.fc1, mlp.fc2}.{weight, bias}
    with ln_1 = attention.output.LayerNorm, ln_2 = output.LayerNorm and attn.qkv stacking attention.self.{query,key,value}
    per head [q_h | k_h | v_h] (pack_heads).  transformer.pooler.* (unused by the reference's forward) and the
    embeddings.position_ids buffer are ignored.  Any other unknown key, and any missing one, raises K2Error naming it: the
    reference loads with strict=False, which would silently keep random weights there."""
    sd = {k: v for k, v in sd.items()
          if not k.startswith("transformer.pooler.") and k != "transformer.embeddings.position_ids"}
    _require_keys(sd, mclip_keys(layers), "M-CLIP text encoder")
    return _stack_to_k2(sd, _MCLIP_TOP, "transformer.encoder.layer.{}.", _MCLIP_LAYER, _MCLIP_QKV, layers, "layers.{}.",
                        "attn.qkv", head_dim)


# the OpenAI `clip` checkpoint (Kandinsky 2.1's ViT-L-14.pt; clip/model.py build_model reads it): one resblock's names
_OPENAI_LAYER = {"ln_1": "ln_1", "ln_2": "ln_2", "attn.out_proj": "attn.proj", "mlp.c_fc": "mlp.fc1", "mlp.c_proj": "mlp.fc2"}
_OPENAI_QKV = ("attn.in_proj_",)
# the keys outside the resblocks: this package's name -> the checkpoint's name, per tower
_OPENAI_TEXT_TOP = {"token_embedding": "token_embedding.weight", "position_embedding": "positional_embedding",
                    "final_ln.weight": "ln_final.weight", "final_ln.bias": "ln_final.bias", "proj.weight": "text_projection"}
_OPENAI_VISION_TOP = {"class_embedding": "visual.class_embedding", "position_embedding": "visual.positional_embedding",
                      "patch_embedding.weight": "visual.conv1.weight", "pre_ln.weight": "visual.ln_pre.weight",
                      "pre_ln.bias": "visual.ln_pre.bias", "post_ln.weight": "visual.ln_post.weight",
                      "post_ln.bias": "visual.ln_post.bias", "proj.weight": "visual.proj"}
# the entries build_model deletes before loading, and the contrastive temperature neither tower uses
_OPENAI_IGNORED = ("input_resolution", "context_length", "vocab_size", "logit_scale")


def openai_clip_keys(text_layers, vision_layers):
    """Every key of an OpenAI CLIP (ViT) state dict with the given resblock counts, without the ones openai_clip_to_k2
    ignores."""
    keys = _stack_keys([*_OPENAI_TEXT_TOP.values(), *_OPENAI_VISION_TOP.values()], "transformer.resblocks.{}.", _OPENAI_LAYER,
                       _OPENAI_QKV, text_layers)
    return keys + _stack_keys((), "visual.transformer.resblocks.{}.", _OPENAI_LAYER, _OPENAI_QKV, vision_layers)


def openai_clip_geometry(sd):
    """The geometry of an OpenAI CLIP (ViT) state dict, read from the tensor shapes as clip/model.py build_model does (there
    is no config): {"text": dict(width, layers, heads, mlp, context, vocab, embed_dim), "vision": dict(width, layers, heads,
    mlp, patch, grid, tokens, image_size, embed_dim)}; heads are of width 64.  K2Error names a key the geometry needs and
    the dict lacks."""
    need = ("ln_final.weight", "visual.conv1.weight", "positional_embedding", "visual.positional_embedding",
            "token_embedding.weight", "text_projection", "visual.proj")
    missing = [k for k in need if k not in sd]
    if missing:
        raise K2Error(f"OpenAI CLIP state dict: missing keys {missing}")

    def layers(prefix):
        return sum(1 for k in sd if re.fullmatch(rf"{re.escape(prefix)}resblocks\.\d+\.attn\.in_proj_weight", k))

    tw, vw = sd["ln_final.weight"].shape[0], sd["visual.conv1.weight"].shape[0]
    P, T = sd["visual.conv1.weight"].shape[-1], sd["visual.positional_embedding"].shape[0]
    G = math.isqrt(T - 1)
    for name, w in (("text", tw), ("vision", vw)):
        if w % 64:
            raise K2Error(f"OpenAI CLIP {name} tower: width {w} is not a multiple of the head width 64")
    if G * G != T - 1:
        raise K2Error(f"OpenAI CLIP vision tower: {T} positions are not a square grid plus the class token")
    text = dict(width=tw, layers=layers("transformer."), heads=tw // 64, mlp=4 * tw,
                context=sd["positional_embedding"].shape[0], vocab=sd["token_embedding.weight"].shape[0],
                embed_dim=sd["text_projection"].shape[1])
    vision = dict(width=vw, layers=layers("visual.transformer."), heads=vw // 64, mlp=4 * vw, patch=P, grid=G, tokens=T,
                  image_size=P * G, embed_dim=sd["visual.proj"].shape[1])
    return {"text": text, "vision": vision}


def openai_clip_to_k2(sd):
    """OpenAI CLIP (ViT) state dict (`clip.load(..., jit=False)` builds its model from it; Kandinsky 2.1's ViT-L-14.pt) ->
    (text, vision, geometry): the two towers' state dicts in this package's names (those of model/clip_text.py and
    model/clip_vision.py) and openai_clip_geometry(sd).
        text:    token_embedding, position_embedding, final_ln.*, proj.weight, layers.{i}.*
        vision:  class_embedding, patch_embedding.weight, position_embedding, pre_ln.*, post_ln.*, proj.weight, layers.{i}.*
    with layers.{i}.{ln_1, ln_2, attn.qkv, attn.proj, mlp.fc1, mlp.fc2}.{weight, bias}: attn.in_proj_{weight,bias} ([q; k; v])
    re-packed per 64-wide head [q_h | k_h | v_h] (pack_heads), attn.out_proj -> attn.proj, mlp.c_fc -> mlp.fc1, mlp.c_proj ->
    mlp.fc2.  text_projection and visual.proj are applied as x @ P there and become the Linear weights P^T here.
    input_resolution / context_length / vocab_size (the entries build_model deletes) and logit_scale are ignored; any other
    unknown key, and any missing one, raises K2Error naming it."""
    sd = {k: v for k, v in sd.items() if k not in _OPENAI_IGNORED}
    geo = openai_clip_geometry(sd)
    _require_keys(sd, openai_clip_keys(geo["text"]["layers"], geo["vision"]["layers"]), "OpenAI CLIP")
    towers = []
    for top, prefix, g in ((_OPENAI_TEXT_TOP, "transformer.resblocks.{}.", geo["text"]),
                           (_OPENAI_VISION_TOP, "visual.transformer.resblocks.{}.", geo["vision"])):
        for i in range(g["layers"]):
            for s in _WB:
                k = f"{prefix.format(i)}attn.in_proj_{s}"
                if sd[k].shape[0] != 3 * g["width"]:
                    raise K2Error(f"OpenAI CLIP state dict: {k} has {sd[k].shape[0]} rows, not 3 x {g['width']}")
        out = _stack_to_k2(sd, top, prefix, _OPENAI_LAYER, _OPENAI_QKV, g["layers"], "layers.{}.", "attn.qkv", 64)
        out["proj.weight"] = out["proj.weight"].t().contiguous()    # applied as x @ P in clip/model.py
        towers.append(out)
    return towers[0], towers[1], geo


def load_openai_clip(path_or_sd):
    """An OpenAI CLIP state dict from a path or as given: a TorchScript archive (what the `clip` package downloads, e.g.
    ViT-L-14.pt: torch.jit.load(...).state_dict()) or a plain torch.save'd state dict.  K2Error names a missing file."""
    if isinstance(path_or_sd, dict):
        return dict(path_or_sd)
    path = os.fspath(path_or_sd)
    if not os.path.exists(path):
        raise K2Error(f"OpenAI CLIP checkpoint {path} not found")
    try:
        m = torch.jit.load(path, map_location="cpu")
    except RuntimeError:
        m = None
    if m is not None:
        return {k: v for k, v in m.state_dict().items()}
    sd = torch.load(path, map_location="cpu", weights_only=True)
    if not isinstance(sd, dict):
        raise K2Error(f"OpenAI CLIP checkpoint {path}: neither a TorchScript archive nor a state dict")
    return sd


def read_json(folder, name, what, required=True):
    """folder/name parsed as JSON.  A missing file raises K2Error naming it (`what` says who asked), or gives None when the
    file is not required."""
    f = os.path.join(folder, name)
    if not os.path.exists(f):
        if required:
            raise K2Error(f"{what}: {f} not found")
        return None
    with open(f, encoding="utf-8") as fh:
        return json.load(fh)


def load_weights(folder, candidates, what):
    """A component's state dict on the CPU from the first of `candidates` (file names in folder, most preferred first) that
    exists: a *.safetensors file through the safetensors package, skipped when that does not import; any other file with
    torch.load (weights_only).  K2Error names the files when none can be read."""
    try:
        from safetensors.torch import load_file
    except ImportError:
        load_file = None
    for name in candidates:
        f = os.path.join(folder, name)
        if not os.path.exists(f):
            continue
        if not name.endswith(".safetensors"):
            return torch.load(f, map_location="cpu", weights_only=True)
        if load_file is not None:
            return load_file(f)
    skipped = load_file is None and any(n.endswith(".safetensors") for n in candidates)
    note = " (safetensors is not installed)" if skipped else ""
    raise K2Error(f"{what}: {' or '.join(os.path.join(folder, n) for n in candidates)} not found{note}")


# this package's MoVQ names -> diffusers VQModel names: (pattern, replacement) applied in order, before the up-block numbering
_MOVQ_RENAME = [(r"^encoder\.down\.(\d+)\.block\.", r"encoder.down_blocks.\1.resnets."),
                (r"^encoder\.down\.(\d+)\.attn\.", r"encoder.down_blocks.\1.attentions."),
                (r"^encoder\.down\.(\d+)\.downsample\.", r"encoder.down_blocks.\1.downsamplers.0."),
                (r"^(encoder|decoder)\.mid\.block_1\.", r"\1.mid_block.resnets.0."),
                (r"^(encoder|decoder)\.mid\.block_2\.", r"\1.mid_block.resnets.1."),
                (r"^(encoder|decoder)\.mid\.attn_1\.", r"\1.mid_block.attentions.0."),
                (r"^(encoder|decoder)\.norm_out\.", r"\1.conv_norm_out."),
                (r"\.upsample\.", ".upsamplers.0."), (r"\.nin_shortcut\.", ".conv_shortcut."),
                (r"(\.attentions\.\d+\.)q\.", r"\1to_q."), (r"(\.attentions\.\d+\.)k\.", r"\1to_k."),
                (r"(\.attentions\.\d+\.)v\.", r"\1to_v."), (r"(\.attentions\.\d+\.)proj_out\.", r"\1to_out.0."),
                (r"^(encoder\..*\.attentions\.\d+\.)norm\.", r"\1group_norm."),
                (r"^(decoder\..*\.attentions\.\d+\.)norm\.", r"\1spatial_norm.")]
# the attention names older diffusers conversions wrote (AttentionBlock, before the Attention refactor)
_MOVQ_LEGACY = re.compile(r"^(.*\.attentions\.\d+\.)(query|key|value|proj_attn)\.(weight|bias)$")
_MOVQ_LEGACY_NAME = {"query": "to_q", "key": "to_k", "value": "to_v", "proj_attn": "to_out.0"}
_MOVQ_LINEAR = re.compile(r"\.attentions\.\d+\.(to_q|to_k|to_v|to_out\.0)\.weight$")


def _movq_names(ddconfig):
    """{this package's key: diffusers VQModel key} for every parameter `vqgan.autoencoder.MOVQ(ddconfig, ...)` registers.
    diffusers numbers the decoder's up_blocks from the lowest resolution, the reference's decoder.up from the highest."""
    from .vqgan.autoencoder import MOVQ
    n = len(ddconfig["ch_mult"])
    names = {}
    for k in MOVQ(ddconfig, 1, ddconfig["z_channels"], device="meta").state_dict():
        d = re.sub(r"^decoder\.up\.(\d+)\.block\.", lambda m: f"decoder.up_blocks.{n - 1 - int(m.group(1))}.resnets.", k)
        d = re.sub(r"^decoder\.up\.(\d+)\.", lambda m: f"decoder.up_blocks.{n - 1 - int(m.group(1))}.", d)
        d = re.sub(r"^(decoder\.up_blocks\.\d+\.)attn\.", r"\1attentions.", d)
        for pat, rep in _MOVQ_RENAME:
            d = re.sub(pat, rep, d)
        names[k] = d
    return names


def diffusers_movq_to_k2(sd, config):
    """diffusers `VQModel` state dict (norm_type "spatial": the Kandinsky 2.2 decoder folders' `movq/`) -> `vqgan.autoencoder.MOVQ`
    keys for the geometry `config` (a MOVQ ddconfig, e.g. the first item of diffusers_compat.movq_config).  The names:
        encoder.down_blocks.{i}.resnets.{j} / .attentions.{j} / .downsamplers.0   -> encoder.down.{i}.block.{j} / .attn.{j} / .downsample
        {en,de}coder.mid_block.resnets.{0,1} / .attentions.0                      -> {en,de}coder.mid.block_{1,2} / .attn_1
        decoder.up_blocks.{i}.resnets.{j} / .attentions.{j} / .upsamplers.0       -> decoder.up.{n-1-i}.block.{j} / .attn.{j} / .upsample
        {en,de}coder.conv_norm_out -> norm_out;  conv_shortcut -> nin_shortcut
        attention group_norm (encoder) / spatial_norm (decoder) -> norm;  to_q / to_k / to_v / to_out.0 -> q / k / v / proj_out
    the SpatialNorm's norm_layer / conv_y / conv_b, conv_in / conv_out, quant_conv, post_quant_conv and quantize.embedding keep
    their names.  The attention's Linear weights [C, C] become 1x1 convolution weights [C, C, 1, 1].  The names older diffusers
    conversions gave the attention projections (query / key / value / proj_attn) are taken as to_q / to_k / to_v / to_out.0.
    Unknown and missing keys raise K2Error naming them.  Restated from diffusers' published layout (diffusers is not a
    dependency)."""
    names = _movq_names(config)
    renamed = {}
    for k, v in sd.items():
        m = _MOVQ_LEGACY.match(k)
        d = f"{m.group(1)}{_MOVQ_LEGACY_NAME[m.group(2)]}.{m.group(3)}" if m else k
        if d in renamed:
            raise K2Error(f"diffusers MoVQ state dict: {k!r} and another key both give {d!r}")
        renamed[d] = v
    _require_keys(renamed, list(names.values()), "diffusers MoVQ")
    out = {}
    for k, d in names.items():
        t = renamed[d]
        out[k] = t.reshape(t.shape[0], -1, 1, 1) if _MOVQ_LINEAR.search(d) else t
    return out


def k2_to_diffusers_movq(sd, config):
    """Inverse of diffusers_movq_to_k2 (export, and the round-trip test): the attention's 1x1 convolution weights become
    Linear weights [C, C].  Unknown and missing keys raise K2Error naming them."""
    names = _movq_names(config)
    _require_keys(sd, list(names), "MoVQ")
    return {d: sd[k].reshape(sd[k].shape[0], -1) if _MOVQ_LINEAR.search(d) else sd[k] for k, d in names.items()}


_DPT_HYBRID_TOP = {"cls_token": "dpt.embeddings.cls_token", "position_embedding": "dpt.embeddings.position_embeddings",
                   "projection.weight": "dpt.embeddings.projection.weight",
                   "projection.bias": "dpt.embeddings.projection.bias"}
_BIT_PREFIX = "dpt.embeddings.backbone."


def transformers_dpt_hybrid_keys(config):
    """Every key of a transformers `DPTForDepthEstimation` state dict with the hybrid (BiT) backbone for a config.json dict,
    including the ones transformers_dpt_hybrid_to_k2 drops."""
    from .model.depth import _bit_layer_shapes, dpt_hybrid_config, k2_hybrid_shapes
    c = dpt_hybrid_config(config)
    keys = _stack_keys([*_DPT_HYBRID_TOP.values(), "dpt.layernorm.weight", "dpt.layernorm.bias"], "dpt.encoder.layer.{}.",
                       _DPT_LAYER, _DPT_QKV, c["num_hidden_layers"])
    keys += [_BIT_PREFIX + k for k in _bit_layer_shapes(c["bit"])]
    keys += [k for k in k2_hybrid_shapes(c) if k.startswith(("neck.", "head."))]
    return keys + [f"neck.fusion_stage.layers.0.residual_layer1.{conv}.{s}" for conv in ("convolution1", "convolution2")
                   for s in _WB]


def transformers_dpt_hybrid_to_k2(sd, config):
    """transformers `DPTForDepthEstimation` state dict with the hybrid backbone (MiDaS v3 DPT-Hybrid, Intel/dpt-hybrid-midas)
    and its config.json dict -> `model.depth.DPTDepthEstimator` names:
        cls_token [H], position_embedding [T, H], projection.{weight, bias} (the 1x1 token projection of the stage-3 map),
        bit.* (dpt.embeddings.backbone.bit.*: the BiT stem and stages, weights not yet standardised),
        layers.{i}.* as transformers_dpt_to_k2 packs them, neck.* (reassemble stages 2 and 3 only) and head.*.
    Dropped on purpose, as in transformers_dpt_to_k2: dpt.layernorm.* and neck.fusion_stage.layers.0.residual_layer1.*.
    Unknown and missing keys raise K2Error naming them."""
    from .model.depth import dpt_hybrid_config
    _require_keys(sd, transformers_dpt_hybrid_keys(config), "transformers DPT-Hybrid")
    out = _stack_to_k2(sd, _DPT_HYBRID_TOP, "dpt.encoder.layer.{}.", _DPT_LAYER, _DPT_QKV,
                       dpt_hybrid_config(config)["num_hidden_layers"], "layers.{}.", "attn.qkv", 64)
    out["cls_token"] = out["cls_token"].reshape(-1)
    out["position_embedding"] = out["position_embedding"][0]
    out.update({k[len(_BIT_PREFIX):]: v for k, v in sd.items() if k.startswith(_BIT_PREFIX)})
    out.update({k: v for k, v in sd.items() if k.startswith(("neck.", "head."))
                and not k.startswith("neck.fusion_stage.layers.0.residual_layer1.")})
    return out
