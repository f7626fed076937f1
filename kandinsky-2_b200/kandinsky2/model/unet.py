"""H100-native Text2ImUNet: the reference's module boundary, compute in libk2b200.so.

Drop-in for kandinsky2/model/text2im_model2_1.py:13-155 (Text2ImUNet / InpaintText2ImUNet) and its base
kandinsky2/model/unet.py:343-611 (UNetModel): same constructor keywords, same state_dict keys and shapes
(so reference checkpoints load unchanged), same forward / del_cache / convert_to_fp16 / dtype surface.
Nothing here computes with torch: forward() replays a pre-built launch list of C-ABI kernels
(include/k2b200.h) over pre-allocated NHWC fp16 buffers, captured in a CUDA graph per input geometry.

Layer program per block (reference file:line in parentheses):
  ResBlock (unet.py:193-220)       norm[GN32+SiLU (+2x up / avg-pool of h and x)] -> conv3x3
                                   -> norm[GN32 * (1+scale) + shift, SiLU] -> conv3x3 with the
                                   skip folded in (identity: epilogue residual; 1x1: extra K segments, and
                                   the torch.cat of the up path is read as two sources)
  AttentionBlock (unet.py:260-269) norm -> qkv GEMM -> attention_d64 (encoder K/V cached per
                                   generation) -> proj GEMM + residual
  norm = ONE k2_gn_apply_fold launch: the statistics come from partial sums the producing conv's epilogue wrote
  time/cond head                   timestep_embedding, time_embed MLP, one batched GEMM for all 36 emb_layers
"""
import os

import torch
import torch.nn as nn

from .. import ops
from .._native import K2Error
from ..launch_plan import LaunchPlan


# the up ResBlocks' first conv (3x3 over the nearest-2x upsampled activations) as four 2x2 phase convolutions (ops.py)
_UP2 = os.environ.get("K2_UP2", "1") != "0"


# diffusers ImageHintTimeEmbedding.input_hint_block: (Cin, Cout, stride) of its eight 3x3 convolutions (SiLU between them)
_HINT_STEM = [(3, 16, 1), (16, 16, 1), (16, 32, 2), (32, 32, 1), (32, 96, 2), (96, 96, 1), (96, 256, 2), (256, 4, 1)]


def _topology(in_ch, mc, mult, nrb, attention_ds):
    """Stages as lists of blocks; block = list of ('conv', cin, cout) | ('res', cin, cout, updown) | ('attn', ch)."""
    ch = mult[0] * mc
    inp = [[("conv", in_ch, ch)]]
    chans = [ch]
    ds = 1
    for level, m in enumerate(mult):
        for _ in range(nrb):
            blk = [("res", ch, m * mc, None)]
            ch = m * mc
            if ds in attention_ds:
                blk.append(("attn", ch))
            inp.append(blk)
            chans.append(ch)
        if level != len(mult) - 1:
            inp.append([("res", ch, ch, "down")])
            chans.append(ch)
            ds *= 2
    mid = [("res", ch, ch, None), ("attn", ch), ("res", ch, ch, None)]
    out = []
    for level, m in list(enumerate(mult))[::-1]:
        for i in range(nrb + 1):
            blk = [("res", ch + chans.pop(), m * mc, None)]
            ch = m * mc
            if ds in attention_ds:
                blk.append(("attn", ch))
            if level and i == nrb:
                blk.append(("res", ch, ch, "up"))
                ds //= 2
            out.append(blk)
    return inp, mid, out


class _Node(nn.Module):
    """Empty container: parameters hang off a tree of these so state_dict keys equal the reference's."""


class Text2ImUNet(nn.Module):
    def __init__(self, model_dim, image_encoder_in_dim=768, text_encoder_in_dim1=1024, text_encoder_in_dim2=768,
                 num_image_embs=10, pooling_type="attention_pooling", *, in_channels, model_channels, out_channels,
                 num_res_blocks, attention_resolutions, dropout=0, channel_mult=(1, 2, 4, 8), conv_resample=True,
                 dims=2, num_classes=None, use_checkpoint=False, use_fp16=False, num_heads=1, num_head_channels=-1,
                 num_heads_upsample=-1, use_scale_shift_norm=False, resblock_updown=False, cache_text_emb=True,
                 use_flash_attention=False, cond_version="2.1", device=None, param_dtype=torch.float32, hint_channels=0):
        super().__init__()
        if not (use_scale_shift_norm and resblock_updown and num_head_channels == 64 and dims == 2 and
                num_classes is None and dropout == 0):
            raise NotImplementedError(
                "k2b200 implements the Kandinsky-2.1/2.2 decoder configuration: use_scale_shift_norm, "
                "resblock_updown, num_head_channels=64, dims=2, dropout=0 (kandinsky2/configs.py:125-149)")
        if cond_version == "2.1" and pooling_type != "from_model":
            raise NotImplementedError("pooling_type='from_model' (CONFIG_2_1) is the implemented conditioning head")
        self.model_dim = model_dim
        self.in_channels = in_channels
        self.model_channels = model_channels
        self.out_channels = out_channels
        self.num_res_blocks = num_res_blocks
        self.attention_resolutions = tuple(attention_resolutions)
        self.channel_mult = tuple(channel_mult)
        self.num_head_channels = num_head_channels
        self.num_image_embs = num_image_embs
        self.pooling_type = pooling_type
        self.cache_text_emb = cache_text_emb
        self.cond_version = cond_version
        # Kandinsky 2.2 ControlNet-depth (BASELINE configs[4]; diffusers addition_embed_type="image_hint"): `hint_channels` of
        # the in_channels come from add_embedding.input_hint_block(hint) instead of the caller's x
        self.hint_channels = hint_channels
        if hint_channels and (cond_version != "2.2" or hint_channels != 4):
            raise NotImplementedError("the hint stem belongs to the 2.2 head and produces 4 feature channels")
        self.use_fp16 = use_fp16
        self.dtype = torch.float16 if use_fp16 else torch.float32  # reported only; storage is always fp16 NHWC
        self.image_encoder_in_dim = image_encoder_in_dim
        self.text_encoder_in_dim1 = text_encoder_in_dim1
        self.text_encoder_in_dim2 = text_encoder_in_dim2
        self.cache = None
        self._packed = None
        self._plans = {}
        self._lora = None        # (factors from checkpoints.lora_to_k2, scale) of the loaded adapter
        self._lora_base = None   # device copies of the unmerged packed attention weights while an adapter is merged
        self.use_cuda_graph = True

        mc = model_channels
        temb = 4 * mc
        self._topo = _topology(in_channels, mc, self.channel_mult, num_res_blocks, self.attention_resolutions)
        kw = dict(device=device, dtype=param_dtype)

        def P(path, *shape):
            node = self
            parts = path.split(".")
            for name in parts[:-1]:
                if name not in node._modules:
                    node.add_module(name, _Node())
                node = node._modules[name]
            node.register_parameter(parts[-1], nn.Parameter(torch.zeros(*shape, **kw), requires_grad=False))

        P("time_embed.0.weight", temb, mc); P("time_embed.0.bias", temb)
        P("time_embed.2.weight", temb, temb); P("time_embed.2.bias", temb)
        for prefix, blocks in (("input_blocks", self._topo[0]), ("middle_block", [self._topo[1]]),
                               ("output_blocks", self._topo[2])):
            for bi, blk in enumerate(blocks):
                for li, layer in enumerate(blk):
                    p = f"{prefix}.{li}." if prefix == "middle_block" else f"{prefix}.{bi}.{li}."
                    if layer[0] == "conv":
                        P(p + "weight", layer[2], layer[1], 3, 3); P(p + "bias", layer[2])
                    elif layer[0] == "res":
                        _, cin, cout, _ = layer
                        P(p + "in_layers.0.weight", cin); P(p + "in_layers.0.bias", cin)
                        P(p + "in_layers.2.weight", cout, cin, 3, 3); P(p + "in_layers.2.bias", cout)
                        P(p + "emb_layers.1.weight", 2 * cout, temb); P(p + "emb_layers.1.bias", 2 * cout)
                        P(p + "out_layers.0.weight", cout); P(p + "out_layers.0.bias", cout)
                        P(p + "out_layers.3.weight", cout, cout, 3, 3); P(p + "out_layers.3.bias", cout)
                        if cin != cout:
                            P(p + "skip_connection.weight", cout, cin, 1, 1); P(p + "skip_connection.bias", cout)
                    else:
                        ch = layer[1]
                        P(p + "norm.weight", ch); P(p + "norm.bias", ch)
                        P(p + "qkv.weight", 3 * ch, ch, 1); P(p + "qkv.bias", 3 * ch)
                        P(p + "encoder_kv.weight", 2 * ch, model_dim, 1); P(p + "encoder_kv.bias", 2 * ch)
                        P(p + "proj_out.weight", ch, ch, 1); P(p + "proj_out.bias", ch)
        ch0 = self.channel_mult[0] * mc
        P("out.0.weight", ch0); P("out.0.bias", ch0)
        P("out.2.weight", out_channels, ch0, 3, 3); P("out.2.bias", out_channels)
        if cond_version == "2.1":
            P("clip_to_seq.weight", model_dim * num_image_embs, image_encoder_in_dim)
            P("clip_to_seq.bias", model_dim * num_image_embs)
            P("to_model_dim_n.weight", model_dim, text_encoder_in_dim1); P("to_model_dim_n.bias", model_dim)
            P("proj_n.weight", temb, text_encoder_in_dim2); P("proj_n.bias", temb)
            P("ln_model_n.weight", temb); P("ln_model_n.bias", temb)
            P("img_layer.weight", temb, image_encoder_in_dim); P("img_layer.bias", temb)
        else:  # Kandinsky 2.2 (diffusers UNet2DConditionModel: ImageProjection + ImageTimeEmbedding)
            P("encoder_hid_proj.image_embeds.weight", model_dim * num_image_embs, image_encoder_in_dim)
            P("encoder_hid_proj.image_embeds.bias", model_dim * num_image_embs)
            P("encoder_hid_proj.norm.weight", model_dim); P("encoder_hid_proj.norm.bias", model_dim)
            P("add_embedding.image_proj.weight", temb, image_encoder_in_dim); P("add_embedding.image_proj.bias", temb)
            P("add_embedding.image_norm.weight", temb); P("add_embedding.image_norm.bias", temb)
            if hint_channels:
                for i, (ci, co, _) in enumerate(_HINT_STEM):
                    P(f"add_embedding.input_hint_block.{2 * i}.weight", co, ci, 3, 3)
                    P(f"add_embedding.input_hint_block.{2 * i}.bias", co)

    @torch.no_grad()
    def init_synthetic_(self, seed=0):
        """Random weights of this architecture, drawn on the parameters' own device (benchmarks: there are no
        checkpoints offline).  Fan-in scaled so activations stay O(1); the reference's zero_module() tensors are
        filled too (a zero-initialised UNet outputs exact zeros, nn.py:73-79)."""
        dev = self._param("time_embed.0.weight").device
        g = torch.Generator(device=dev).manual_seed(seed)
        for name, prm in self.named_parameters():
            if name.endswith("bias"):
                prm.normal_(0.0, 0.05, generator=g)
            elif prm.dim() == 1:
                prm.normal_(0.0, 0.1, generator=g).add_(1.0)
            else:
                fan_in = prm[0].numel()
                prm.normal_(0.0, fan_in ** -0.5, generator=g)
        self._invalidate()
        return self

    # ---------------------------------------------------------------- reference surface
    def convert_to_fp16(self):
        """Reference: casts the conv torso to fp16 (fp16_util.py:9-16). Here activations and conv weights are
        always fp16 with fp32 accumulation / GroupNorm / softmax; only the reported dtype changes."""
        self.use_fp16 = True
        self.dtype = torch.float16

    def convert_to_fp32(self):
        raise NotImplementedError("the sm_90a path stores activations in fp16 (BASELINE north_star); no fp32 torso")

    def del_cache(self):
        self.cache = None

    def load_state_dict(self, state_dict, strict=True, assign=False):
        self._invalidate()
        return super().load_state_dict(state_dict, strict=strict, assign=assign)

    def _apply(self, fn, recurse=True):
        self._invalidate()
        return super()._apply(fn, recurse)

    def _invalidate(self):
        self._packed = None
        self._lora_base = None
        self._plans = {}
        self.cache = None

    # ---------------------------------------------------------------- packing (once per checkpoint)
    def _param(self, key):
        node = self
        for name in key.split("."):
            node = node._modules[name] if name in node._modules else node._parameters[name]
        return node

    def finalize(self, release_params=False):
        """Re-layout the weights for the kernels (fp16 [Cout][taps*Cin] K-major, fp32 biases / gains)."""
        dev = self._param("time_embed.0.weight").device
        if dev.type != "cuda":
            raise K2Error("Text2ImUNet must live on a CUDA sm_90 device (module.to('cuda')); there is no CPU path")
        f32 = lambda k: self._param(k).detach().to(torch.float32).contiguous()
        pk = {"res": {}, "attn": {}}
        film_w, film_b, off = [], [], 0
        for prefix, blocks in (("input_blocks", self._topo[0]), ("middle_block", [self._topo[1]]),
                               ("output_blocks", self._topo[2])):
            for bi, blk in enumerate(blocks):
                for li, layer in enumerate(blk):
                    p = f"{prefix}.{li}." if prefix == "middle_block" else f"{prefix}.{bi}.{li}."
                    if layer[0] == "conv":
                        pk["stem_w"] = ops.pack_stem_weight(self._param(p + "weight"))
                        pk["stem_b"] = f32(p + "bias")
                    elif layer[0] == "res":
                        _, cin, cout, updown = layer
                        d = dict(g1=f32(p + "in_layers.0.weight"), b1=f32(p + "in_layers.0.bias"),
                                 w1=ops.pack_conv_weight(self._param(p + "in_layers.2.weight")),
                                 c1=f32(p + "in_layers.2.bias"),
                                 g2=f32(p + "out_layers.0.weight"), b2=f32(p + "out_layers.0.bias"),
                                 c2=f32(p + "out_layers.3.bias"), film_off=off)
                        if updown == "up":  # conv over the nearest-2x upsampled h as four 2x2 phase convs (ops.py)
                            d["w1u"] = ops.pack_conv_weight_up2(self._param(p + "in_layers.2.weight"))
                        w2 = ops.pack_conv_weight(self._param(p + "out_layers.3.weight"))
                        if cin != cout:
                            d["wskip_raw"] = self._param(p + "skip_connection.weight").detach()
                            d["c2"] = d["c2"] + f32(p + "skip_connection.bias")
                        d["w2"] = w2
                        film_w.append(f32(p + "emb_layers.1.weight")); film_b.append(f32(p + "emb_layers.1.bias"))
                        off += 2 * cout
                        pk["res"][p] = d
                    else:
                        ch = layer[1]
                        pk["attn"][p] = dict(
                            g=f32(p + "norm.weight"), b=f32(p + "norm.bias"),
                            wqkv=ops.pack_conv_weight(self._param(p + "qkv.weight")), bqkv=f32(p + "qkv.bias"),
                            wenc=ops.pack_conv_weight(self._param(p + "encoder_kv.weight")), benc=f32(p + "encoder_kv.bias"),
                            wproj=ops.pack_conv_weight(self._param(p + "proj_out.weight")), bproj=f32(p + "proj_out.bias"))
        # all 2*Cout x temb emb_layers of the network as ONE weight (one GEMV-like launch per step), stored fp16:
        # it is the only per-step weight stream that is pure bandwidth (the reference keeps it fp32, fp16_util.py:13)
        pk["film_w"] = torch.cat(film_w, 0).to(torch.float16).contiguous()
        pk["film_b"] = torch.cat(film_b, 0).contiguous()
        pk["film_total"] = off
        pk["te0_w"], pk["te0_b"] = f32("time_embed.0.weight"), f32("time_embed.0.bias")
        pk["te2_w"], pk["te2_b"] = f32("time_embed.2.weight"), f32("time_embed.2.bias")
        pk["out_g"], pk["out_b"] = f32("out.0.weight"), f32("out.0.bias")
        pk["out_w"] = ops.pad_rows(ops.pack_conv_weight(self._param("out.2.weight")), 16)
        pk["out_c"] = f32("out.2.bias")
        if self.cond_version == "2.1":
            for k in ("clip_to_seq", "to_model_dim_n", "proj_n", "ln_model_n", "img_layer"):
                pk[k + "_w"], pk[k + "_b"] = f32(k + ".weight"), f32(k + ".bias")
        else:
            pk["ip_w"], pk["ip_b"] = f32("encoder_hid_proj.image_embeds.weight"), f32("encoder_hid_proj.image_embeds.bias")
            pk["ipn_w"], pk["ipn_b"] = f32("encoder_hid_proj.norm.weight"), f32("encoder_hid_proj.norm.bias")
            pk["ae_w"], pk["ae_b"] = f32("add_embedding.image_proj.weight"), f32("add_embedding.image_proj.bias")
            pk["aen_w"], pk["aen_b"] = f32("add_embedding.image_norm.weight"), f32("add_embedding.image_norm.bias")
            if self.hint_channels:
                hw = []
                for i, (ci, co, _) in enumerate(_HINT_STEM):
                    w = self._param(f"add_embedding.input_hint_block.{2 * i}.weight")
                    wp = ops.pack_stem_weight(w) if i == 0 else ops.pack_conv_weight(w)
                    hw.append((ops.pad_rows(wp, 16), f32(f"add_embedding.input_hint_block.{2 * i}.bias")))
                pk["hint"] = hw
        self._packed = pk
        self._plans = {}
        self.cache = None
        self._lora_base = None
        if self._lora is not None:  # a loaded adapter survives re-packing (load_state_dict, .to)
            self._merge_lora()
        if release_params:
            for prm in self.parameters():
                prm.data = torch.empty(0, device=dev, dtype=prm.dtype)
        return self

    # ---------------------------------------------------------------- LoRA adapters, merged into the packed weights
    _LORA_WEIGHTS = (("wqkv", "qkv"), ("wenc", "encoder_kv"), ("wproj", "proj_out"))

    @property
    def lora_scale(self):
        """Scale of the loaded LoRA adapter, None when there is none."""
        return None if self._lora is None else self._lora[1]

    def load_lora(self, state_dict, scale=1.0):
        """Merge a LoRA adapter of the attention blocks -- diffusers' `LoRAAttnAddedKVProcessor` weights as
        `save_attn_procs` / `AttnProcsLayers` write them (checkpoints.lora_to_k2) -- into the packed weights:
        W = W_base + scale * up @ down, computed by k2_lora_merge in fp32 and rounded once to fp16 (diffusers' fuse_lora).
        The merge writes the packed tensors in place, so captured launch plans and step graphs keep their addresses and
        need no rebuild; the cached conditioning is dropped because the encoder K/V projections use the merged weights.
        On first use the unmerged packed weights are copied on the device (restored by unload_lora).  Loading again
        replaces the adapter (adapters do not stack; a new scale means loading again).  state_dict() never changes."""
        factors = self.lora_factors(state_dict)
        if self._packed is None:
            self.finalize()
        self._lora = (factors, float(scale))
        self._merge_lora()

    def lora_factors(self, state_dict):
        """{packed weight key: (up, down)} of an adapter of this UNet's attention blocks (checkpoints.lora_to_k2)."""
        from ..checkpoints import lora_to_k2
        return lora_to_k2(state_dict, in_channels=self.in_channels, model_channels=self.model_channels,
                          channel_mult=self.channel_mult, num_res_blocks=self.num_res_blocks,
                          attention_ds=self.attention_resolutions, model_dim=self.model_dim,
                          head_dim=self.num_head_channels)

    def unload_lora(self):
        """Restore the unmerged packed weights (bit-exact), free their copy and drop the cached conditioning."""
        if self._lora_base is not None and self._packed is not None:
            for p, a in self._packed["attn"].items():
                for name, _ in self._LORA_WEIGHTS:
                    a[name].copy_(self._lora_base[p][name])
        self._lora = None
        self._lora_base = None
        self.cache = None

    def lora_weights(self):
        """(adapter key, unmerged weight, packed weight) of every packed attention weight an adapter changes, the form
        ops.lora_merge_weights takes; the unmerged weight is the packed one while no adapter is merged."""
        for p, a in self._packed["attn"].items():
            base = a if self._lora_base is None else self._lora_base[p]
            for name, target in self._LORA_WEIGHTS:
                yield p + target + ".weight", base[name], a[name]

    def _merge_lora(self):
        if self._lora_base is None:
            self._lora_base = {p: {name: a[name].clone() for name, _ in self._LORA_WEIGHTS}
                               for p, a in self._packed["attn"].items()}
        ops.lora_merge_weights(self.lora_weights(), *self._lora)
        self.cache = None

    def _skip_weight(self, d, c0, c1):
        """[W2 | Wskip] packed for the (conv3x3 of h, 1x1 of x0, 1x1 of x1) K segments."""
        key = ("wcat", c0, c1)
        if key not in d:
            ws = ops.pack_conv_weight(d["wskip_raw"], split=(c0, c1) if c1 else None)
            d[key] = torch.cat([d["w2"], ws], 1).contiguous()
        return d[key]

    # ---------------------------------------------------------------- conditioning (once per generation)
    def hint_features(self, hint):
        """diffusers ImageHintTimeEmbedding.input_hint_block: hint fp32 [N, 3, 8h, 8w] -> features fp32 NCHW [N, 4, h, w]
        (eight 3x3 convolutions on tensor cores, SiLU between them, three of them stride 2 = 'same' conv + keeping the even
        pixels).  Runs once per generation."""
        pk = self._packed
        hint = hint.float().contiguous()
        h = None
        for i, ((ci, co, stride), (w, b)) in enumerate(zip(_HINT_STEM, pk["hint"])):
            last = i + 1 == len(_HINT_STEM)
            if i == 0:
                h = ops.conv_gemm([(ops.stem_im2col(hint), 1)], w, co, bias=b)
            else:
                h = ops.conv_gemm([(h, 9)], w, co, bias=b, out_mode=1 if last else 0)
            if stride == 2:
                h = ops.subsample2(h, 0, 0)
            if not last:
                ops.silu_f16_(h)
        return h

    def get_text_emb(self, full_emb=None, pooled_emb=None, image_emb=None, hint=None):
        """text2im_model2_1.py:57-80. Returns and caches dict(xf_proj fp32 [N,4mc], xf_out fp16 [N,ctx,model_dim],
        enc_kv {attention layer -> fp16 [N,ctx,2C]}): the encoder K/V projections are constant over the
        sampling loop, so they are hoisted out of the per-step forward."""
        if self.cache is not None and self.cache_text_emb:
            return self.cache
        if self._packed is None:
            self.finalize()
        pk = self._packed
        md = self.model_dim
        image_emb = image_emb.float().contiguous()
        N = image_emb.shape[0]
        if self.cond_version == "2.1":
            clip_seq = ops.linear(image_emb, pk["clip_to_seq_w"], pk["clip_to_seq_b"]).reshape(N, self.num_image_embs, md)
            full = full_emb.float().contiguous()
            tok = ops.linear(full.reshape(-1, full.shape[-1]), pk["to_model_dim_n_w"], pk["to_model_dim_n_b"])
            xf = torch.cat([clip_seq, tok.reshape(N, -1, md)], 1).contiguous()
            proj = ops.layernorm(ops.linear(pooled_emb.float().contiguous(), pk["proj_n_w"], pk["proj_n_b"]),
                                 pk["ln_model_n_w"], pk["ln_model_n_b"])
            xf_proj = ops.linear(image_emb, pk["img_layer_w"], pk["img_layer_b"], add=proj)
        else:
            tok = ops.linear(image_emb, pk["ip_w"], pk["ip_b"]).reshape(N * self.num_image_embs, md)
            xf = ops.layernorm(tok, pk["ipn_w"], pk["ipn_b"]).reshape(N, self.num_image_embs, md)
            xf_proj = ops.layernorm(ops.linear(image_emb, pk["ae_w"], pk["ae_b"]), pk["aen_w"], pk["aen_b"])
        xf16 = ops.f32_to_f16(xf)
        enc_kv = {}
        for p, a in pk["attn"].items():
            enc_kv[p] = ops.gemm_rows(xf16, a["wenc"], a["wenc"].shape[0], bias=a["benc"])
        out = dict(xf_proj=xf_proj, xf_out=xf16, enc_kv=enc_kv)
        if self.hint_channels:
            if hint is None:
                raise K2Error("this UNet was built with a ControlNet hint stem: pass hint= [N, 3, 8h, 8w]")
            out["hint_feat"] = self.hint_features(hint)
        if self.cache_text_emb:
            self.cache = out
        return out

    def bind_slot(self, plan, slot, negative_emb, positive_emb, wenc=None, full_emb=None, pooled_emb=None, hint=None):
        """Write the conditioning of slot `slot` of a plan of N = 2 S rows into the plan's xf_proj and encoder K/V rows, leaving
        every other row and every buffer address (so a CUDA graph captured on the plan) as it is.  Image embeddings are
        [image_encoder_in_dim].  Kandinsky 2.2: negative_emb goes to row `slot`, positive_emb to row S + slot.  Kandinsky 2.1
        (the conditional rows first): row `slot` takes positive_emb, full_emb[0] and pooled_emb[0], row S + slot takes
        negative_emb, full_emb[1] and pooled_emb[1] (full_emb [2, text_len, text_encoder_in_dim1], pooled_emb [2,
        text_encoder_in_dim2]: the conditional and unconditional rows the text encoder gives for one prompt).
        Each output row of get_text_emb depends on its input row alone, but the encoder K/V GEMM picks its split-K factor
        from its row count (k2_conv_gemm), which changes the fp32 summation order; so the rows are computed at the plan's batch
        (the other input rows zero), and a slot's conditioning has the same bits in every slot and, at S = 1, those
        generate_text2img(batch_size=1) binds.  The model's cached conditioning is left untouched.
        wenc ({attention layer -> packed encoder_kv weight}, or None = the packed weights): the weights the slot's encoder K/V
        rows are computed with, e.g. the encoder_kv weights an adapter merges (the batcher's per-request adapters).
        hint (ControlNet UNets only, which need it): the slot's depth map [1, 3, 8h, 8w]; its hint features are computed by
        the hint stem at the plan's batch, the map in rows `slot` and S + slot and zeros elsewhere, since the stem's
        convolutions too pick split-K from the row count: at S = 1 they are what generate_controlnet binds."""
        v21 = self.cond_version == "2.1"
        if bool(self.hint_channels) != (hint is not None):
            raise K2Error("bind_slot: a ControlNet UNet needs hint= (the slot's depth map), a text2img UNet takes none")
        if v21 != (full_emb is not None) or v21 != (pooled_emb is not None):
            raise K2Error("bind_slot: the Kandinsky 2.1 UNet needs full_emb and pooled_emb, the 2.2 one takes neither")
        S = plan.N // 2
        if not 0 <= slot < S:
            raise K2Error(f"bind_slot: slot {slot} outside [0, {S})")
        first, second = (positive_emb, negative_emb) if v21 else (negative_emb, positive_emb)
        emb = torch.zeros(plan.N, negative_emb.shape[-1], device=plan.dev, dtype=torch.float32)
        emb[slot] = first.reshape(-1).to(emb.device, torch.float32)
        emb[S + slot] = second.reshape(-1).to(emb.device, torch.float32)
        text = {}
        if v21:
            for name, t in (("full_emb", full_emb), ("pooled_emb", pooled_emb)):
                rows = torch.zeros((plan.N,) + tuple(t.shape[1:]), device=plan.dev, dtype=torch.float32)
                rows[slot] = t[0]
                rows[S + slot] = t[1]
                text[name] = rows
        if hint is not None:
            rows = torch.zeros((plan.N,) + tuple(hint.shape[1:]), device=plan.dev, dtype=torch.float32)
            rows[slot] = rows[S + slot] = hint[0].to(plan.dev, torch.float32)
            text["hint"] = rows
        saved, keep = self.cache, self.cache_text_emb
        self.cache, self.cache_text_emb = None, False
        try:
            cond = self.get_text_emb(image_emb=emb, **text)
        finally:
            self.cache, self.cache_text_emb = saved, keep
        if wenc is not None:
            attn = self._packed["attn"]
            cond["enc_kv"] = {p: ops.gemm_rows(cond["xf_out"], w, w.shape[0], bias=attn[p]["benc"]) for p, w in wenc.items()}
        plan.bind_rows(cond, (slot, S + slot))

    # ---------------------------------------------------------------- forward
    def forward(self, x, timesteps, full_emb=None, pooled_emb=None, image_emb=None, inpaint_image=None,
                inpaint_mask=None, hint=None):
        """x [N, 4, h, w] (any float dtype), timesteps [N] -> [N, out_channels, h, w] in x.dtype
        (text2im_model2_1.py:85-103; inpaint variant :146-155)."""
        if not x.is_cuda:
            raise K2Error("k2b200 UNet: input must be a CUDA tensor (no CPU fallback)")
        if self._packed is None:
            self.finalize()
        cond = self.get_text_emb(full_emb=full_emb, pooled_emb=pooled_emb, image_emb=image_emb, hint=hint)
        N, _, H, W = x.shape
        plan = self._plan(N, H, W, cond["xf_out"].shape[1])
        plan.bind(cond)
        plan.x_in.copy_(x)
        plan.t_in.copy_(timesteps)
        if self._inpainting:
            plan.img_in.copy_(inpaint_image) if inpaint_image is not None else plan.img_in.zero_()
            plan.mask_in.copy_(inpaint_mask) if inpaint_mask is not None else plan.mask_in.zero_()
        plan.run(self.use_cuda_graph)
        return plan.out.to(x.dtype) if x.dtype != torch.float32 else plan.out.clone()

    _inpainting = False

    def _plan(self, N, H, W, ctx):
        key = (N, H, W, ctx)
        if key not in self._plans:
            self._plans[key] = _Plan(self, N, H, W, ctx)
        return self._plans[key]


class InpaintText2ImUNet(Text2ImUNet):
    """text2im_model2_1.py:131-155: the stem sees cat([x, inpaint_image*inpaint_mask, inpaint_mask])."""
    _inpainting = True

    def __init__(self, *args, **kwargs):
        kwargs = dict(kwargs)
        self._latent_channels = kwargs["in_channels"]
        kwargs["in_channels"] = kwargs["in_channels"] * 2 + 1
        super().__init__(*args, **kwargs)


class _Plan(LaunchPlan):
    """Static launch list + buffers of one forward at a fixed (N, H, W); replayed eagerly or as a CUDA graph."""

    def __init__(self, model, N, H, W, ctx, attn_slabs=None):
        """attn_slabs (or None: the packed weights): dict(map=device int32 [N], layers={attention layer -> (wqkv fp16
        [slabs, 3C, C], wproj fp16 [slabs, C, C])}).  Image n's qkv and proj_out GEMMs then multiply slab map[n] of its
        layer's tables (k2_conv_gemm_wmap), read when the launch runs: rewriting the map or a slab changes what a replay of
        the plan computes without moving a buffer."""
        pk = model._packed
        dev = pk["te0_w"].device
        super().__init__(dev, N)
        self.m = model
        self.N, self.H, self.W, self.ctx = N, H, W, ctx
        f32 = dict(device=dev, dtype=torch.float32)
        lat = model._latent_channels if model._inpainting else model.in_channels - model.hint_channels
        self.x_in = torch.zeros(N, lat, H, W, **f32)
        if model.hint_channels:
            self.hint_in = torch.zeros(N, model.hint_channels, H, W, **f32)
        self.t_in = torch.zeros(N, **f32)
        if model._inpainting:
            self.img_in = torch.zeros(N, lat, H, W, **f32)
            self.mask_in = torch.zeros(N, 1, H, W, **f32)
        self.out = torch.empty(N, model.out_channels, H, W, **f32)
        self.xf_proj = torch.zeros(N, 4 * model.model_channels, **f32)
        self.enc_kv = {}
        self._bound = None
        self.attn_slabs = attn_slabs
        self._build()

    def bind(self, cond):
        """Point the plan at this generation's conditioning (copied into the plan's static buffers)."""
        if self._bound is cond:
            return
        self.xf_proj.copy_(cond["xf_proj"])
        if self.m.hint_channels:
            self.hint_in.copy_(cond["hint_feat"])
        for p, buf in self.enc_kv.items():
            src = cond["enc_kv"][p]
            if buf.shape != src.shape:
                raise K2Error("context length changed between forwards: call del_cache() and rebuild the plan")
            buf.copy_(src)
        self._bound = cond

    def bind_rows(self, cond, rows):
        """Copy rows `rows` of a get_text_emb result computed at this plan's batch into the plan's conditioning buffers, in
        place (Text2ImUNet.bind_slot)."""
        idx = torch.tensor(rows, device=self.dev, dtype=torch.long)
        self.xf_proj[idx] = cond["xf_proj"][idx]
        if self.m.hint_channels:
            self.hint_in[idx] = cond["hint_feat"][idx]
        for p, buf in self.enc_kv.items():
            src = cond["enc_kv"][p]
            if buf.shape != src.shape:
                raise K2Error("bind_rows: the conditioning was not computed at this plan's batch and context length")
            buf[idx] = src[idx]
        self._bound = None

    # program -----------------------------------------------------------------------------------
    def _build(self):
        m, pk, N = self.m, self.m._packed, self.N
        S = self._add
        mc = m.model_channels
        temb = 4 * mc
        f32 = dict(device=self.dev, dtype=torch.float32)
        e0 = torch.empty(N, mc, **f32)
        e1 = torch.empty(N, temb, **f32)
        emb = torch.empty(N, temb, **f32)
        film = torch.empty(N, pk["film_total"], **f32)
        # the time embedding and all 36 FiLM projections (one 215 MB weight stream) run on a forked branch next to the stem
        # conv and the first ResBlock's norm -> conv; the first FiLM consumer joins it
        B_ = self._side
        B_(lambda: ops.timestep_embedding(self.t_in, mc, out=e0), "timestep_embedding")
        B_(lambda: ops.linear(e0, pk["te0_w"], pk["te0_b"], silu_out=True, out=e1), "linear")
        B_(lambda: ops.linear(e1, pk["te2_w"], pk["te2_b"], add=self.xf_proj, out=emb), "linear")
        B_(lambda: ops.linear(emb, pk["film_w"], pk["film_b"], silu_in=True, out=film), "linear")
        self.film = film

        H, W = self.H, self.W
        inp, mid, out = m._topo
        # stem: fp32 NCHW -> 3x3 patches -> GEMM
        cin = inp[0][0][1]
        kpad = (9 * cin + 63) // 64 * 64
        patches = self._new(N, H, W, kpad)
        h = self._new(N, H, W, inp[0][0][2])
        if m._inpainting:
            S(lambda: ops.stem_im2col(self.x_in, self.img_in, self.mask_in, mul23=True, kpad=kpad, out=patches), "stem_im2col")
        elif m.hint_channels:  # conv_in sees cat([x, hint features])
            S(lambda: ops.stem_im2col(self.x_in, self.hint_in, kpad=kpad, out=patches), "stem_im2col")
        else:
            S(lambda: ops.stem_im2col(self.x_in, kpad=kpad, out=patches), "stem_im2col")
        self._conv([(patches, 1)], pk["stem_w"], h.shape[-1], h, 2 * N * H * W * h.shape[-1] * 9 * cin, bias=pk["stem_b"])
        hs = [h]
        for bi, blk in enumerate(inp[1:], start=1):
            for li, layer in enumerate(blk):
                h = self._layer(f"input_blocks.{bi}.{li}.", layer, h, None)
            hs.append(h)
        for li, layer in enumerate(mid):
            h = self._layer(f"middle_block.{li}.", layer, h, None)
        for bi, blk in enumerate(out):
            skip = hs.pop()
            for li, layer in enumerate(blk):
                h = self._layer(f"output_blocks.{bi}.{li}.", layer, h, skip if li == 0 else None)
        # head: GN32 + SiLU + conv3x3 -> fp32 NCHW (unet.py:559-563; text2im_model2_1.py:101-102)
        hn = self._tmp("h1", *h.shape)
        self._norm(h, None, pk["out_g"], pk["out_b"], hn)
        S(lambda: ops.conv_gemm([(hn, 9)], pk["out_w"], m.out_channels, bias=pk["out_c"], out=self.out, out_mode=1),
          "conv_gemm", 2 * N * H * W * m.out_channels * 9 * h.shape[-1])
        self._join()

    def _layer(self, p, layer, a, b):
        pk, N, S = self.m._packed, self.N, self._add
        if layer[0] == "res":
            _, cin, cout, updown = layer
            d = pk["res"][p]
            Hi, Wi = a.shape[1], a.shape[2]
            Ho, Wo = (Hi, Wi) if updown is None else ((Hi // 2, Wi // 2) if updown == "down" else (Hi * 2, Wi * 2))
            h1 = self._tmp("h1", N, Ho, Wo, cin)
            h2 = self._tmp("h2", N, Ho, Wo, cout)
            h3 = self._tmp("h3", N, Ho, Wo, cout)
            o = self._new(N, Ho, Wo, cout)
            film = self.film[:, d["film_off"]:d["film_off"] + 2 * cout]
            flops1 = 2 * N * Ho * Wo * cout * 9 * cin  # of the reference graph (the up2 path executes 4/9 of them)
            if updown is None:
                xres = None
                self._norm(a, b, d["g1"], d["b1"], h1)
                self._conv([(h1, 9)], d["w1"], cout, h2, flops1, bias=d["c1"], part_slot="part_h2")
            elif updown == "up" and _UP2:
                # unet.py:198-203: h = conv(upsample(silu(norm(x)))), x = upsample(x).  The upsampled h is never written: the
                # conv runs over the low-resolution h as four 2x2 phase convolutions (k2b200.h, taps = 4)
                xres = self._tmp("xres", N, Ho, Wo, cin)
                h1s = self._tmp("h1s", N, Hi, Wi, cin)
                self._norm(a, b, d["g1"], d["b1"], h1s)
                self._side(lambda: ops.upsample2x(a, out=xres), "upsample")
                self._conv([(h1s, 4)], d["w1u"], cout, h2, flops1, bias=d["c1"], part_slot="part_h2")
            else:
                xres = self._tmp("xres", N, Ho, Wo, cin)
                self._norm(a, b, d["g1"], d["b1"], h1, resample=1 if updown == "down" else 2, xres=xres)
                self._conv([(h1, 9)], d["w1"], cout, h2, flops1, bias=d["c1"], part_slot="part_h2")
            self._join()  # FiLM rows (first ResBlock) / the skip upsampling (up ResBlocks) come from the forked branch
            self._norm(h2, None, d["g2"], d["b2"], h3, film=film)
            if cin == cout:
                if b is not None:
                    raise NotImplementedError("identity skip over a concatenated input")
                res = xres if xres is not None else a
                self._conv([(h3, 9)], d["w2"], cout, o, 2 * N * Ho * Wo * cout * 9 * cout, bias=d["c2"], residual=res)
            else:
                if updown is not None:
                    raise NotImplementedError("resampling ResBlock with a channel change")
                c0 = a.shape[-1]
                c1 = b.shape[-1] if b is not None else 0
                wcat = self.m._skip_weight(d, c0, c1)
                srcs = [(h3, 9), (a, 1)] + ([(b, 1)] if b is not None else [])
                self._conv(srcs, wcat, cout, o, 2 * N * Ho * Wo * cout * (9 * cout + cin), bias=d["c2"])
            return o
        # attention
        ch = layer[1]
        d = pk["attn"][p]
        heads = ch // 64
        _, Hh, Ww, _ = a.shape
        T = Hh * Ww
        xn = self._tmp("h1", N, Hh, Ww, ch)
        qkv = self._tmp("qkv", N, T, 3 * ch)
        att = self._tmp("att", N, T, ch)
        o = self._new(N, Hh, Ww, ch)
        enc = self._new(N, self.ctx, 2 * ch)
        self.enc_kv[p] = enc
        self._norm(a, None, d["g"], d["b"], xn, act=0)
        wproj, mapped = d["wproj"], {}
        if self.attn_slabs is None:
            self._gemm(xn.view(N, T, ch), d["wqkv"], 3 * ch, qkv, 2 * N * T * 3 * ch * ch, bias=d["bqkv"])
        else:
            # batched GEMMs over the N images of T tokens, image n with slab map[n]
            wqkv, wproj = self.attn_slabs["layers"][p]
            mapped = dict(w_map=self.attn_slabs["map"], n_slabs=wqkv.shape[0])
            self._conv([(xn, 1)], wqkv[0], 3 * ch, qkv.view(N, Hh, Ww, 3 * ch), 2 * N * T * 3 * ch * ch, bias=d["bqkv"],
                       want_stats=False, w_batch_stride=wqkv.stride(0), **mapped)
            mapped["w_batch_stride"] = wproj.stride(0)
            wproj = wproj[0]
        S(lambda: ops.attention_d64(qkv, heads, enc, out=att), "attention", 4 * N * T * (T + self.ctx) * ch)
        self._conv([(att.view(N, Hh, Ww, ch), 1)], wproj, ch, o, 2 * N * T * ch * ch, bias=d["bproj"], residual=a, **mapped)
        return o
