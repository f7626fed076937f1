"""TEST INFRASTRUCTURE (oracle): the Kandinsky 2.2 MoVQ in diffusers' form, restated (diffusers is not installed).

  VQMODEL_22         <- movq/config.json of the Kandinsky 2.2 decoder folders as restated here: a `VQModel` with norm_type
                        "spatial", block_out_channels (128, 256, 256, 512), two resnets per level, attention at the last level
  VQMODEL_TINY       <- the same layout at oracle/movq_oracle.py's DDCONFIG_TINY geometry
  vqmodel_spec       <- the state dict of `VQModel(**config)` under diffusers' names: Encoder (DownEncoderBlock2D /
                        AttnDownEncoderBlock2D, UNetMidBlock2D, conv_norm_out), quant_conv, quantize.embedding, post_quant_conv,
                        Decoder (UNetMidBlock2D and Up*DecoderBlock2D with SpatialNorm, up_blocks numbered from the lowest
                        resolution), attention as `Attention` with Linear to_q / to_k / to_v / to_out.0
  vqmodel_encode     <- VQModel.encode(x).latents = quant_conv(Encoder(x)): Downsample2D with padding 0 pads (0, 1, 0, 1) and
                        convolves with stride 2
  vqmodel_decode     <- VQModel.decode(h, force_not_quantize=True) = Decoder(post_quant_conv(h), h): SpatialNorm with the
                        latent nearest-resized to each feature map, single-head attention with residual

Restated, so unpinned.  What is pinned (tests/test_cpu_movq22.py): after kandinsky2.checkpoints.diffusers_movq_to_k2, oracle
movq_oracle.movq_decode / movq_encode (the reference's own network) equal these forwards in fp32."""
import torch
import torch.nn.functional as F

VQMODEL_22 = {
    "_class_name": "VQModel", "act_fn": "silu", "block_out_channels": [128, 256, 256, 512],
    "down_block_types": ["DownEncoderBlock2D", "DownEncoderBlock2D", "DownEncoderBlock2D", "AttnDownEncoderBlock2D"],
    "in_channels": 3, "latent_channels": 4, "layers_per_block": 2, "norm_num_groups": 32, "norm_type": "spatial",
    "num_vq_embeddings": 16384, "out_channels": 3, "sample_size": 32, "scaling_factor": 0.18215,
    "up_block_types": ["AttnUpDecoderBlock2D", "UpDecoderBlock2D", "UpDecoderBlock2D", "UpDecoderBlock2D"],
    "vq_embed_dim": 4}
VQMODEL_TINY = dict(VQMODEL_22, block_out_channels=[32, 64], layers_per_block=1, num_vq_embeddings=64,
                    down_block_types=["DownEncoderBlock2D", "AttnDownEncoderBlock2D"],
                    up_block_types=["AttnUpDecoderBlock2D", "UpDecoderBlock2D"])


def _conv(p, cout, cin, k, spec):
    spec += [(p + "weight", (cout, cin, k, k)), (p + "bias", (cout,))]


def _vec(p, c, spec):
    spec += [(p + "weight", (c,)), (p + "bias", (c,))]


def _spatial(p, c, zc, spec):
    _vec(p + "norm_layer.", c, spec)
    _conv(p + "conv_y.", c, zc, 1, spec)
    _conv(p + "conv_b.", c, zc, 1, spec)


def _resnet(p, cin, cout, zc, spec):
    """ResnetBlock2D (zc None: GroupNorm) or its SpatialNorm form (zc: the latent's channels)."""
    for norm, conv, ci in (("norm1.", "conv1.", cin), ("norm2.", "conv2.", cout)):
        _vec(p + norm, ci, spec) if zc is None else _spatial(p + norm, ci, zc, spec)
        _conv(p + conv, cout, ci, 3, spec)
    if cin != cout:
        _conv(p + "conv_shortcut.", cout, cin, 1, spec)


def _attention(p, c, zc, spec):
    _vec(p + "group_norm.", c, spec) if zc is None else _spatial(p + "spatial_norm.", c, zc, spec)
    for n in ("to_q.", "to_k.", "to_v.", "to_out.0."):
        spec += [(p + n + "weight", (c, c)), (p + n + "bias", (c,))]


def vqmodel_spec(cfg):
    """[(diffusers key, shape)] of VQModel(**cfg) with norm_type "spatial"."""
    boc, nl, zc = cfg["block_out_channels"], cfg["layers_per_block"], cfg["latent_channels"]
    ed, n = cfg["vq_embed_dim"], len(cfg["block_out_channels"])
    spec = []
    _conv("encoder.conv_in.", boc[0], cfg["in_channels"], 3, spec)
    cout = boc[0]
    for i, kind in enumerate(cfg["down_block_types"]):
        cin, cout = cout, boc[i]
        p = f"encoder.down_blocks.{i}."
        for j in range(nl):
            _resnet(p + f"resnets.{j}.", cin if j == 0 else cout, cout, None, spec)
            if kind.startswith("Attn"):
                _attention(p + f"attentions.{j}.", cout, None, spec)
        if i != n - 1:
            _conv(p + "downsamplers.0.conv.", cout, cout, 3, spec)
    c = boc[-1]
    _resnet("encoder.mid_block.resnets.0.", c, c, None, spec)
    _attention("encoder.mid_block.attentions.0.", c, None, spec)
    _resnet("encoder.mid_block.resnets.1.", c, c, None, spec)
    _vec("encoder.conv_norm_out.", c, spec)
    _conv("encoder.conv_out.", zc, c, 3, spec)
    _conv("quant_conv.", ed, zc, 1, spec)
    spec += [("quantize.embedding.weight", (cfg["num_vq_embeddings"], ed))]
    _conv("post_quant_conv.", zc, ed, 1, spec)
    _conv("decoder.conv_in.", c, zc, 3, spec)
    _resnet("decoder.mid_block.resnets.0.", c, c, zc, spec)
    _attention("decoder.mid_block.attentions.0.", c, zc, spec)
    _resnet("decoder.mid_block.resnets.1.", c, c, zc, spec)
    rev = boc[::-1]
    cout = rev[0]
    for i, kind in enumerate(cfg["up_block_types"]):
        cin, cout = cout, rev[i]
        p = f"decoder.up_blocks.{i}."
        for j in range(nl + 1):
            _resnet(p + f"resnets.{j}.", cin if j == 0 else cout, cout, zc, spec)
            if kind.startswith("Attn"):
                _attention(p + f"attentions.{j}.", cout, zc, spec)
        if i != n - 1:
            _conv(p + "upsamplers.0.conv.", cout, cout, 3, spec)
    _spatial("decoder.conv_norm_out.", boc[0], zc, spec)
    _conv("decoder.conv_out.", cfg["out_channels"], boc[0], 3, spec)
    return spec


def _norm(x, sd, p, zq):
    """GroupNorm(32, eps 1e-6) (zq None) or SpatialNorm: norm(f) * conv_y(zq') + conv_b(zq'), zq' nearest-resized to f."""
    if zq is None:
        return F.group_norm(x, 32, sd[p + "weight"], sd[p + "bias"], 1e-6)
    z = F.interpolate(zq, size=x.shape[-2:], mode="nearest")
    n = F.group_norm(x, 32, sd[p + "norm_layer.weight"], sd[p + "norm_layer.bias"], 1e-6)
    return n * F.conv2d(z, sd[p + "conv_y.weight"], sd[p + "conv_y.bias"]) + F.conv2d(z, sd[p + "conv_b.weight"], sd[p + "conv_b.bias"])


def _resnet_fwd(x, sd, p, zq):
    h = F.conv2d(F.silu(_norm(x, sd, p + "norm1.", zq)), sd[p + "conv1.weight"], sd[p + "conv1.bias"], padding=1)
    h = F.conv2d(F.silu(_norm(h, sd, p + "norm2.", zq)), sd[p + "conv2.weight"], sd[p + "conv2.bias"], padding=1)
    if p + "conv_shortcut.weight" in sd:
        x = F.conv2d(x, sd[p + "conv_shortcut.weight"], sd[p + "conv_shortcut.bias"])
    return x + h


def _attention_fwd(x, sd, p, zq):
    """Attention(heads=1, dim_head=C, residual_connection=True): tokens [B, HW, C], Linear projections, softmax(q k^T / sqrt C)."""
    h = _norm(x, sd, p + ("group_norm." if zq is None else "spatial_norm."), zq)
    B, C, H, W = h.shape
    t = h.reshape(B, C, H * W).transpose(1, 2)
    q, k, v = (F.linear(t, sd[p + f"to_{n}.weight"], sd[p + f"to_{n}.bias"]) for n in "qkv")
    a = torch.softmax(q @ k.transpose(1, 2) * C ** -0.5, dim=-1) @ v
    o = F.linear(a, sd[p + "to_out.0.weight"], sd[p + "to_out.0.bias"])
    return o.transpose(1, 2).reshape(B, C, H, W) + x


def vqmodel_encode(sd, cfg, x):
    """image [B, in_channels, H, W] -> VQModel.encode(x).latents [B, vq_embed_dim, H / 2^(n-1), ...], fp32."""
    n, nl = len(cfg["block_out_channels"]), cfg["layers_per_block"]
    h = F.conv2d(x, sd["encoder.conv_in.weight"], sd["encoder.conv_in.bias"], padding=1)
    for i, kind in enumerate(cfg["down_block_types"]):
        p = f"encoder.down_blocks.{i}."
        for j in range(nl):
            h = _resnet_fwd(h, sd, p + f"resnets.{j}.", None)
            if kind.startswith("Attn"):
                h = _attention_fwd(h, sd, p + f"attentions.{j}.", None)
        if i != n - 1:
            h = F.conv2d(F.pad(h, (0, 1, 0, 1)), sd[p + "downsamplers.0.conv.weight"], sd[p + "downsamplers.0.conv.bias"], stride=2)
    h = _resnet_fwd(h, sd, "encoder.mid_block.resnets.0.", None)
    h = _attention_fwd(h, sd, "encoder.mid_block.attentions.0.", None)
    h = _resnet_fwd(h, sd, "encoder.mid_block.resnets.1.", None)
    h = F.silu(_norm(h, sd, "encoder.conv_norm_out.", None))
    h = F.conv2d(h, sd["encoder.conv_out.weight"], sd["encoder.conv_out.bias"], padding=1)
    return F.conv2d(h, sd["quant_conv.weight"], sd["quant_conv.bias"])


def vqmodel_decode(sd, cfg, latents):
    """VQModel.decode(latents, force_not_quantize=True).sample: [B, vq_embed_dim, h, w] -> [B, out_channels, 2^(n-1) h, ...]."""
    n, nl = len(cfg["block_out_channels"]), cfg["layers_per_block"]
    zq = latents
    h = F.conv2d(latents, sd["post_quant_conv.weight"], sd["post_quant_conv.bias"])
    h = F.conv2d(h, sd["decoder.conv_in.weight"], sd["decoder.conv_in.bias"], padding=1)
    h = _resnet_fwd(h, sd, "decoder.mid_block.resnets.0.", zq)
    h = _attention_fwd(h, sd, "decoder.mid_block.attentions.0.", zq)
    h = _resnet_fwd(h, sd, "decoder.mid_block.resnets.1.", zq)
    for i, kind in enumerate(cfg["up_block_types"]):
        p = f"decoder.up_blocks.{i}."
        for j in range(nl + 1):
            h = _resnet_fwd(h, sd, p + f"resnets.{j}.", zq)
            if kind.startswith("Attn"):
                h = _attention_fwd(h, sd, p + f"attentions.{j}.", zq)
        if i != n - 1:
            h = F.interpolate(h, scale_factor=2.0, mode="nearest")
            h = F.conv2d(h, sd[p + "upsamplers.0.conv.weight"], sd[p + "upsamplers.0.conv.bias"], padding=1)
    h = F.silu(_norm(h, sd, "decoder.conv_norm_out.", zq))
    return F.conv2d(h, sd["decoder.conv_out.weight"], sd["decoder.conv_out.bias"], padding=1)
