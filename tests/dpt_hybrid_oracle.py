"""TEST INFRASTRUCTURE (oracle): transformers' DPTForDepthEstimation with the hybrid backbone (MiDaS v3 DPT-Hybrid, a BiT
ResNet-50 in front of ViT-B/16; Intel/dpt-hybrid-midas, the estimator of ControlNet's MidasDetector), restated in torch from
transformers' key names, and the writer of the golden fixture tests/golden/dpt_hybrid_tiny.pt:

    python -m tests.dpt_hybrid_oracle

  forward   <- the BiT stem (weight-standardised 7x7 stride-2 conv with TF-SAME padding, GroupNorm + ReLU, 3x3 stride-2 max
               pool padded with 0), the bottleneck stages (stride 2 with TF-SAME padding in the first block of stages 2 and
               3), the 1x1 token projection + CLS + resized position embedding, the ViT layers, and the neck (stages 0 / 1 take
               the BiT maps, 2 / 3 the hidden states after backbone_out_indices[2:]), fusion and head of tests/dpt_oracle.py
               on a gh x gw patch grid.  dtype=torch.float16 runs the same ops on fp16 weights and activations (the fp16
               calibration of the GPU tests).

The fixture (transformers 5.5.0) holds a tiny model with the real BiT widths (64-channel stem, stages 256 / 512 / 1024, 32
groups) and depths [1, 2, 1] and a 128-wide, 2-head, 4-layer ViT (image_size 64), at four input sizes: 64 x 64 through
DPTForDepthEstimation.forward, and 128 x 128, 64 x 96 and 80 x 80 (an odd 5 x 5 grid) through transformers' own modules
composed as forward composes them (embeddings with interpolate_pos_encoding, the layers, neck(hidden, gh, gw), head) --
forward itself accepts only image_size and reshapes the tokens to a square.  It stores, per size, the seed of the pixel
values (fixture_pixels regenerates them), predicted_depth and the per-channel means of the BiT stage maps, and the full
stage maps (fp16) at 64 x 64.  The writer asserts that the composition equals forward at 64 x 64 and that the oracle
matches transformers within 1e-5 before writing."""
import os

import torch
import torch.nn.functional as F

from oracle import synth
from tests import dpt_oracle as do

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "dpt_hybrid_tiny.pt")

_BIT = dict(model_type="bit", layer_type="bottleneck", global_padding="same", embedding_dynamic_padding=True,
            out_features=["stage1", "stage2", "stage3"], hidden_sizes=[256, 512, 1024, 2048], embedding_size=64,
            num_groups=32, hidden_act="relu")
# Intel/dpt-hybrid-midas's geometry (as its config.json is expected to read; nothing in the package relies on these numbers)
CFG_HYBRID = dict(is_hybrid=True, hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072,
                  image_size=384, patch_size=16, backbone_out_indices=[2, 5, 8, 11], neck_hidden_sizes=[256, 512, 768, 768],
                  reassemble_factors=[1, 1, 1, 0.5], fusion_hidden_size=256, readout_type="project",
                  backbone_featmap_shape=[1, 1024, 24, 24], neck_ignore_stages=[0, 1],
                  backbone_config=dict(_BIT, depths=[3, 4, 9]))
CFG_TINY = dict(CFG_HYBRID, hidden_size=128, num_hidden_layers=4, num_attention_heads=2, intermediate_size=256, image_size=64,
                backbone_out_indices=[0, 1, 2, 3], neck_hidden_sizes=[256, 512, 128, 128], fusion_hidden_size=64,
                backbone_featmap_shape=[1, 1024, 4, 4], backbone_config=dict(_BIT, depths=[1, 2, 1]))
SIZES = ((64, 64), (128, 128), (64, 96), (80, 80))   # the first through forward, the rest composed
BIT = "dpt.embeddings.backbone.bit."
# head.head.4.bias of the synthetic weights at the Intel/dpt-hybrid-midas geometry: there the last convolution's output before
# the bias has median -8.3 and spread 2.3 (384 x 384, seed 31), so that 12 leaves a depth map that is positive almost everywhere
REAL_LAST_BIAS = 12.0


def transformers_model(cfg, sd=None):
    from transformers import DPTConfig, DPTForDepthEstimation
    m = DPTForDepthEstimation(DPTConfig(**cfg)).eval()
    if sd is not None:
        m.load_state_dict(sd, strict=True)
    return m


def hybrid_spec(cfg):
    """[(transformers name, shape)] of a hybrid DPTForDepthEstimation of the config (read off transformers' model)."""
    return [(k, tuple(v.shape)) for k, v in transformers_model(cfg).state_dict().items()]


def spec_from_config(cfg):
    """The same spec without transformers: the plain DPT's ViT / neck / head names with the hybrid's embeddings, BiT and
    neck stages; used where transformers is not installed."""
    from kandinsky2.checkpoints import transformers_dpt_hybrid_keys
    from kandinsky2.model.depth import _bit_layer_shapes, dpt_hybrid_config, k2_hybrid_shapes
    c = dpt_hybrid_config(cfg)
    shapes = {k: s for k, s in do.dpt_spec(dict(cfg, is_hybrid=False))}
    shapes.update({BIT[:-4] + k: s for k, s in _bit_layer_shapes(c["bit"]).items()})
    shapes.update({k: s for k, s in k2_hybrid_shapes(c).items() if k.startswith(("neck.", "head."))})
    H = c["hidden_size"]
    shapes.update({"dpt.embeddings.projection.weight": (H, c["bit"]["channels"][2], 1, 1),
                   "dpt.embeddings.projection.bias": (H,)})
    return [(k, shapes[k]) for k in transformers_dpt_hybrid_keys(cfg)]


def synth_weights(cfg, seed, spec=None, last_bias=do.LAST_BIAS):
    """Synthetic transformers-named weights: oracle/synth.py, BiT GroupNorm gamma 1 + 0.1 N(0, 1) and beta 0.1 N(0, 1), a
    unit-normal CLS token, position embeddings at 0.1 scale, and the last bias at last_bias."""
    sd = synth.synth_state_dict(spec if spec is not None else spec_from_config(cfg), seed=seed)
    g = torch.Generator().manual_seed(seed)
    for k in sorted(sd):
        if k.startswith(BIT) and ".norm" in k:
            sd[k] = (1.0 if k.endswith("weight") else 0.0) + 0.1 * torch.randn(sd[k].shape, generator=g)
    sd["dpt.embeddings.cls_token"] = torch.randn(sd["dpt.embeddings.cls_token"].shape, generator=g)
    sd["dpt.embeddings.position_embeddings"] = 0.1 * torch.randn(sd["dpt.embeddings.position_embeddings"].shape, generator=g)
    sd["head.head.4.bias"] = torch.full((1,), float(last_bias))
    return sd


def _pad_same(x, k, s, value=0.0):
    """DynamicPad2d: TF-SAME padding of x for a k x k stride-s window."""
    def pad(n):
        return max((-(-n // s) - 1) * s + k - n, 0)
    ph, pw = pad(x.shape[2]), pad(x.shape[3])
    return F.pad(x, [pw // 2, pw - pw // 2, ph // 2, ph - ph // 2], value=value) if ph or pw else x


def standardized(w):
    """WeightStandardizedConv2d's weight, as transformers computes it (batch_norm over [1, Cout, in * kh * kw], eps 1e-8)."""
    return F.batch_norm(w.reshape(1, w.shape[0], -1), None, None, training=True, momentum=0.0, eps=1e-8).reshape_as(w)


def _conv_ws(x, w, k, stride):
    if stride == 1:
        return F.conv2d(x, standardized(w), padding=(k - 1) // 2)
    return F.conv2d(_pad_same(x, k, stride), standardized(w), stride=stride)


@torch.no_grad()
def bit_forward(sd, cfg, x, dtype=torch.float32):
    """The BiT backbone -> [stage-1, stage-2, stage-3 map] (NCHW, dtype)."""
    w = lambda k: sd[BIT + k].to(x.device, dtype)  # noqa: E731
    gn = lambda t, n: F.group_norm(t, 32, w(n + ".weight"), w(n + ".bias"), 1e-5)  # noqa: E731
    x = F.relu(gn(_conv_ws(x.to(dtype), w("embedder.convolution.weight"), 7, 2), "embedder.norm"))
    x = F.max_pool2d(_pad_same(x, 3, 2, 0.0), 3, 2)
    maps = []
    for s, depth in enumerate(cfg["backbone_config"]["depths"]):
        for l in range(depth):
            p, stride = f"encoder.stages.{s}.layers.{l}.", 2 if s > 0 and l == 0 else 1
            short = gn(_conv_ws(x, w(p + "downsample.conv.weight"), 1, stride), p + "downsample.norm") if l == 0 else x
            h = F.relu(gn(_conv_ws(x, w(p + "conv1.weight"), 1, 1), p + "norm1"))
            h = F.relu(gn(_conv_ws(h, w(p + "conv2.weight"), 3, stride), p + "norm2"))
            x = F.relu(gn(_conv_ws(h, w(p + "conv3.weight"), 1, 1), p + "norm3") + short)
        maps.append(x)
    return maps


@torch.no_grad()
def forward(sd, cfg, pixels, dtype=torch.float32, with_maps=False):
    """transformers names, pixel_values fp32 [B, 3, h, w] (multiples of 16) -> predicted_depth fp32 [B, h', w'] (and the BiT
    maps with with_maps)."""
    c = do.cfg_with_defaults(cfg)
    dev = pixels.device
    w = lambda k: sd[k].to(dev, dtype)  # noqa: E731
    H, heads = c["hidden_size"], c["num_attention_heads"]
    B, gh, gw = pixels.shape[0], pixels.shape[2] // 16, pixels.shape[3] // 16
    maps = bit_forward(sd, c, pixels, dtype)
    emb = F.conv2d(maps[2], w("dpt.embeddings.projection.weight"), w("dpt.embeddings.projection.bias")).flatten(2)
    pos = w("dpt.embeddings.position_embeddings")
    g0 = int((pos.shape[1] - 1) ** 0.5)
    grid = F.interpolate(pos[0, 1:].reshape(1, g0, g0, -1).permute(0, 3, 1, 2), size=(gh, gw), mode="bilinear")
    pos = torch.cat([pos[:, :1], grid.permute(0, 2, 3, 1).reshape(1, gh * gw, -1)], 1)
    h = torch.cat([w("dpt.embeddings.cls_token").expand(B, -1, -1), emb.transpose(1, 2)], 1) + pos
    hidden = []
    for i in range(c["backbone_out_indices"][-1] + 1):
        p = f"dpt.encoder.layer.{i}."
        lin = lambda t, n: F.linear(t, w(p + n + ".weight"), w(p + n + ".bias"))  # noqa: E731
        y = F.layer_norm(h, (H,), w(p + "layernorm_before.weight"), w(p + "layernorm_before.bias"), c["layer_norm_eps"])
        q, k, v = (lin(y, "attention.attention." + n).reshape(B, -1, heads, H // heads).transpose(1, 2)
                   for n in ("query", "key", "value"))
        a = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, -1, H)
        h = lin(a, "attention.output.dense") + h
        y = F.layer_norm(h, (H,), w(p + "layernorm_after.weight"), w(p + "layernorm_after.bias"), c["layer_norm_eps"])
        h = lin(F.gelu(lin(y, "intermediate.dense")), "output.dense") + h
        if i in c["backbone_out_indices"][2:]:
            hidden.append(h)
    rs = "neck.reassemble_stage."
    feats = [F.conv2d(maps[i], w(f"neck.convs.{i}.weight"), padding=1) for i in (0, 1)]
    for i, hs in zip((2, 3), hidden):
        tok = hs[:, 1:]
        r = F.gelu(F.linear(torch.cat([tok, hs[:, :1].expand_as(tok)], -1), w(f"{rs}readout_projects.{i}.0.weight"),
                            w(f"{rs}readout_projects.{i}.0.bias")))
        r = r.permute(0, 2, 1).reshape(B, H, gh, gw)
        r = F.conv2d(r, w(f"{rs}layers.{i}.projection.weight"), w(f"{rs}layers.{i}.projection.bias"))
        f = c["reassemble_factors"][i]
        if f > 1:
            r = F.conv_transpose2d(r, w(f"{rs}layers.{i}.resize.weight"), w(f"{rs}layers.{i}.resize.bias"), stride=int(f))
        elif f < 1:
            r = F.conv2d(r, w(f"{rs}layers.{i}.resize.weight"), w(f"{rs}layers.{i}.resize.bias"), stride=2, padding=1)
        feats.append(F.conv2d(r, w(f"neck.convs.{i}.weight"), padding=1))
    sdd = {k: v.to(dev) for k, v in sd.items() if k.startswith("neck.fusion_stage.")}
    fused = None
    for j, fe in enumerate(feats[::-1]):
        p = f"neck.fusion_stage.layers.{j}."
        if fused is None:
            x = fe
        else:
            if fe.shape != fused.shape:
                fe = F.interpolate(fe, size=fused.shape[2:], mode="bilinear", align_corners=False)
            x = fused + do._unit(fe, sdd, p + "residual_layer1.", dtype)
        x = do._unit(x, sdd, p + "residual_layer2.", dtype)
        x = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)
        fused = F.conv2d(x, w(p + "projection.weight"), w(p + "projection.bias"))
    x = F.conv2d(fused, w("head.head.0.weight"), w("head.head.0.bias"), padding=1)
    x = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)
    x = F.relu(F.conv2d(x, w("head.head.2.weight"), w("head.head.2.bias"), padding=1))
    x = F.relu(F.conv2d(x, w("head.head.4.weight"), w("head.head.4.bias")))
    out = x.squeeze(1).float()
    return (out, [m.float() for m in maps]) if with_maps else out


@torch.no_grad()
def transformers_compose(model, pix):
    """DPTForDepthEstimation.forward composed from transformers' own modules at any size that is a multiple of 16: the
    embeddings with interpolate_pos_encoding, the layers one by one, the neck with the real patch grid, the head."""
    cfg = model.config
    gh, gw = pix.shape[2] // 16, pix.shape[3] // 16
    eo = model.dpt.embeddings(pix, interpolate_pos_encoding=True)
    h, hidden = eo.last_hidden_states, list(eo.intermediate_activations)
    for i, layer in enumerate(model.dpt.encoder.layer):
        h = layer(h)
        h = h[0] if isinstance(h, tuple) else h
        if i in cfg.backbone_out_indices[2:]:
            hidden.append(h)
    return model.head(model.neck(hidden, gh, gw)), list(eo.intermediate_activations)


def sample_pixels(h, w, seed, B=1):
    """Seeded pixel values in [-1, 1]: a smooth gradient plus noise."""
    g = torch.Generator().manual_seed(seed)
    yy, xx = torch.meshgrid(torch.linspace(-1, 1, h), torch.linspace(-1, 1, w), indexing="ij")
    base = torch.stack([xx, yy, xx * yy])[None].expand(B, -1, -1, -1)
    return (0.6 * base + 0.3 * torch.randn(B, 3, h, w, generator=g)).clamp(-1, 1).contiguous()


def fixture_pixels(g):
    """The pixel values of one fixture size, regenerated from its seed (sample_pixels; torch's CPU generator) and checked
    against the float64 sum the writer recorded."""
    pix = sample_pixels(*g["size"], seed=g["pixel_seed"])
    assert abs(pix.double().sum().item() - g["pixel_sum"]) <= 1e-9 * pix.numel(), "sample_pixels no longer reproduces"
    return pix


def write_fixture():
    """Per size: the pixel seed (and the float64 sum of the pixels), transformers' predicted_depth and the per-channel means
    of the three BiT stage maps; the full stage maps, rounded to fp16, at the native size only (they are most of the bytes)."""
    import transformers
    fx = dict(transformers_version=transformers.__version__, weight_seed=5, config=CFG_TINY, sizes={})
    spec = hybrid_spec(CFG_TINY)
    assert sorted(k for k, _ in spec) == sorted(k for k, _ in spec_from_config(CFG_TINY))
    sd = synth_weights(CFG_TINY, fx["weight_seed"], spec)
    model = transformers_model(CFG_TINY, sd)
    for n, (h, w) in enumerate(SIZES):
        pix = sample_pixels(h, w, seed=100 + n)
        ref, maps = transformers_compose(model, pix)
        native = (h, w) == (CFG_TINY["image_size"],) * 2
        if native:
            with torch.no_grad():
                fwd = model(pixel_values=pix).predicted_depth
            assert torch.equal(fwd, ref), "the composition differs from forward at the native size"
            ref = fwd
        mine, my_maps = forward(sd, CFG_TINY, pix, with_maps=True)
        rel = ((mine - ref).norm() / ref.norm()).item()
        assert rel <= 1e-5, ((h, w), rel)
        for a, b in zip(my_maps, maps):
            assert ((a - b).norm() / b.norm()).item() <= 1e-5
        pos = (ref > 0).float().mean().item()
        assert pos > 0.5, ((h, w), pos)
        g = dict(size=(h, w), pixel_seed=100 + n, pixel_sum=pix.double().sum().item(), predicted_depth=ref.clone(),
                 bit_channel_means=[m.mean((0, 2, 3)).clone() for m in maps])
        if native:
            g["bit_maps"] = [m.half() for m in maps]   # rounded to fp16: enough to localise a mismatch
        fx["sizes"][(h, w)] = g
        print(f"{h} x {w}: oracle rel-L2 {rel:.1e}, positive {pos:.3f}, depth {tuple(ref.shape)}")
    torch.save(fx, FIXTURE)
    print("wrote", FIXTURE, os.path.getsize(FIXTURE), "bytes")


if __name__ == "__main__":
    import sys
    sys.path.insert(0, os.path.join(ROOT, "kandinsky-2_b200"))
    write_fixture()
