"""TEST INFRASTRUCTURE (oracle): transformers' DPTForDepthEstimation with a plain ViT backbone (Intel/dpt-large, the default
model of the depth-estimation pipeline that builds the Kandinsky 2.2 ControlNet-depth hint), restated in torch from
transformers' key names, and the writer of the golden fixture tests/golden/dpt_tiny.pt:

    python -m tests.dpt_oracle

  dpt_spec / synth_weights  <- a DPTForDepthEstimation state dict of a config, synthetic (oracle/synth.py)
  forward                   <- DPTForDepthEstimation.forward: patch conv + CLS + (resized) position embedding, pre-LN ViT
                               layers (scaled-dot-product attention, exact GELU), the hidden states after
                               backbone_out_indices, the reassemble stage (readout "project", projection, ConvTranspose2d /
                               identity / stride-2 conv), the neck convs, the fusion stage, the depth head -> fp32 [B, S', S']
  dtype=torch.float16 runs the same ops on fp16 weights and activations, so it rounds where transformers' fp16 model does
  (the fp16 calibration of the GPU tests).

The fixture holds (with the transformers version that wrote it), for two tiny configs (an even 4 x 4 patch grid, and an odd
5 x 5 grid whose processor size differs from image_size, so the position embedding is resized and the fusion stage's
align_corners=False resize runs), transformers' processor output and predicted_depth on seeded images, and the
depth-estimation pipeline's predicted_depth and uint8 depth image of each image run alone. The writer
asserts that the oracle matches transformers within 1e-5 and kandinsky2's preprocess within 1e-6 before writing.  The GPU
tests read only the fixture."""
import os

import numpy as np
import torch
import torch.nn.functional as F

from oracle import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "dpt_tiny.pt")

# Intel/dpt-large's geometry (as its config.json is expected to read; nothing in the package relies on these numbers)
CFG_LARGE = dict(hidden_size=1024, num_hidden_layers=24, num_attention_heads=16, intermediate_size=4096, image_size=384,
                 patch_size=16, backbone_out_indices=[5, 11, 17, 23], neck_hidden_sizes=[256, 512, 1024, 1024],
                 fusion_hidden_size=256, layer_norm_eps=1e-12, reassemble_factors=[4, 2, 1, 0.5])
_TINY = dict(hidden_size=128, num_hidden_layers=4, num_attention_heads=2, intermediate_size=256, patch_size=16,
             backbone_out_indices=[0, 1, 2, 3], neck_hidden_sizes=[32, 64, 128, 128], fusion_hidden_size=64,
             layer_norm_eps=1e-12, reassemble_factors=[4, 2, 1, 0.5])
# (name, config, preprocessor config): the even grid at image_size, and an odd 5 x 5 grid from a 3 x 3 position embedding
TINY = (("even", dict(_TINY, image_size=64), dict(size={"height": 64, "width": 64}, resample=3)),
        ("odd", dict(_TINY, image_size=48), dict(size={"height": 80, "width": 80}, resample=2)))
IMAGES = (("landscape", "RGB", 97, 61), ("portrait", "RGB", 50, 83), ("rgba", "RGBA", 64, 64), ("gray", "L", 75, 70))
LAST_BIAS = 0.5   # head.head.4.bias: with synthetic weights most pre-ReLU outputs are then positive


def cfg_with_defaults(cfg):
    c = dict(layer_norm_eps=1e-12, readout_type="project")
    c.update(cfg)
    return c


def dpt_spec(cfg):
    """[(transformers name, shape)] of a plain-ViT DPTForDepthEstimation of the config."""
    H, P, F_, I = cfg["hidden_size"], cfg["patch_size"], cfg["fusion_hidden_size"], cfg["intermediate_size"]
    T = (cfg["image_size"] // P) ** 2 + 1
    spec = [("dpt.embeddings.cls_token", (1, 1, H)), ("dpt.embeddings.position_embeddings", (1, T, H)),
            ("dpt.embeddings.patch_embeddings.projection.weight", (H, 3, P, P)),
            ("dpt.embeddings.patch_embeddings.projection.bias", (H,)), ("dpt.layernorm.weight", (H,)),
            ("dpt.layernorm.bias", (H,))]
    for i in range(cfg["num_hidden_layers"]):
        p = f"dpt.encoder.layer.{i}."
        for n, shape in (("attention.attention.query", (H, H)), ("attention.attention.key", (H, H)),
                         ("attention.attention.value", (H, H)), ("attention.output.dense", (H, H)),
                         ("intermediate.dense", (I, H)), ("output.dense", (H, I))):
            spec += [(p + n + ".weight", shape), (p + n + ".bias", (shape[0],))]
        spec += [(p + n + s, (H,)) for n in ("layernorm_before", "layernorm_after") for s in (".weight", ".bias")]
    rs = "neck.reassemble_stage."
    for i, (C, f) in enumerate(zip(cfg["neck_hidden_sizes"], cfg["reassemble_factors"])):
        spec += [(f"{rs}readout_projects.{i}.0.weight", (H, 2 * H)), (f"{rs}readout_projects.{i}.0.bias", (H,)),
                 (f"{rs}layers.{i}.projection.weight", (C, H, 1, 1)), (f"{rs}layers.{i}.projection.bias", (C,))]
        if f != 1:
            k = int(f) if f > 1 else 3
            spec += [(f"{rs}layers.{i}.resize.weight", (C, C, k, k)), (f"{rs}layers.{i}.resize.bias", (C,))]
        spec.append((f"neck.convs.{i}.weight", (F_, C, 3, 3)))
    for j in range(len(cfg["neck_hidden_sizes"])):
        p = f"neck.fusion_stage.layers.{j}."
        spec += [(p + "projection.weight", (F_, F_, 1, 1)), (p + "projection.bias", (F_,))]
        for u in ("residual_layer1", "residual_layer2"):
            for cv in ("convolution1", "convolution2"):
                spec += [(f"{p}{u}.{cv}.weight", (F_, F_, 3, 3)), (f"{p}{u}.{cv}.bias", (F_,))]
    spec += [("head.head.0.weight", (F_ // 2, F_, 3, 3)), ("head.head.0.bias", (F_ // 2,)),
             ("head.head.2.weight", (32, F_ // 2, 3, 3)), ("head.head.2.bias", (32,)), ("head.head.4.weight", (1, 32, 1, 1)),
             ("head.head.4.bias", (1,))]
    return spec


def synth_weights(cfg, seed):
    """Synthetic transformers-named weights: oracle/synth.py, with a unit-normal CLS token, position embeddings at 0.1 scale,
    and the last bias at LAST_BIAS so that the final ReLU leaves a depth map that is not degenerate."""
    sd = synth.synth_state_dict(dpt_spec(cfg), seed=seed)
    g = torch.Generator().manual_seed(seed)
    sd["dpt.embeddings.cls_token"] = torch.randn(sd["dpt.embeddings.cls_token"].shape, generator=g)
    sd["dpt.embeddings.position_embeddings"] = 0.1 * torch.randn(sd["dpt.embeddings.position_embeddings"].shape, generator=g)
    sd["head.head.4.bias"] = torch.full((1,), LAST_BIAS)
    return sd


def _unit(x, sd, p, dtype):
    r = x
    x = F.conv2d(F.relu(x), sd[p + "convolution1.weight"].to(dtype), sd[p + "convolution1.bias"].to(dtype), padding=1)
    x = F.conv2d(F.relu(x), sd[p + "convolution2.weight"].to(dtype), sd[p + "convolution2.bias"].to(dtype), padding=1)
    return x + r


@torch.no_grad()
def forward(sd, cfg, pixels, dtype=torch.float32):
    """transformers names, pixel_values fp32 [B, 3, S, S] -> predicted_depth fp32 [B, S', S']."""
    c = cfg_with_defaults(cfg)
    w = lambda k: sd[k].to(dtype)  # noqa: E731
    H, P, heads = c["hidden_size"], c["patch_size"], c["num_attention_heads"]
    x = pixels.to(dtype)
    B, S = x.shape[0], x.shape[2]
    G = S // P
    emb = F.conv2d(x, w("dpt.embeddings.patch_embeddings.projection.weight"),
                   w("dpt.embeddings.patch_embeddings.projection.bias"), stride=P).flatten(2).transpose(1, 2)
    pos = w("dpt.embeddings.position_embeddings")
    g0 = int((pos.shape[1] - 1) ** 0.5)
    grid = F.interpolate(pos[0, 1:].reshape(1, g0, g0, -1).permute(0, 3, 1, 2), size=(G, G), mode="bilinear")
    pos = torch.cat([pos[:, :1], grid.permute(0, 2, 3, 1).reshape(1, G * G, -1)], 1)
    h = torch.cat([w("dpt.embeddings.cls_token").expand(B, -1, -1), emb], 1) + pos
    hidden = []
    for i in range(c["num_hidden_layers"]):
        p = f"dpt.encoder.layer.{i}."
        lin = lambda t, n: F.linear(t, w(p + n + ".weight"), w(p + n + ".bias"))  # noqa: E731
        y = F.layer_norm(h, (H,), w(p + "layernorm_before.weight"), w(p + "layernorm_before.bias"), c["layer_norm_eps"])
        q, k, v = (lin(y, "attention.attention." + n).reshape(B, -1, heads, H // heads).transpose(1, 2)
                   for n in ("query", "key", "value"))
        a = F.scaled_dot_product_attention(q, k, v).transpose(1, 2).reshape(B, -1, H)
        h = lin(a, "attention.output.dense") + h
        y = F.layer_norm(h, (H,), w(p + "layernorm_after.weight"), w(p + "layernorm_after.bias"), c["layer_norm_eps"])
        h = lin(F.gelu(lin(y, "intermediate.dense")), "output.dense") + h
        if i in c["backbone_out_indices"]:
            hidden.append(h)
    rs, feats = "neck.reassemble_stage.", []
    for i, (hs, f) in enumerate(zip(hidden, c["reassemble_factors"])):
        tok = hs[:, 1:]
        r = F.gelu(F.linear(torch.cat([tok, hs[:, :1].expand_as(tok)], -1), w(f"{rs}readout_projects.{i}.0.weight"),
                            w(f"{rs}readout_projects.{i}.0.bias")))
        r = r.permute(0, 2, 1).reshape(B, H, G, G)
        r = F.conv2d(r, w(f"{rs}layers.{i}.projection.weight"), w(f"{rs}layers.{i}.projection.bias"))
        if f > 1:
            r = F.conv_transpose2d(r, w(f"{rs}layers.{i}.resize.weight"), w(f"{rs}layers.{i}.resize.bias"), stride=int(f))
        elif f < 1:
            r = F.conv2d(r, w(f"{rs}layers.{i}.resize.weight"), w(f"{rs}layers.{i}.resize.bias"), stride=2, padding=1)
        feats.append(F.conv2d(r, w(f"neck.convs.{i}.weight"), padding=1))
    fused = None
    for j, fe in enumerate(feats[::-1]):
        p = f"neck.fusion_stage.layers.{j}."
        if fused is None:
            x = fe
        else:
            if fe.shape != fused.shape:
                fe = F.interpolate(fe, size=fused.shape[2:], mode="bilinear", align_corners=False)
            x = fused + _unit(fe, sd, p + "residual_layer1.", dtype)
        x = _unit(x, sd, p + "residual_layer2.", dtype)
        x = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)
        fused = F.conv2d(x, w(p + "projection.weight"), w(p + "projection.bias"))
    x = F.conv2d(fused, w("head.head.0.weight"), w("head.head.0.bias"), padding=1)
    x = F.interpolate(x, scale_factor=2, mode="bilinear", align_corners=True)
    x = F.relu(F.conv2d(x, w("head.head.2.weight"), w("head.head.2.bias"), padding=1))
    x = F.relu(F.conv2d(x, w("head.head.4.weight"), w("head.head.4.bias")))
    return x.squeeze(1).float()


def transformers_model(cfg, sd):
    from transformers import DPTConfig, DPTForDepthEstimation
    m = DPTForDepthEstimation(DPTConfig(**cfg)).eval()
    m.load_state_dict(sd, strict=True)
    return m


def transformers_processor(proc):
    from transformers.models.dpt.image_processing_pil_dpt import DPTImageProcessorPil
    return DPTImageProcessorPil(**proc)


def sample_images(seed=0):
    """[(name, PIL image)]: seeded noise over a smooth gradient, in the modes and sizes of IMAGES."""
    from PIL import Image
    rng = np.random.default_rng(seed)
    out = []
    for name, mode, w, h in IMAGES:
        yy, xx = np.mgrid[0:h, 0:w]
        base = np.stack([xx / w, yy / h, (xx + yy) / (w + h)], -1) * 200
        a = np.clip(base + rng.normal(0, 25, base.shape), 0, 255).astype(np.uint8)
        img = Image.fromarray(a, "RGB")
        if mode == "RGBA":
            img = img.convert("RGBA")
        elif mode == "L":
            img = img.convert("L")
        out.append((name, img))
    return out


def pipeline_depths(model, proc, images):
    """transformers' depth-estimation pipeline on the model -> (uint8 depth arrays, fp32 predicted_depth per image)."""
    from transformers import pipeline
    pipe = pipeline("depth-estimation", model=model, image_processor=transformers_processor(proc), device="cpu")
    outs = [pipe(img) for img in images]
    return [np.array(o["depth"]) for o in outs], [o["predicted_depth"].float() for o in outs]


def write_fixture():
    import transformers

    from kandinsky2.model.depth import preprocess_images, preprocessor_settings
    fx = dict(transformers_version=transformers.__version__, weight_seed=11, image_seed=0, configs={})
    images = sample_images(fx["image_seed"])
    for name, cfg, proc in TINY:
        sd = synth_weights(cfg, fx["weight_seed"])
        model = transformers_model(cfg, sd)
        tp = transformers_processor(proc)
        S = proc["size"]["height"]
        # RGB as the pipeline's load_image converts it
        pix = torch.cat([tp(img.convert("RGB"), return_tensors="pt")["pixel_values"] for _, img in images])
        ours = preprocess_images([img for _, img in images], preprocessor_settings(proc, cfg["image_size"]), S)
        perr = (ours - pix).abs().max().item()
        assert perr <= 1e-6, (name, perr)
        with torch.no_grad():
            ref = model(pixel_values=pix).predicted_depth
        mine = forward(sd, cfg, pix)
        rel = ((mine - ref).norm() / ref.norm()).item()
        assert rel <= 1e-5, (name, rel)
        pos = (ref > 0).float().mean().item()
        assert pos > 0.5, (name, pos)   # not a degenerate map
        u8, pred = pipeline_depths(model, proc, [img for _, img in images])
        fx["configs"][name] = dict(config=cfg, preprocessor=proc, pixel_values=pix, predicted_depth=ref,
                                   pipeline_predicted_depth=pred, depth_u8=[torch.from_numpy(a) for a in u8])
        print(f"{name}: preprocess max-abs {perr:.1e}, oracle rel-L2 {rel:.1e}, positive {pos:.3f}, depth {tuple(ref.shape)}")
    torch.save(fx, FIXTURE)
    print("wrote", FIXTURE)


if __name__ == "__main__":
    import sys
    sys.path.insert(0, os.path.join(ROOT, "kandinsky-2_b200"))
    write_fixture()
