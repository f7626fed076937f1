"""TEST INFRASTRUCTURE (oracle): the CLIP image tower of the Kandinsky 2.2 prior pipeline (transformers'
`CLIPVisionModelWithProjection`, which the reference builds at kandinsky2_2_model.py:24), restated from the math in torch, and
the writer of its golden fixture tests/golden/clip_vision_tiny.pt:

    python -m tests.clip_vision_oracle

  clip_vision_spec     <- the transformers state dict of a config (key names as transformers writes them)
  synth_weights        <- oracle/synth.py-style synthetic weights for it (the patch embedding scaled by fan_in^-1/2 like a
                          Linear weight)
  forward              <- CLIPVisionModelWithProjection.forward from transformers names: patch conv, CLS, position embedding,
                          pre_layrnorm, pre-LN encoder layers (eager attention, exact GELU), post_layernorm of the CLS row,
                          visual_projection.  dtype=torch.float16 rounds where transformers' fp16 model does (fp16 inputs to
                          every op, softmax in fp32 then rounded).
  forward_k2           <- the same network from kandinsky2's names (checkpoints.transformers_clip_vision_to_k2), fp32
  sample_images        <- the deterministic PIL images whose CLIPImageProcessor outputs the fixture pins

The fixture (77 KB) is written by running transformers (the PIL backend of CLIPImageProcessor, `CLIPImageProcessorPil`, which
resizes with PIL bicubic; transformers 5's default CLIPImageProcessor runs on torchvision instead) and asserts that the oracle
and kandinsky2's preprocess agree with it before writing."""
import math
import os

import numpy as np
import torch
import torch.nn.functional as F

from oracle import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "clip_vision_tiny.pt")

# ViT-bigG/14 as kandinsky-2-2-prior/image_encoder is expected to configure it (not checked against the real file)
CONFIG_BIGG = dict(hidden_size=1664, intermediate_size=8192, num_hidden_layers=48, num_attention_heads=16, image_size=224,
                   patch_size=14, projection_dim=1280, hidden_act="gelu", layer_norm_eps=1e-5, num_channels=3)
CONFIG_TINY = dict(hidden_size=208, intermediate_size=256, num_hidden_layers=2, num_attention_heads=2, image_size=56,
                   patch_size=14, projection_dim=32, hidden_act="gelu", layer_norm_eps=1e-5, num_channels=3)   # 17 tokens
CONFIG_TINY_26 = dict(CONFIG_TINY, image_size=70, num_hidden_layers=1)                                         # 26 tokens
IMAGES = (("landscape", "RGB", 320, 200), ("portrait", "RGB", 180, 300), ("small_square", "RGB", 100, 100),
          ("exact", "RGB", 224, 224), ("rgba", "RGBA", 250, 240), ("gray", "L", 230, 260))


def clip_vision_spec(cfg):
    H, I, P = cfg["hidden_size"], cfg["intermediate_size"], cfg["patch_size"]
    T = (cfg["image_size"] // P) ** 2 + 1
    p = "vision_model."
    spec = [(p + "embeddings.class_embedding", (H,)), (p + "embeddings.patch_embedding.weight", (H, 3, P, P)),
            (p + "embeddings.position_embedding.weight", (T, H)), (p + "pre_layrnorm.weight", (H,)),
            (p + "pre_layrnorm.bias", (H,))]
    for i in range(cfg["num_hidden_layers"]):
        lp = f"{p}encoder.layers.{i}."
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            spec += [(f"{lp}self_attn.{n}.weight", (H, H)), (f"{lp}self_attn.{n}.bias", (H,))]
        spec += [(lp + "layer_norm1.weight", (H,)), (lp + "layer_norm1.bias", (H,)), (lp + "mlp.fc1.weight", (I, H)),
                 (lp + "mlp.fc1.bias", (I,)), (lp + "mlp.fc2.weight", (H, I)), (lp + "mlp.fc2.bias", (H,)),
                 (lp + "layer_norm2.weight", (H,)), (lp + "layer_norm2.bias", (H,))]
    return spec + [(p + "post_layernorm.weight", (H,)), (p + "post_layernorm.bias", (H,)),
                   ("visual_projection.weight", (cfg["projection_dim"], H))]


def synth_weights(cfg, seed):
    sd = synth.synth_state_dict(clip_vision_spec(cfg), seed=seed)
    k = "vision_model.embeddings.patch_embedding.weight"
    sd[k] = sd[k] / math.sqrt(sd[k][0].numel())
    return sd


def _attention(q, k, v, heads, dtype):
    B, T, H = q.shape
    d = H // heads
    q, k, v = (t.view(B, T, heads, d).transpose(1, 2) for t in (q, k, v))
    w = torch.matmul(q, k.transpose(-1, -2)) * d ** -0.5
    w = torch.softmax(w, dim=-1, dtype=torch.float32).to(dtype)
    return torch.matmul(w, v).transpose(1, 2).reshape(B, T, H)


def _tower(emb, layers, post, proj, cfg, dtype):
    """emb [B, T, H] (after the position embedding); layers: per layer (ln1, (wq, bq), (wk, bk), (wv, bv), (wo, bo), ln2, fc1,
    fc2) with ln = (weight, bias) -> (last_hidden_state, image_embeds), fp32."""
    H, eps, heads = cfg["hidden_size"], cfg["layer_norm_eps"], cfg["num_attention_heads"]
    h = emb
    for ln1, q, k, v, o, ln2, fc1, fc2 in layers:
        y = F.layer_norm(h, (H,), *ln1, eps=eps)
        a = _attention(F.linear(y, *q), F.linear(y, *k), F.linear(y, *v), heads, dtype)
        h = h + F.linear(a, *o)
        y = F.layer_norm(h, (H,), *ln2, eps=eps)
        h = h + F.linear(F.gelu(F.linear(y, *fc1)), *fc2)
    pooled = F.layer_norm(h[:, 0], (H,), *post, eps=eps)
    return h.float(), F.linear(pooled, proj).float()


def _embed(pixel_values, w_patch, cls, pos, dtype):
    x = F.conv2d(pixel_values.to(dtype), w_patch, stride=w_patch.shape[-1]).flatten(2).transpose(1, 2)
    return torch.cat([cls.expand(x.shape[0], 1, -1), x], dim=1) + pos[None]


def forward(sd, cfg, pixel_values, dtype=torch.float32):
    """transformers names -> (last_hidden_state [B, T, H], image_embeds [B, projection_dim]), both fp32."""
    sd = {k: v.to(dtype) for k, v in sd.items()}
    p = "vision_model."
    g = lambda n: (sd[n + ".weight"], sd[n + ".bias"])  # noqa: E731
    emb = _embed(pixel_values, sd[p + "embeddings.patch_embedding.weight"], sd[p + "embeddings.class_embedding"],
                 sd[p + "embeddings.position_embedding.weight"], dtype)
    emb = F.layer_norm(emb, (cfg["hidden_size"],), *g(p + "pre_layrnorm"), eps=cfg["layer_norm_eps"])
    layers = []
    for i in range(cfg["num_hidden_layers"]):
        lp = f"{p}encoder.layers.{i}."
        layers.append((g(lp + "layer_norm1"), g(lp + "self_attn.q_proj"), g(lp + "self_attn.k_proj"), g(lp + "self_attn.v_proj"),
                       g(lp + "self_attn.out_proj"), g(lp + "layer_norm2"), g(lp + "mlp.fc1"), g(lp + "mlp.fc2")))
    return _tower(emb, layers, g(p + "post_layernorm"), sd["visual_projection.weight"], cfg, dtype)


def forward_k2(sd, cfg, pixel_values):
    """kandinsky2 names (attn.qkv packed per head [q_h | k_h | v_h]) -> the same outputs as forward, fp32."""
    H, heads = cfg["hidden_size"], cfg["num_attention_heads"]
    d = H // heads
    g = lambda n: (sd[n + ".weight"].float(), sd[n + ".bias"].float())  # noqa: E731
    emb = _embed(pixel_values, sd["patch_embedding.weight"].float(), sd["class_embedding"].float(),
                 sd["position_embedding"].float(), torch.float32)
    emb = F.layer_norm(emb, (H,), *g("pre_ln"), eps=cfg["layer_norm_eps"])
    layers = []
    for i in range(cfg["num_hidden_layers"]):
        w, b = g(f"layers.{i}.attn.qkv")
        wq, wk, wv = (w.view(heads, 3, d, H)[:, j].reshape(H, H) for j in range(3))
        bq, bk, bv = (b.view(heads, 3, d)[:, j].reshape(H) for j in range(3))
        p = f"layers.{i}."
        layers.append((g(p + "ln_1"), (wq, bq), (wk, bk), (wv, bv), g(p + "attn.proj"), g(p + "ln_2"), g(p + "mlp.fc1"),
                       g(p + "mlp.fc2")))
    return _tower(emb, layers, g("post_ln"), sd["proj.weight"].float(), cfg, torch.float32)


def sample_images():
    """[(name, PIL image)]: deterministic noise with a smooth gradient, in the modes and sizes of IMAGES."""
    from PIL import Image
    out = []
    for i, (name, mode, w, h) in enumerate(IMAGES):
        rng = np.random.default_rng(100 + i)
        ch = {"RGB": 3, "RGBA": 4, "L": 1}[mode]
        yy, xx = np.mgrid[0:h, 0:w]
        base = (127 + 100 * np.sin(xx / 17.0 + i) * np.cos(yy / 23.0))[..., None]
        a = np.clip(base + rng.normal(0, 30, (h, w, ch)), 0, 255).astype(np.uint8)
        out.append((name, Image.fromarray(a[..., 0] if ch == 1 else a, mode)))
    return out


def transformers_outputs(sd, cfg, pixel_values):
    """transformers' own CLIPVisionModelWithProjection (eager attention, fp32) on sd."""
    from transformers import CLIPVisionConfig, CLIPVisionModelWithProjection
    model = CLIPVisionModelWithProjection(CLIPVisionConfig(**cfg, attn_implementation="eager")).eval()
    model.load_state_dict(sd, strict=True)
    with torch.no_grad():
        o = model(pixel_values=pixel_values)
    return o.last_hidden_state.float(), o.image_embeds.float()


def transformers_preprocess(img):
    """transformers' CLIPImageProcessorPil with its defaults -> (uint8 center crop [3, 224, 224], pixel_values [3, 224, 224])."""
    from transformers.models.clip.image_processing_pil_clip import CLIPImageProcessorPil
    proc = CLIPImageProcessorPil()
    pv = torch.from_numpy(np.asarray(proc(images=img, return_tensors="np")["pixel_values"][0])).float()
    crop = CLIPImageProcessorPil(do_rescale=False, do_normalize=False)(images=img, return_tensors="np")["pixel_values"][0]
    return torch.from_numpy(np.asarray(crop).round().astype(np.uint8)), pv


def sha256(t):
    """Hex SHA-256 of a CPU tensor's bytes (C order)."""
    import hashlib
    return hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()


def _pixels(batch, size, seed):
    return torch.randn(batch, 3, size, size, generator=torch.Generator().manual_seed(seed))


def tower_pixels(t):
    """The pixel_values of a fixture tower entry, regenerated from its seed (CPU generator) and checked against the stored
    digest, so the fixture need not hold them."""
    pix = _pixels(t["batch"], t["cfg"]["image_size"], t["pixel_seed"])
    assert sha256(pix) == t["pixel_sha256"], "torch.randn no longer reproduces the fixture's pixel_values"
    return pix


def write_fixture():
    """The fixture holds what cannot be regenerated: transformers' outputs, and per image the SHA-256 of the uint8 center crop,
    its first row and the first row of the normalised values.  Weights and pixel values are regenerated from their seeds
    (pixel values checked by digest); keeping the crops themselves would make the file 1.1 MB."""
    import transformers

    from kandinsky2.model.clip_vision import preprocess_images
    towers = []
    for n, cfg in enumerate((CONFIG_TINY, CONFIG_TINY_26)):
        wseed, pseed, batch = 3 + n, 40 + n, 2 - n
        sd = synth_weights(cfg, wseed)
        pix = _pixels(batch, cfg["image_size"], pseed)
        hid, emb = transformers_outputs(sd, cfg, pix)
        ohid, oemb = forward(sd, cfg, pix)
        rel = max(((ohid - hid).norm() / hid.norm()).item(), ((oemb - emb).norm() / emb.norm()).item())
        assert rel <= 1e-5, f"oracle deviates from transformers by rel {rel}"
        towers.append(dict(cfg=cfg, weight_seed=wseed, pixel_seed=pseed, batch=batch, pixel_sha256=sha256(pix),
                           last_hidden_state=hid, image_embeds=emb))
    crop_sha, crop_rows, rows = {}, {}, {}
    for name, img in sample_images():
        crop, pv = transformers_preprocess(img)
        mine = preprocess_images(img)[0]
        assert (mine - pv).abs().max().item() <= 1e-6, name
        crop_sha[name] = sha256(crop)
        crop_rows[name] = crop[:, :1].clone()
        rows[name] = pv[:, :1].clone()
    torch.save(dict(transformers_version=transformers.__version__, towers=towers, crop_sha256=crop_sha, crop_rows=crop_rows,
                    normalised_rows=rows), FIXTURE)
    print(f"wrote {FIXTURE} (transformers {transformers.__version__}, {os.path.getsize(FIXTURE)} bytes)")


if __name__ == "__main__":
    import sys
    sys.path.insert(0, os.path.join(ROOT, "kandinsky-2_b200"))
    write_fixture()
