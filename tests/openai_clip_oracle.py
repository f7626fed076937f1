"""TEST INFRASTRUCTURE (oracle): OpenAI CLIP (ViT), the Kandinsky 2.1 prior pipeline's ViT-L/14 (`clip.load` in
kandinsky2_1_model.py:64-67), restated from the math in torch from the OpenAI names (clip/model.py), the `clip` image
transform, and the writer of the golden fixture tests/golden/openai_clip_tiny.pt:

    python -m tests.openai_clip_oracle

  openai_spec / synth_weights  <- an OpenAI CLIP state dict of a geometry, synthetic (oracle/synth.py)
  text_forward                 <- generate_clip_emb's tower lines (kandinsky2_1_model.py:159-166): token + positional
                                  embedding, pre-LN resblocks (causal mask, QuickGELU), ln_final, the argmax row @ text_projection
  vision_forward               <- VisionTransformer.forward: conv1, class embedding, positional embedding, ln_pre, resblocks,
                                  ln_post of the CLS row @ proj
  dtype=torch.float16 rounds where the fp16 model does: fp16 weights (LayerNorm parameters stay fp32, as clip's
  convert_weights leaves them) and fp16 activations, LayerNorm in fp32, softmax in fp32 then rounded to fp16.
  text_forward_k2 / vision_forward_k2 <- the same network from kandinsky2's names (checkpoints.openai_clip_to_k2), fp32
  clip_transform               <- torchvision's Compose of clip's _transform (the fixture's preprocessing reference)

The fixture is written with transformers' CLIPModel (hidden_act="quick_gelu", eos_token_id=2: the argmax pooling) on the
synthetic weights converted to transformers names, and torchvision; the writer asserts that the oracle matches transformers
(rel <= 1e-5) and that kandinsky2's preprocess_openai matches torchvision bit for bit before writing.  The GPU tests read only
the fixture."""
import hashlib
import math
import os

import numpy as np
import torch
import torch.nn.functional as F

from oracle import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "openai_clip_tiny.pt")
MEAN = (0.48145466, 0.4578275, 0.40821073)
STD = (0.26862954, 0.26130258, 0.27577711)

# ViT-L/14 as clip's build_model reads it from ViT-L-14.pt
GEO_L14 = dict(text_width=768, text_layers=12, context=77, vocab=49408, embed_dim=768, vision_width=1024, vision_layers=24,
               patch=14, image_size=224)
GEO_TINY = dict(text_width=128, text_layers=2, context=16, vocab=1000, embed_dim=96, vision_width=128, vision_layers=2,
                patch=14, image_size=56)
IMAGES = (("landscape_odd", "RGB", 321, 200), ("portrait_odd", "RGB", 181, 300), ("small", "RGB", 100, 97),
          ("exact", "RGB", 224, 224), ("rgba", "RGBA", 251, 240), ("gray", "L", 230, 263))


def openai_spec(geo):
    """[(OpenAI name, shape)] of a ViT CLIP of the geometry (without logit_scale and build_model's deleted entries)."""
    tw, vw, P = geo["text_width"], geo["vision_width"], geo["patch"]
    T = (geo["image_size"] // P) ** 2 + 1
    spec = [("positional_embedding", (geo["context"], tw)), ("text_projection", (tw, geo["embed_dim"])),
            ("token_embedding.weight", (geo["vocab"], tw)), ("ln_final.weight", (tw,)), ("ln_final.bias", (tw,)),
            ("visual.class_embedding", (vw,)), ("visual.positional_embedding", (T, vw)), ("visual.proj", (vw, geo["embed_dim"])),
            ("visual.conv1.weight", (vw, 3, P, P)), ("visual.ln_pre.weight", (vw,)), ("visual.ln_pre.bias", (vw,)),
            ("visual.ln_post.weight", (vw,)), ("visual.ln_post.bias", (vw,))]
    for prefix, W, L in (("transformer.", tw, geo["text_layers"]), ("visual.transformer.", vw, geo["vision_layers"])):
        for i in range(L):
            lp = f"{prefix}resblocks.{i}."
            spec += [(lp + "attn.in_proj_weight", (3 * W, W)), (lp + "attn.in_proj_bias", (3 * W,)),
                     (lp + "attn.out_proj.weight", (W, W)), (lp + "attn.out_proj.bias", (W,)), (lp + "ln_1.weight", (W,)),
                     (lp + "ln_1.bias", (W,)), (lp + "mlp.c_fc.weight", (4 * W, W)), (lp + "mlp.c_fc.bias", (4 * W,)),
                     (lp + "mlp.c_proj.weight", (W, 4 * W)), (lp + "mlp.c_proj.bias", (W,)), (lp + "ln_2.weight", (W,)),
                     (lp + "ln_2.bias", (W,))]
    return spec


def synth_weights(geo, seed):
    """Synthetic OpenAI-named weights: oracle/synth.py, with the positional embeddings at 0.1 scale, the class embedding a
    unit normal, and the projections (applied as x @ P) scaled by their fan-in, rows."""
    sd = synth.synth_state_dict(openai_spec(geo), seed=seed)
    for k in ("text_projection", "visual.proj"):
        sd[k] = sd[k] * math.sqrt(sd[k].shape[1] / sd[k].shape[0])
    for k in ("positional_embedding", "visual.positional_embedding"):
        sd[k] = 0.1 * sd[k] * math.sqrt(sd[k].shape[1])
    sd["visual.class_embedding"] = sd["visual.class_embedding"] - 1.0
    return sd


def quick_gelu(x):
    return x * torch.sigmoid(1.702 * x)


def _ln(x, w, b):
    return F.layer_norm(x.float(), (x.shape[-1],), w.float(), b.float(), eps=1e-5).to(x.dtype)


def _attention(q, k, v, heads, causal, dtype):
    B, T, W = q.shape
    d = W // heads
    q, k, v = (t.reshape(B, T, heads, d).transpose(1, 2) for t in (q, k, v))
    s = torch.matmul(q.float(), k.float().transpose(-1, -2)) * d ** -0.5
    if causal:
        s = s + torch.full((T, T), float("-inf")).triu(1).to(s.device)
    w = torch.softmax(s, dim=-1).to(dtype)
    return torch.matmul(w, v).transpose(1, 2).reshape(B, T, W)


def _resblocks(x, layers, heads, causal, dtype):
    """layers: per block (ln_1, (wq, bq), (wk, bk), (wv, bv), (wo, bo), ln_2, c_fc, c_proj) with ln = (weight, bias)."""
    for ln1, q, k, v, o, ln2, fc, proj in layers:
        y = _ln(x, *ln1)
        x = x + F.linear(_attention(F.linear(y, *q), F.linear(y, *k), F.linear(y, *v), heads, causal, dtype), *o)
        x = x + F.linear(quick_gelu(F.linear(_ln(x, *ln2), *fc)), *proj)
    return x


def _openai_layers(sd, prefix, L, dtype):
    out = []
    for i in range(L):
        p = f"{prefix}resblocks.{i}."
        g = lambda n: (sd[p + n + ".weight"].to(dtype), sd[p + n + ".bias"].to(dtype))  # noqa: E731
        wq, wk, wv = sd[p + "attn.in_proj_weight"].to(dtype).chunk(3)
        bq, bk, bv = sd[p + "attn.in_proj_bias"].to(dtype).chunk(3)
        ln = lambda n: (sd[p + n + ".weight"], sd[p + n + ".bias"])  # noqa: E731
        out.append((ln("ln_1"), (wq, bq), (wk, bk), (wv, bv), g("attn.out_proj"), ln("ln_2"), g("mlp.c_fc"), g("mlp.c_proj")))
    return out


def _k2_layers(sd, L):
    out = []
    for i in range(L):
        p = f"layers.{i}."
        g = lambda n: (sd[p + n + ".weight"].float(), sd[p + n + ".bias"].float())  # noqa: E731
        w, b = g("attn.qkv")
        W = w.shape[1]
        heads = W // 64
        wq, wk, wv = (w.view(heads, 3, 64, W)[:, j].reshape(W, W) for j in range(3))
        bq, bk, bv = (b.view(heads, 3, 64)[:, j].reshape(W) for j in range(3))
        out.append((g("ln_1"), (wq, bq), (wk, bk), (wv, bv), g("attn.proj"), g("ln_2"), g("mlp.fc1"), g("mlp.fc2")))
    return out


def text_forward(sd, tokens, dtype=torch.float32):
    """OpenAI names, tokens int [n, context] -> (txt_feat_seq [n, context, width] = ln_final rows, txt_feat [n, embed_dim]),
    both fp32."""
    tw = sd["ln_final.weight"].shape[0]
    L = sum(1 for k in sd if k.startswith("transformer.resblocks.") and k.endswith("attn.in_proj_weight"))
    tokens = tokens.long()
    x = sd["token_embedding.weight"].to(dtype)[tokens] + sd["positional_embedding"].to(dtype)
    x = _resblocks(x, _openai_layers(sd, "transformer.", L, dtype), tw // 64, True, dtype)
    x = _ln(x, sd["ln_final.weight"], sd["ln_final.bias"])
    pooled = x[torch.arange(x.shape[0], device=x.device), tokens.argmax(dim=-1)]
    return x.float(), (pooled @ sd["text_projection"].to(dtype)).float()


def vision_forward(sd, pixels, dtype=torch.float32):
    """OpenAI names, pixels fp32 [B, 3, S, S] -> (last resblock output [B, T, width], image embedding [B, embed_dim]), fp32."""
    w = sd["visual.conv1.weight"].to(dtype)
    W = w.shape[0]
    L = sum(1 for k in sd if k.startswith("visual.transformer.resblocks.") and k.endswith("attn.in_proj_weight"))
    x = F.conv2d(pixels.to(dtype), w, stride=w.shape[-1]).flatten(2).transpose(1, 2)
    cls = sd["visual.class_embedding"].to(dtype).expand(x.shape[0], 1, W)
    x = torch.cat([cls, x], dim=1) + sd["visual.positional_embedding"].to(dtype)
    x = _ln(x, sd["visual.ln_pre.weight"], sd["visual.ln_pre.bias"])
    x = _resblocks(x, _openai_layers(sd, "visual.transformer.", L, dtype), W // 64, False, dtype)
    pooled = _ln(x[:, 0], sd["visual.ln_post.weight"], sd["visual.ln_post.bias"])
    return x.float(), (pooled @ sd["visual.proj"].to(dtype)).float()


def text_forward_k2(sd, tokens):
    """kandinsky2's text names (checkpoints.openai_clip_to_k2) -> text_forward's outputs, fp32."""
    L = sum(1 for k in sd if k.endswith("attn.qkv.weight"))
    tokens = tokens.long()
    x = sd["token_embedding"].float()[tokens] + sd["position_embedding"].float()
    x = _resblocks(x, _k2_layers(sd, L), x.shape[-1] // 64, True, torch.float32)
    x = _ln(x, sd["final_ln.weight"], sd["final_ln.bias"])
    return x, F.linear(x[torch.arange(x.shape[0], device=x.device), tokens.argmax(dim=-1)], sd["proj.weight"].float())


def vision_forward_k2(sd, pixels):
    """kandinsky2's vision names -> vision_forward's outputs, fp32."""
    L = sum(1 for k in sd if k.endswith("attn.qkv.weight"))
    w = sd["patch_embedding.weight"].float()
    W = w.shape[0]
    x = F.conv2d(pixels.float(), w, stride=w.shape[-1]).flatten(2).transpose(1, 2)
    x = torch.cat([sd["class_embedding"].float().expand(x.shape[0], 1, W), x], dim=1) + sd["position_embedding"].float()
    x = _ln(x, sd["pre_ln.weight"], sd["pre_ln.bias"])
    x = _resblocks(x, _k2_layers(sd, L), W // 64, False, torch.float32)
    return x, F.linear(_ln(x[:, 0], sd["post_ln.weight"], sd["post_ln.bias"]), sd["proj.weight"].float())


# ---------------------------------------------------------------------------------------------------------------------------
# transformers / torchvision references (fixture writer only)
# ---------------------------------------------------------------------------------------------------------------------------
def to_transformers(sd, geo):
    """OpenAI names -> transformers CLIPModel names (the conversion transformers' convert_clip_original_pytorch_to_hf does)."""
    out = {"text_model.embeddings.token_embedding.weight": sd["token_embedding.weight"],
           "text_model.embeddings.position_embedding.weight": sd["positional_embedding"],
           "text_model.final_layer_norm.weight": sd["ln_final.weight"], "text_model.final_layer_norm.bias": sd["ln_final.bias"],
           "text_projection.weight": sd["text_projection"].t().contiguous(),
           "vision_model.embeddings.class_embedding": sd["visual.class_embedding"],
           "vision_model.embeddings.patch_embedding.weight": sd["visual.conv1.weight"],
           "vision_model.embeddings.position_embedding.weight": sd["visual.positional_embedding"],
           "vision_model.pre_layrnorm.weight": sd["visual.ln_pre.weight"], "vision_model.pre_layrnorm.bias": sd["visual.ln_pre.bias"],
           "vision_model.post_layernorm.weight": sd["visual.ln_post.weight"],
           "vision_model.post_layernorm.bias": sd["visual.ln_post.bias"],
           "visual_projection.weight": sd["visual.proj"].t().contiguous(), "logit_scale": torch.tensor(2.6592)}
    for tower, prefix, L in (("text", "transformer.", geo["text_layers"]), ("vision", "visual.transformer.", geo["vision_layers"])):
        for i in range(L):
            p, h = f"{prefix}resblocks.{i}.", f"{tower}_model.encoder.layers.{i}."
            for n, w, b in zip("qkv", sd[p + "attn.in_proj_weight"].chunk(3), sd[p + "attn.in_proj_bias"].chunk(3)):
                out[f"{h}self_attn.{n}_proj.weight"], out[f"{h}self_attn.{n}_proj.bias"] = w, b
            for a, b in (("attn.out_proj", "self_attn.out_proj"), ("ln_1", "layer_norm1"), ("ln_2", "layer_norm2"),
                         ("mlp.c_fc", "mlp.fc1"), ("mlp.c_proj", "mlp.fc2")):
                for s in ("weight", "bias"):
                    out[f"{h}{b}.{s}"] = sd[f"{p}{a}.{s}"]
    return out


def transformers_outputs(sd, geo, tokens, pixels):
    """transformers' CLIPModel (eager attention, fp32, quick_gelu, eos_token_id 2) -> (text seq, text emb, image emb)."""
    from transformers import CLIPConfig, CLIPModel
    tc = dict(vocab_size=geo["vocab"], hidden_size=geo["text_width"], intermediate_size=4 * geo["text_width"],
              num_hidden_layers=geo["text_layers"], num_attention_heads=geo["text_width"] // 64,
              max_position_embeddings=geo["context"], hidden_act="quick_gelu", eos_token_id=2, bos_token_id=0, pad_token_id=1)
    vc = dict(hidden_size=geo["vision_width"], intermediate_size=4 * geo["vision_width"], num_hidden_layers=geo["vision_layers"],
              num_attention_heads=geo["vision_width"] // 64, image_size=geo["image_size"], patch_size=geo["patch"],
              hidden_act="quick_gelu")
    cfg = CLIPConfig(text_config=tc, vision_config=vc, projection_dim=geo["embed_dim"])
    cfg._attn_implementation = "eager"
    model = CLIPModel(cfg).eval()
    model.load_state_dict(to_transformers(sd, geo), strict=True)
    with torch.no_grad():
        t = model.text_model(input_ids=tokens.long())
        v = model.vision_model(pixel_values=pixels)
        return (t.last_hidden_state.float(), model.text_projection(t.pooler_output).float(),
                model.visual_projection(v.pooler_output).float())


def clip_transform(size=224):
    """clip's _transform(size) with torchvision."""
    from torchvision.transforms import CenterCrop, Compose, InterpolationMode, Normalize, Resize, ToTensor
    return Compose([Resize(size, interpolation=InterpolationMode.BICUBIC), CenterCrop(size), lambda im: im.convert("RGB"),
                    ToTensor(), Normalize(MEAN, STD)])


def sample_images():
    """[(name, PIL image)]: deterministic noise over a smooth gradient, in the modes and sizes of IMAGES."""
    from PIL import Image
    out = []
    for i, (name, mode, w, h) in enumerate(IMAGES):
        rng = np.random.default_rng(300 + i)
        ch = {"RGB": 3, "RGBA": 4, "L": 1}[mode]
        yy, xx = np.mgrid[0:h, 0:w]
        base = (127 + 100 * np.sin(xx / 13.0 + i) * np.cos(yy / 19.0))[..., None]
        a = np.clip(base + rng.normal(0, 30, (h, w, ch)), 0, 255).astype(np.uint8)
        out.append((name, Image.fromarray(a[..., 0] if ch == 1 else a, mode)))
    return out


def sha256(t):
    return hashlib.sha256(t.contiguous().numpy().tobytes()).hexdigest()


def sample_tokens(geo, seed, n=3):
    """int32 [n, context] rows like padded_tokens_and_mask's: sot, ids, eot (the largest id), zero padding; the last row is
    full length."""
    g = torch.Generator().manual_seed(seed)
    V, T = geo["vocab"], geo["context"]
    out = torch.zeros(n, T, dtype=torch.int32)
    for r in range(n):
        L = T if r == n - 1 else 2 + r * 3
        out[r, :L] = torch.randint(1, V - 2, (L,), generator=g, dtype=torch.int32)
        out[r, 0], out[r, L - 1] = V - 2, V - 1
    return out


def sample_pixels(geo, seed, batch=2):
    return torch.randn(batch, 3, geo["image_size"], geo["image_size"], generator=torch.Generator().manual_seed(seed))


def write_fixture():
    """The fixture holds transformers' outputs on the tiny geometry (weights, tokens and pixels are regenerated from their
    seeds) and, per sample image, the SHA-256 and first row of torchvision's clip transform output."""
    import torchvision
    import transformers

    from kandinsky2.model.clip_vitl14 import preprocess_openai
    geo, wseed, tseed, pseed = GEO_TINY, 11, 12, 13
    sd = synth_weights(geo, wseed)
    tokens, pixels = sample_tokens(geo, tseed), sample_pixels(geo, pseed)
    seq, temb, iemb = transformers_outputs(sd, geo, tokens, pixels)
    oseq, otemb = text_forward(sd, tokens)
    _, oiemb = vision_forward(sd, pixels)
    rel = max(((a - b).norm() / b.norm()).item() for a, b in ((oseq, seq), (otemb, temb), (oiemb, iemb)))
    assert rel <= 1e-5, f"oracle deviates from transformers by rel {rel}"
    pix_sha, rows, tf = {}, {}, clip_transform()
    for name, img in sample_images():
        ref = tf(img)
        assert torch.equal(preprocess_openai(img)[0], ref), name
        pix_sha[name], rows[name] = sha256(ref), ref[:, :1].clone()
    torch.save(dict(transformers_version=transformers.__version__, torchvision_version=torchvision.__version__, geo=geo,
                    weight_seed=wseed, token_seed=tseed, pixel_seed=pseed, tokens=tokens, pixel_sha256=sha256(pixels),
                    txt_feat_seq=seq, txt_feat=temb, image_emb=iemb, preprocess_sha256=pix_sha, preprocess_rows=rows),
               FIXTURE)
    print(f"wrote {FIXTURE} (transformers {transformers.__version__}, torchvision {torchvision.__version__}, "
          f"{os.path.getsize(FIXTURE)} bytes; oracle vs transformers rel {rel:.1e})")


if __name__ == "__main__":
    import sys
    sys.path.insert(0, os.path.join(ROOT, "kandinsky-2_b200"))
    write_fixture()
