"""The CLIP image tower of the Kandinsky 2.2 prior pipeline: a transformers `CLIPVisionModelWithProjection` (ViT-bigG/14 in
`kandinsky-2-2-prior/image_encoder`), which the reference builds at `kandinsky2_2_model.py:24` and diffusers runs for the
default decoder negative (`get_zero_embed`), the image items of `interpolate` and the PIL images of the emb2emb prior.

The tower is read from the checkpoint's `config.json` (hidden 1664, 48 layers, 16 heads of 104, MLP 8192, patch 14, image 224,
projection 1280, exact GELU for ViT-bigG/14); what is not implemented is refused with K2Error: any `hidden_act` but "gelu", any
head width but 104.  Compute, per batch size one LaunchPlan replayed as one CUDA graph:
    k2_clip_patchify -> ONE GEMM: patch conv + class embedding (K column 3 P^2) + position embedding (the epilogue residual),
    pre_layrnorm, then the pre-LayerNorm layers of model/encoder.py (q / k / v packed per head) with k2_attention_heads as the
    attention,
    post_layernorm on the CLS rows (a strided view), fp16 -> fp32, and the bias-free visual_projection in fp32 (ops.linear).
fp16 storage, fp32 accumulation, fp32 softmax with P rounded to fp16 before PV, the prior's LayerNorm statistics.

Parity: tests/test_cpu_clip_vision.py pins the oracle (tests/clip_vision_oracle.py) and `preprocess` to transformers
(tests/golden/clip_vision_tiny.pt); tests/test_gpu_zz_clip_vision.py runs the tower against the golden and, at full size on
synthetic weights, against the fp32 oracle.
"""
import math

import numpy as np
import torch

from .. import ops
from .._native import K2Error
from ..launch_plan import LaunchPlan
from .encoder import (Tower, clip_config, f16, f32, layer_shapes, pack_layers, pack_patch_embed, record_layers,
                      record_patch_embed)

OPENAI_CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
# CLIPImageProcessor as kandinsky-2-2-prior's image_processor configures it (transformers' defaults for CLIP)
DEFAULT_PREPROCESSOR = dict(do_convert_rgb=True, do_resize=True, size={"shortest_edge": 224}, resample=3, do_center_crop=True,
                            crop_size={"height": 224, "width": 224}, do_rescale=True, rescale_factor=1 / 255, do_normalize=True,
                            image_mean=list(OPENAI_CLIP_MEAN), image_std=list(OPENAI_CLIP_STD))
_REQUIRED = ("hidden_size", "intermediate_size", "num_hidden_layers", "num_attention_heads", "image_size", "patch_size",
             "projection_dim")


def tower_config(config):
    """The transformers CLIPVisionConfig dict -> the geometry this module implements; K2Error for anything else.  A key that
    is absent takes transformers' default (hidden_act "quick_gelu", layer_norm_eps 1e-5, num_channels 3)."""
    c = clip_config(config, _REQUIRED, "vision", 104)
    if int(config.get("num_channels", 3)) != 3:
        raise K2Error("CLIP vision tower: only 3-channel images are implemented")
    if c["image_size"] % c["patch_size"]:
        raise K2Error("CLIP vision tower: image_size must be a multiple of patch_size")
    c["tokens"] = (c["image_size"] // c["patch_size"]) ** 2 + 1
    c["kp"] = (3 * c["patch_size"] ** 2 + 1 + 63) // 64 * 64
    return c


def preprocess_images(images, config=None):
    """CLIPImageProcessor (transformers' PIL backend, restated) -> fp32 [B, 3, crop, crop] on the CPU.  Per image: convert to
    RGB (RGBA drops alpha, L is replicated), resize the shortest edge to size["shortest_edge"] with the long edge
    int(S * long / short) (PIL, `resample`), center-crop at ((h - ch) // 2, (w - cw) // 2) (zero-padded if smaller), then
    float32(uint8 * rescale_factor in float64), then (x - mean) / std in float32.  config: a preprocessor_config.json dict
    (defaults: DEFAULT_PREPROCESSOR)."""
    from PIL import Image
    cfg = dict(DEFAULT_PREPROCESSOR)
    cfg.update(config or {})
    if isinstance(images, Image.Image):
        images = [images]
    out = []
    for img in images:
        if cfg["do_convert_rgb"] and img.mode != "RGB":
            img = img.convert("RGB")
        if cfg["do_resize"]:
            S = int(cfg["size"]["shortest_edge"])
            w, h = img.size
            short, long = (w, h) if w <= h else (h, w)
            new_long = int(S * long / short)
            nh, nw = (new_long, S) if w <= h else (S, new_long)
            img = img.resize((nw, nh), resample=int(cfg["resample"]))
        a = np.array(img)
        if a.ndim == 2:
            a = a[:, :, None]
        a = a.transpose(2, 0, 1)
        if cfg["do_center_crop"]:
            ch, cw = int(cfg["crop_size"]["height"]), int(cfg["crop_size"]["width"])
            a = _center_crop(a, ch, cw)
        out.append(rescale_normalize(a, cfg))
    return torch.stack(out)


def rescale_normalize(x, cfg):
    """The end of transformers' image processors on a uint8 CHW array -> fp32 CHW tensor: float32(x * rescale_factor in
    float64) when do_rescale, then (x - image_mean) / image_std in float32 when do_normalize (model/depth.py's
    DPTImageProcessorPil ends the same way)."""
    if cfg["do_rescale"]:
        x = (x.astype(np.float64) * cfg["rescale_factor"]).astype(np.float32)
    if cfg["do_normalize"]:
        x = x.astype(np.float32) if not np.issubdtype(x.dtype, np.floating) else x
        mean = np.array(cfg["image_mean"], dtype=x.dtype)
        std = np.array(cfg["image_std"], dtype=x.dtype)
        x = ((x.T - mean) / std).T
    return torch.from_numpy(np.ascontiguousarray(x)).float()


def _center_crop(a, ch, cw):
    """transformers' image_transforms.center_crop on a CHW array."""
    h, w = a.shape[1:]
    top, left = (h - ch) // 2, (w - cw) // 2
    if top >= 0 and left >= 0 and top + ch <= h and left + cw <= w:
        return a[:, top:top + ch, left:left + cw]
    nh, nw = max(ch, h), max(cw, w)
    big = np.zeros((a.shape[0], nh, nw), dtype=a.dtype)
    tp, lp = math.ceil((nh - h) / 2), math.ceil((nw - w) / 2)
    big[:, tp:tp + h, lp:lp + w] = a
    top, left = top + tp, left + lp
    return big[:, max(0, top):min(nh, top + ch), max(0, left):min(nw, left + cw)]


class CLIPVisionTower(Tower):
    """CLIPVisionModelWithProjection on this package's kernels.  sd: state dict in this module's names
    (checkpoints.transformers_clip_vision_to_k2); config: the transformers config.json dict; preprocessor_config: the
    image processor's dict (None = DEFAULT_PREPROCESSOR)."""

    what = "CLIP vision tower"
    act = "gelu"   # the layers' MLP activation (encoder.ACTIVATIONS)

    def __init__(self, sd, config, device="cuda", preprocessor_config=None):
        self.cfg, self.device = tower_config(config), torch.device(device)
        self.preprocessor_config = preprocessor_config
        self._take(sd, self._want())

    def _want(self):
        """{name: shape} of the state dict this tower takes."""
        c = self.cfg
        H, P, T = c["hidden_size"], c["patch_size"], c["tokens"]
        want = {"class_embedding": (H,), "patch_embedding.weight": (H, 3, P, P), "position_embedding": (T, H),
                "pre_ln.weight": (H,), "pre_ln.bias": (H,), "post_ln.weight": (H,), "post_ln.bias": (H,),
                "proj.weight": (c["projection_dim"], H)}
        want.update({f"layers.{i}.{k}": s for i in range(c["num_hidden_layers"])
                     for k, s in layer_shapes(H, c["intermediate_size"]).items()})
        return want

    @classmethod
    def from_transformers(cls, state_dict, config, device="cuda", preprocessor_config=None):
        """From a transformers CLIPVisionModelWithProjection state dict and its config.json dict; packs the weights."""
        from ..checkpoints import transformers_clip_vision_to_k2
        c = tower_config(config)
        sd = transformers_clip_vision_to_k2(state_dict, head_dim=c["head_dim"])
        return cls(sd, config, device, preprocessor_config).finalize()

    def _pack(self):
        """fp16 GEMM weights [N, K] (the patch embedding as [H, Kp] with the class embedding in column 3 P^2,
        pack_patch_embed), fp32 biases / LayerNorm parameters / projection, the fp16 position embedding."""
        c, dev, sd = self.cfg, self.device, self.sd
        return {"embed": pack_patch_embed(sd["patch_embedding.weight"], sd["class_embedding"], c["kp"], dev),
                "pos": f16(sd["position_embedding"], dev),
                "pre_ln": (f32(sd["pre_ln.weight"], dev), f32(sd["pre_ln.bias"], dev)),
                "post_ln": (f32(sd["post_ln.weight"], dev), f32(sd["post_ln.bias"], dev)),
                "proj": f32(sd["proj.weight"], dev),
                "layers": pack_layers(lambda i, name: sd[f"layers.{i}.{name}"], c["num_hidden_layers"], dev)}

    def _new_plan(self, B):
        return _TowerPlan(self, B)

    def attend(self, qkv, out):
        """The layers' attention: qkv fp16 [B, T, heads * 3 head_dim] (per head [q | k | v]) -> out fp16 [B, T, hidden]."""
        c = self.cfg
        return ops.attention_heads(qkv, c["num_attention_heads"], c["head_dim"], c["head_dim"] ** -0.5, out=out)

    def preprocess(self, images):
        """PIL image(s) -> fp32 pixel_values [B, 3, S, S] on the CPU (preprocess_images with this tower's processor config)."""
        return preprocess_images(images, self.preprocessor_config)

    @torch.no_grad()
    def forward(self, pixel_values, use_graph=True):
        """pixel_values fp32 [B, 3, S, S] -> (last_hidden_state fp16 [B, T, hidden], image_embeds fp32 [B, projection_dim]), on
        the device.  One CUDA graph replay of the batch size's launch plan (use_graph=False: the same launches one by one)."""
        S = self.cfg["image_size"]
        if pixel_values.dim() != 4 or tuple(pixel_values.shape[1:]) != (3, S, S):
            raise K2Error(f"{self.what}: pixel_values must be [B, 3, {S}, {S}], got {list(pixel_values.shape)}")
        plan = self._plan(pixel_values.shape[0])
        plan.pix.copy_(pixel_values)
        plan.run(use_graph)
        return plan.hidden.clone(), plan.out.clone()

    def image_embeds(self, pixel_values, use_graph=True):
        """pixel_values fp32 [B, 3, S, S] -> image_embeds fp32 [B, projection_dim] on the device."""
        return self.forward(pixel_values, use_graph)[1]

    def __call__(self, image):
        """The embedders' clip_image protocol: a PIL image -> fp32 [1, projection_dim] on the CPU."""
        return self.image_embeds(self.preprocess(image).to(self.device)).float().cpu()

    def zero_embed(self):
        """diffusers' get_zero_embed: the tower on an all-zero pixel_values tensor [1, 3, S, S] (zeros after normalisation,
        not a black image) -> fp32 [1, projection_dim] on the device."""
        S = self.cfg["image_size"]
        return self.image_embeds(torch.zeros(1, 3, S, S, device=self.device))


class _TowerPlan(LaunchPlan):
    """The tower at B images as one static launch list over fixed buffers (replayed as one CUDA graph): pix -> patchify ->
    embedding GEMM (+ position embedding, tiled over the batch once here) -> pre LayerNorm -> L layers -> post LayerNorm of the
    CLS rows -> fp32 -> projection.  self.hidden is the last layer's output (transformers' last_hidden_state), self.out the
    image embeddings."""

    def __init__(self, tower, B):
        super().__init__(tower.device, B)
        self.t, self.B = tower, B
        c = tower.cfg
        S, T, H = c["image_size"], c["tokens"], c["hidden_size"]
        self.pix = torch.zeros(B, 3, S, S, device=self.dev, dtype=torch.float32)
        self.pos = tower._packed["pos"].expand(B, T, H).contiguous()
        self.out = torch.zeros(B, c["projection_dim"], device=self.dev, dtype=torch.float32)
        self._build()

    def _build(self):
        c, pk, B, S = self.t.cfg, self.t._packed, self.B, self._add
        T, H, hd, heads, eps = c["tokens"], c["hidden_size"], c["head_dim"], c["num_attention_heads"], c["layer_norm_eps"]
        emb = record_patch_embed(self, self.pix, pk["embed"], self.pos, c["patch_size"], c["kp"])
        x = self._new(B, T, H)
        S(lambda: ops.layernorm_f16(emb, *pk["pre_ln"], eps=eps, out=x), "layernorm")
        h = record_layers(self, x, pk["layers"], self.t.attend, 4 * B * heads * T * T * hd, eps, act=self.t.act)
        self.hidden = h
        cls, cls32 = self._new(B, H), torch.empty(B, H, device=self.dev, dtype=torch.float32)
        S(lambda: ops.layernorm_f16(h[:, 0], *pk["post_ln"], eps=eps, out=cls), "layernorm")
        S(lambda: ops.f16_to_f32(cls, out=cls32), "widen")
        S(lambda: ops.linear(cls32, pk["proj"], out=self.out), "linear", 2 * B * H * c["projection_dim"])
