"""The depth estimator behind the Kandinsky 2.2 ControlNet-depth hint: transformers' `DPTForDepthEstimation` with a plain ViT
backbone (`is_hybrid` false, no `backbone_config`; `Intel/dpt-large` is the default model of transformers' depth-estimation
pipeline, which diffusers' kandinsky-2-2-controlnet-depth documentation uses to build the hint).

The network is read from the checkpoint's `config.json` (for Intel/dpt-large: hidden 1024, 24 layers, 16 heads of 64, MLP
4096, patch 16, image 384, backbone_out_indices [5, 11, 17, 23], neck sizes [256, 512, 1024, 1024], fusion 256); what is
not implemented is refused with K2Error naming the key (dpt_config).  Compute, per batch size one LaunchPlan replayed as
one CUDA graph:
    backbone  k2_clip_patchify -> ONE GEMM: patch conv + CLS column + (position embedding + conv bias on the patch rows) as
              the residual, then the pre-LayerNorm layers of model/encoder.py with k2_attention_d64, recorded in segments
              that end at each backbone_out_indices layer, so each kept hidden state has a buffer of its own;
    neck      per stage: k2_readout_rows_f16 ([token | CLS] rows) -> Linear(2H -> H) GEMM -> GELU -> 1x1 projection GEMM ->
              resize (factor 4 / 2: ConvTranspose2d as one GEMM with the bias tiled, then k2_depth_to_space_f16; 1: none;
              0.5: the stride-1 3x3 convolution, then every second pixel: k2_subsample2_nhwc for an even grid, or for an odd
              grid k2_bilinear_f16 with align_corners, whose source index is then exactly 2i) -> bias-free 3x3 conv;
    fusion    from the deepest stage up: [bilinear resize of the stage to the running map (align_corners=False; only where
              the sizes differ, i.e. odd patch grids) -> running + unit1(stage)], unit2, bilinear x2 (align_corners=True),
              1x1 projection; unit(x) = conv3x3(relu(conv3x3(relu(x)))) + x with k2_relu_f16.  The sum running + unit1
              is the last convolution's epilogue: the running map is a second, 1x1 source of that GEMM with an identity
              weight block (exact products, one fp32 sum, one rounding);
    head      conv3x3 -> bilinear x2 (align_corners=True) -> conv3x3 -> ReLU -> 1x1 conv to one channel, fp32 NCHW out
              (k2_conv_gemm out_mode 1) -> k2_relu_f32.
fp16 storage, fp32 accumulation, the prior's LayerNorm statistics.  Not run, as in transformers: the final LayerNorm
(`dpt.layernorm`: the neck reads the raw per-layer hidden states) and the first fusion layer's residual_layer1 (it gets no
residual); their keys are accepted and dropped by checkpoints.transformers_dpt_to_k2.

Host side: preprocess restates transformers' DPTImageProcessorPil (RGB, PIL resize with the configured resample, rescale,
normalise; only a square output that is a multiple of the patch size is accepted); depth restates the depth-estimation
pipeline's postprocess (bicubic resize to the image's size, min-max to [0, 255], uint8) except that a constant map gives
zeros where transformers divides by zero; make_hint restates the hint builder of diffusers' kandinsky-2-2-controlnet-depth
documentation.

The hybrid (is_hybrid: MiDaS v3 DPT-Hybrid, Intel/dpt-hybrid-midas, the estimator of ControlNet's MidasDetector) replaces the
patch embedding with a BiT ResNet backbone (_HybridPlan) and takes any input size that is a multiple of 16; midas_hint
restates the ControlNet notebook's make_hint(img, MidasDetector()).  Parity: tests/test_cpu_dpt_hybrid.py,
tests/test_gpu_zz_dpt_hybrid.py.

Parity: tests/test_cpu_dpt.py pins the oracle (tests/dpt_oracle.py), preprocess and postprocess to transformers
(tests/golden/dpt_tiny.pt); tests/test_gpu_zz_depth.py runs the estimator against the golden and, at the Intel/dpt-large
geometry on synthetic weights, against the fp32 oracle.
"""
import math
import os

import numpy as np
import torch

from .. import ops
from .._native import K2Error
from ..checkpoints import load_weights, read_json
from ..launch_plan import LaunchPlan
from .clip_vision import rescale_normalize
from .encoder import Tower, f32, layer_shapes, pack_layers, pack_patch_embed, record_layers, record_patch_embed

# transformers' DPTConfig defaults, for keys a config.json leaves out
_CONFIG_DEFAULTS = dict(hidden_size=768, num_hidden_layers=12, num_attention_heads=12, intermediate_size=3072,
                        hidden_act="gelu", layer_norm_eps=1e-12, image_size=384, patch_size=16, num_channels=3, is_hybrid=False,
                        qkv_bias=True, backbone_out_indices=[2, 5, 8, 11], readout_type="project",
                        reassemble_factors=[4, 2, 1, 0.5], neck_hidden_sizes=[96, 192, 384, 768], fusion_hidden_size=256,
                        head_in_index=-1, use_batch_norm_in_fusion_residual=False, use_bias_in_fusion_residual=None,
                        add_projection=False, backbone_config=None, backbone=None)
# DPTImageProcessorPil's defaults (resample 3 = PIL BICUBIC; mean / std are IMAGENET_STANDARD_*)
DEFAULT_PREPROCESSOR = dict(do_resize=True, size={"height": 384, "width": 384}, resample=3, do_rescale=True,
                            rescale_factor=1 / 255, do_normalize=True, image_mean=[0.5, 0.5, 0.5], image_std=[0.5, 0.5, 0.5],
                            keep_aspect_ratio=False, ensure_multiple_of=1, do_pad=False)


def dpt_config(config):
    """The transformers DPTConfig dict -> the geometry this module implements; K2Error naming the key for anything else."""
    c = dict(_CONFIG_DEFAULTS)
    c.update({k: v for k, v in config.items() if k in _CONFIG_DEFAULTS})
    refuse = [("is_hybrid", c["is_hybrid"], "the hybrid (BiT) DPT"),
              ("backbone_config", c["backbone_config"] is not None, "a separate backbone"),
              ("backbone", c["backbone"] is not None, "a separate backbone"),
              ("readout_type", c["readout_type"] != "project", f"readout_type {c['readout_type']!r}"),
              ("hidden_act", c["hidden_act"] != "gelu", f"hidden_act {c['hidden_act']!r}"),
              ("use_batch_norm_in_fusion_residual", c["use_batch_norm_in_fusion_residual"], "batch norm in the fusion units"),
              ("use_bias_in_fusion_residual", c["use_bias_in_fusion_residual"] is False, "bias-free fusion units"),
              ("add_projection", c["add_projection"], "the head's extra projection"),
              ("head_in_index", c["head_in_index"] != -1, f"head_in_index {c['head_in_index']}"),
              ("qkv_bias", not c["qkv_bias"], "bias-free q / k / v"),
              ("num_channels", c["num_channels"] != 3, f"{c['num_channels']}-channel images")]
    for key, bad, what in refuse:
        if bad:
            raise K2Error(f"DPT config: {key}: {what} is not implemented (only the plain-ViT DPT of Intel/dpt-large)")
    for k in ("hidden_size", "num_hidden_layers", "num_attention_heads", "intermediate_size", "image_size", "patch_size",
              "fusion_hidden_size"):
        if not isinstance(c[k], int) or isinstance(c[k], bool) or c[k] <= 0:
            raise K2Error(f"DPT config: {k} must be a positive integer, got {c[k]!r}")
    H, heads = c["hidden_size"], c["num_attention_heads"]
    if H % heads or H // heads != 64:
        raise K2Error(f"DPT config: num_attention_heads: head width {H / heads:g} is not implemented (only 64)")
    factors = [float(f) for f in c["reassemble_factors"]]
    if any(f not in (4.0, 2.0, 1.0, 0.5) for f in factors):
        raise K2Error(f"DPT config: reassemble_factors {c['reassemble_factors']}: only 4, 2, 1 and 0.5 are implemented")
    idx, sizes = [int(i) for i in c["backbone_out_indices"]], [int(s) for s in c["neck_hidden_sizes"]]
    if not (len(idx) == len(sizes) == len(factors)) or not idx:
        raise K2Error("DPT config: backbone_out_indices, neck_hidden_sizes and reassemble_factors must have one entry per "
                      "neck stage")
    if idx != sorted(set(idx)) or idx[0] < 0 or idx[-1] >= c["num_hidden_layers"]:
        raise K2Error(f"DPT config: backbone_out_indices {idx} must be increasing layer indices below num_hidden_layers")
    if c["image_size"] % c["patch_size"]:
        raise K2Error("DPT config: image_size must be a multiple of patch_size")
    if any(s % 8 for s in sizes) or c["fusion_hidden_size"] % 16 or H % 8:
        raise K2Error("DPT config: neck_hidden_sizes and hidden_size must be multiples of 8, fusion_hidden_size of 16")
    c.update(reassemble_factors=factors, backbone_out_indices=idx, neck_hidden_sizes=sizes, head_dim=64,
             layer_norm_eps=float(c["layer_norm_eps"]), kp=(3 * c["patch_size"] ** 2 + 1 + 63) // 64 * 64)
    return c


# transformers' BitConfig defaults as DPTConfig fills them in for a hybrid model without a backbone_config
_BIT_DEFAULTS = dict(num_channels=3, embedding_size=64, hidden_sizes=[256, 512, 1024, 2048], depths=[3, 4, 9],
                     layer_type="bottleneck", hidden_act="relu", global_padding="same", num_groups=32,
                     embedding_dynamic_padding=True, output_stride=32, width_factor=1,
                     out_features=["stage1", "stage2", "stage3"])
BIT_GN_EPS = 1e-5   # BitGroupNormActivation
BIT_WS_EPS = 1e-8   # WeightStandardizedConv2d in every BiT layer


def _make_div(v, divisor=8):
    """transformers' modeling_bit.make_div."""
    n = max(divisor, int(v + divisor / 2) // divisor * divisor)
    return n + divisor if n < 0.9 * v else n


def dpt_hybrid_config(config):
    """The transformers DPTConfig dict of a hybrid DPT (MiDaS v3 DPT-Hybrid: BiT ResNet + ViT, Intel/dpt-hybrid-midas) -> the
    geometry this module implements; K2Error naming the key for anything else.  The ViT, neck and head follow dpt_config's
    rules; c["bit"] holds the backbone: stem width, three stages' channels, bottleneck widths and depths."""
    if not config.get("is_hybrid"):
        raise K2Error("DPT-Hybrid config: is_hybrid: the config is not a hybrid DPT")
    plain = {k: v for k, v in config.items() if k not in ("is_hybrid", "backbone_config", "backbone")}
    c = dpt_config(plain)
    bc = dict(_BIT_DEFAULTS)
    bc.update({k: v for k, v in (config.get("backbone_config") or {}).items() if k in _BIT_DEFAULTS})

    def refuse(key, what):
        raise K2Error(f"DPT-Hybrid config: {key}: {what} is not implemented (only the BiT bottleneck backbone of "
                      f"Intel/dpt-hybrid-midas)")
    if config.get("backbone") is not None:
        refuse("backbone", "a named backbone")
    mt = (config.get("backbone_config") or {}).get("model_type", "bit")
    if mt != "bit":
        refuse("backbone_config.model_type", repr(mt))
    checks = [("layer_type", bc["layer_type"] == "bottleneck"),
              ("global_padding", str(bc["global_padding"]).lower() == "same"),
              ("embedding_dynamic_padding", bc["embedding_dynamic_padding"] is True),
              ("out_features", list(bc["out_features"]) == ["stage1", "stage2", "stage3"]),
              ("depths", len(bc["depths"]) == 3 and all(isinstance(d, int) and d > 0 for d in bc["depths"])),
              ("width_factor", bc["width_factor"] == 1),
              ("hidden_act", bc["hidden_act"] == "relu"),
              ("num_groups", bc["num_groups"] == 32),
              ("output_stride", bc["output_stride"] >= 16),
              ("num_channels", bc["num_channels"] == 3),
              ("hidden_sizes", len(bc["hidden_sizes"]) >= 3)]
    for key, ok in checks:
        if not ok:
            refuse(f"backbone_config.{key}", f"{key} {bc[key]!r}")
    chans = [_make_div(h) for h in bc["hidden_sizes"][:3]]
    mids = [_make_div(ch * 0.25) for ch in chans]
    stem = int(bc["embedding_size"])
    if any(ch % 64 for ch in chans + mids + [stem]):
        refuse("backbone_config.hidden_sizes", "stage or stem widths that are not multiples of 64")
    if c["patch_size"] != 16:
        refuse("patch_size", f"patch_size {c['patch_size']} (the BiT stage-3 map is at 1/16)")
    if len(c["neck_hidden_sizes"]) != 4:
        refuse("neck_hidden_sizes", "a neck without four stages")
    if c["neck_hidden_sizes"][:2] != chans[:2]:
        refuse("neck_hidden_sizes", f"neck_hidden_sizes[0:2] {c['neck_hidden_sizes'][:2]} other than the BiT stage-1 / "
               f"stage-2 channels {chans[:2]}")
    fm = config.get("backbone_featmap_shape", [1, 1024, 24, 24])
    if fm is None or len(fm) < 2 or fm[1] != chans[2]:
        refuse("backbone_featmap_shape", f"backbone_featmap_shape {fm} whose channels are not the BiT stage-3 channels "
               f"{chans[2]}")
    if list(config.get("neck_ignore_stages", [0, 1])) != [0, 1]:
        refuse("neck_ignore_stages", f"neck_ignore_stages {config.get('neck_ignore_stages')}")
    c.update(is_hybrid=True, bit=dict(stem=stem, channels=chans, mids=mids, depths=[int(d) for d in bc["depths"]]),
             kp=_pad64(chans[2] + 1))
    return c


def _pad64(n):
    return (n + 63) // 64 * 64


def _bit_layer_shapes(b):
    """{name: shape} of the BiT backbone under this module's names (bit.*, transformers' names below
    dpt.embeddings.backbone.bit)."""
    want = {"bit.embedder.convolution.weight": (b["stem"], 3, 7, 7), "bit.embedder.norm.weight": (b["stem"],),
            "bit.embedder.norm.bias": (b["stem"],)}
    cin = b["stem"]
    for s, (ch, mid, depth) in enumerate(zip(b["channels"], b["mids"], b["depths"])):
        for l in range(depth):
            lp = f"bit.encoder.stages.{s}.layers.{l}."
            for conv, shape in (("1", (mid, cin, 1, 1)), ("2", (mid, mid, 3, 3)), ("3", (ch, mid, 1, 1))):
                want[f"{lp}conv{conv}.weight"] = shape
                want.update({f"{lp}norm{conv}.{k}": (shape[0],) for k in ("weight", "bias")})
            if l == 0:
                want.update({f"{lp}downsample.conv.weight": (ch, cin, 1, 1), f"{lp}downsample.norm.weight": (ch,),
                             f"{lp}downsample.norm.bias": (ch,)})
            cin = ch
    return want


def k2_hybrid_shapes(c):
    """{name: shape} of the state dict a hybrid DPTDepthEstimator takes (checkpoints.transformers_dpt_hybrid_to_k2's output):
    the plain DPT's ViT, neck stages 2 and 3, neck convolutions, fusion and head, the BiT backbone (bit.*) and the token
    projection over the stage-3 map (projection.*) in place of the patch embedding."""
    H = c["hidden_size"]
    rs = "neck.reassemble_stage."
    want = {k: s for k, s in k2_shapes(c).items()
            if not k.startswith(("patch_embedding.", f"{rs}readout_projects.0.", f"{rs}readout_projects.1.",
                                 f"{rs}layers.0.", f"{rs}layers.1."))}
    want.update({"projection.weight": (H, c["bit"]["channels"][2], 1, 1), "projection.bias": (H,)})
    want.update(_bit_layer_shapes(c["bit"]))
    return want


def standardize_weight(w, eps=BIT_WS_EPS):
    """WeightStandardizedConv2d's weight in float64: per output channel over in * kh * kw, (w - mean) / sqrt(biased var +
    eps)."""
    w = w.detach().double()
    flat = w.reshape(w.shape[0], -1)
    mean = flat.mean(1, keepdim=True)
    var = ((flat - mean) ** 2).mean(1, keepdim=True)
    return ((flat - mean) / torch.sqrt(var + eps)).reshape(w.shape)


def k2_shapes(c):
    """{name: shape} of the state dict DPTDepthEstimator takes (checkpoints.transformers_dpt_to_k2's output) for config c."""
    H, P, F = c["hidden_size"], c["patch_size"], c["fusion_hidden_size"]
    T0 = (c["image_size"] // P) ** 2 + 1
    want = {"cls_token": (H,), "position_embedding": (T0, H), "patch_embedding.weight": (H, 3, P, P),
            "patch_embedding.bias": (H,)}
    want.update({f"layers.{i}.{k}": s for i in range(c["num_hidden_layers"])
                 for k, s in layer_shapes(H, c["intermediate_size"]).items()})
    rs = "neck.reassemble_stage."
    for i, (C, f) in enumerate(zip(c["neck_hidden_sizes"], c["reassemble_factors"])):
        want.update({f"{rs}readout_projects.{i}.0.weight": (H, 2 * H), f"{rs}readout_projects.{i}.0.bias": (H,),
                     f"{rs}layers.{i}.projection.weight": (C, H, 1, 1), f"{rs}layers.{i}.projection.bias": (C,),
                     f"neck.convs.{i}.weight": (F, C, 3, 3)})
        if f != 1:
            k = int(f) if f > 1 else 3
            want.update({f"{rs}layers.{i}.resize.weight": (C, C, k, k), f"{rs}layers.{i}.resize.bias": (C,)})
        fp = f"neck.fusion_stage.layers.{i}."
        want.update({fp + "projection.weight": (F, F, 1, 1), fp + "projection.bias": (F,)})
        for unit in (("residual_layer1", "residual_layer2") if i else ("residual_layer2",)):
            for conv in ("convolution1", "convolution2"):
                want.update({f"{fp}{unit}.{conv}.weight": (F, F, 3, 3), f"{fp}{unit}.{conv}.bias": (F,)})
    want.update({"head.head.0.weight": (F // 2, F, 3, 3), "head.head.0.bias": (F // 2,), "head.head.2.weight": (32, F // 2, 3, 3),
                 "head.head.2.bias": (32,), "head.head.4.weight": (1, 32, 1, 1), "head.head.4.bias": (1,)})
    return want


def preprocessor_settings(preprocessor_config, image_size):
    """DPTImageProcessorPil's settings: DEFAULT_PREPROCESSOR updated with a preprocessor_config.json dict (None: the defaults at
    the model's image_size).  An integer `size` means a square of that side."""
    cfg = dict(DEFAULT_PREPROCESSOR, size={"height": image_size, "width": image_size})
    cfg.update(preprocessor_config or {})
    if isinstance(cfg["size"], int):
        cfg["size"] = {"height": cfg["size"], "width": cfg["size"]}
    if cfg.get("do_pad"):
        raise K2Error("DPT preprocessing: do_pad is not implemented")
    return cfg


def _constrain_to_multiple_of(val, multiple):
    x = round(val / multiple) * multiple
    return math.ceil(val / multiple) * multiple if x < 0 else x


def resize_output_size(h, w, cfg):
    """DPTImageProcessorPil's get_resize_output_image_size -> (height, width)."""
    oh, ow = int(cfg["size"]["height"]), int(cfg["size"]["width"])
    sh, sw = oh / h, ow / w
    if cfg["keep_aspect_ratio"]:
        if abs(1 - sw) < abs(1 - sh):
            sh = sw
        else:
            sw = sh
    m = int(cfg["ensure_multiple_of"])
    return _constrain_to_multiple_of(sh * h, m), _constrain_to_multiple_of(sw * w, m)


def preprocess_images(images, cfg, size):
    """DPTImageProcessorPil (restated) -> fp32 [B, 3, size, size] on the CPU.  Per image: convert to RGB, resize with PIL
    (`resample`) to resize_output_size, float32(uint8 * rescale_factor in float64), (x - mean) / std in float32.  An image whose
    processed size is not size x size raises K2Error (the ViT DPT runs square patch grids only)."""
    from PIL import Image
    if isinstance(images, Image.Image):
        images = [images]
    out = []
    for img in images:
        if img.mode != "RGB":
            img = img.convert("RGB")
        if cfg["do_resize"]:
            nh, nw = resize_output_size(img.size[1], img.size[0], cfg)
            img = img.resize((nw, nh), resample=int(cfg["resample"]))
        if img.size != (size, size):
            raise K2Error(f"DPT preprocessing: the image is processed to {img.size[1]} x {img.size[0]}; only the square "
                          f"{size} x {size} input of this estimator is implemented")
        out.append(rescale_normalize(np.array(img).transpose(2, 0, 1), cfg))
    return torch.stack(out)


def depth_image(predicted, height, width):
    """The depth-estimation pipeline's postprocess of one map: fp32 predicted depth [S', S'] -> PIL "L" image of height x width:
    bicubic resize (align_corners=False), (d - min) / (max - min), * 255, uint8 (truncation), in float32.  A constant map
    gives all zeros (transformers divides by zero there)."""
    from PIL import Image
    d = torch.nn.functional.interpolate(predicted.float().cpu()[None, None], size=(height, width), mode="bicubic",
                                        align_corners=False).squeeze().numpy()
    lo, hi = d.min(), d.max()
    d = np.zeros_like(d) if hi == lo else (d - lo) / (hi - lo)
    return Image.fromarray((d * 255).astype("uint8"))


def make_hint(image, estimator):
    """diffusers' make_hint for kandinsky-2-2-controlnet-depth: the estimator's uint8 depth image of `image`, repeated over three
    channels, / 255 -> float32 [3, H, W] in [0, 1] on the CPU."""
    d = np.array(estimator.depth([image])[0])[:, :, None]
    d = np.concatenate([d, d, d], axis=2)
    return (torch.from_numpy(d).float() / 255.0).permute(2, 0, 1)


def hwc3(x):
    """ControlNet's annotator.util.HWC3: uint8 [H, W] / [H, W, 1 | 3 | 4] -> uint8 [H, W, 3]; grey is repeated, RGBA is
    composited over white in float32, clipped and truncated."""
    if x.dtype != np.uint8:
        raise K2Error(f"midas_hint: images must be uint8, got {x.dtype}")
    if x.ndim == 2:
        x = x[:, :, None]
    C = x.shape[2]
    if C == 3:
        return x
    if C == 1:
        return np.concatenate([x, x, x], axis=2)
    if C == 4:
        color = x[:, :, 0:3].astype(np.float32)
        alpha = x[:, :, 3:4].astype(np.float32) / 255.0
        return (color * alpha + 255.0 * (1.0 - alpha)).clip(0, 255).astype(np.uint8)
    raise K2Error(f"midas_hint: {C}-channel images are not implemented")


def resize_image_size(h, w, resolution):
    """ControlNet's annotator.util.resize_image target size -> (height, width, k): k = resolution / min(h, w), both sides
    scaled by k and rounded to multiples of 64."""
    k = float(resolution) / min(float(h), float(w))
    return int(np.round(h * k / 64.0)) * 64, int(np.round(w * k / 64.0)) * 64, k


def resize_image(img, resolution):
    """ControlNet's annotator.util.resize_image: cv2.resize to resize_image_size with INTER_LANCZOS4 when enlarging (k > 1),
    else INTER_AREA.  An image already at its target size is returned as it is (cv2.resize returns such an image unchanged
    with either flag), and cv2 is imported only when the size changes; a resize without cv2 installed raises K2Error."""
    H, W, k = resize_image_size(img.shape[0], img.shape[1], resolution)
    if (H, W) == img.shape[:2]:
        return img
    try:
        import cv2
    except ImportError as e:
        raise K2Error(f"midas_hint: resizing {img.shape[1]} x {img.shape[0]} to {W} x {H} needs cv2 (opencv-python), which "
                      "is not installed") from e
    return cv2.resize(img, (W, H), interpolation=cv2.INTER_LANCZOS4 if k > 1 else cv2.INTER_AREA)


def midas_pixels(img):
    """MidasDetector's input: uint8 HWC -> fp32 [1, 3, H, W] = float32(u8) / 127.5 - 1 (no resize, no image processor)."""
    return torch.from_numpy(img.astype(np.float32) / np.float32(127.5) - np.float32(1.0)).permute(2, 0, 1)[None].contiguous()


def midas_depth_u8(d):
    """MidasDetector's depth image: fp32 depth [H, W] (numpy) -> d - min, / max, * 255, clip to [0, 255], uint8 (truncation),
    in float32.  A constant map gives zeros (MidasDetector divides by zero there)."""
    d = d.astype(np.float32) - d.min()
    mx = d.max()
    d = np.zeros_like(d) if mx == 0 else d / mx
    return (d * np.float32(255.0)).clip(0, 255).astype(np.uint8)


def midas_hint(image, estimator):
    """The ControlNet notebook's make_hint(img, MidasDetector()), restated from ControlNet's annotator/util.py (HWC3,
    resize_image) and annotator/midas/__init__.py; this restatement is not pinned to that code by a test:
        img = resize_image(HWC3(uint8 image), resolution = its width); depth = estimator's predicted depth of
        float32(img) / 127.5 - 1 at img's size; hint = HWC3(midas_depth_u8(depth)) / 255 -> fp32 [3, H, W] on the CPU.
    image: a PIL image or a uint8 numpy array (HW, HWC).  estimator: a hybrid DPTDepthEstimator (any input size that is a
    multiple of 16; resize_image's multiples of 64 always are).  MidasDetector's normal map is not computed (make_hint
    discards it)."""
    x = np.array(image)
    img = resize_image(hwc3(x), x.shape[1])
    pred = estimator.predicted_depth(midas_pixels(img).to(estimator.device))[0].cpu().numpy()
    d = hwc3(midas_depth_u8(pred))
    return torch.from_numpy(d.copy()).float().div(255.0).permute(2, 0, 1)


def resize_pos_embed(pos, grid):
    """DPTViTEmbeddings._resize_pos_embed in fp32 on the host: pos [1 + G0^2, H] -> [1 + gh gw, H], the grid part resized
    bilinearly (align_corners=False) to grid = (gh, gw), or to a square grid x grid for an integer."""
    gh, gw = (grid, grid) if isinstance(grid, int) else grid
    g0 = int(math.sqrt(pos.shape[0] - 1))
    p = pos[1:].float().reshape(1, g0, g0, -1).permute(0, 3, 1, 2)
    p = torch.nn.functional.interpolate(p, size=(gh, gw), mode="bilinear")
    return torch.cat([pos[:1].float(), p.permute(0, 2, 3, 1).reshape(gh * gw, -1)])


class DPTDepthEstimator(Tower):
    """DPTForDepthEstimation (plain ViT) on this package's kernels.  sd: state dict in this module's names
    (checkpoints.transformers_dpt_to_k2); config: the transformers config.json dict; preprocessor_config: the image
    processor's preprocessor_config.json dict (None: DPTImageProcessorPil's defaults at the model's image_size).  The input
    size is the processor's; the position embedding is resized to its patch grid once, on the host."""

    what = "DPT"

    def __init__(self, sd, config, device="cuda", preprocessor_config=None):
        self.hybrid = bool(config.get("is_hybrid"))
        c = dpt_hybrid_config(config) if self.hybrid else dpt_config(config)
        self.cfg, self.device = c, torch.device(device)
        self.proc = preprocessor_settings(preprocessor_config, c["image_size"])
        S = int(self.proc["size"]["height"])
        if int(self.proc["size"]["width"]) != S or S % c["patch_size"] or S <= 0:
            raise K2Error(f"DPT preprocessing: size {self.proc['size']}: only a square input that is a multiple of the patch "
                          f"size {c['patch_size']} is implemented")
        self.size, self.grid = S, S // c["patch_size"]
        self._take(sd, k2_hybrid_shapes(c) if self.hybrid else k2_shapes(c))

    @classmethod
    def from_transformers(cls, state_dict, config, preprocessor_config=None, device="cuda"):
        """From a transformers DPTForDepthEstimation state dict and its config.json dict (plain or hybrid, after
        `is_hybrid`); packs the weights."""
        from ..checkpoints import transformers_dpt_hybrid_to_k2, transformers_dpt_to_k2
        remap = transformers_dpt_hybrid_to_k2 if config.get("is_hybrid") else transformers_dpt_to_k2
        return cls(remap(state_dict, config), config, device, preprocessor_config).finalize()

    @classmethod
    def from_pretrained(cls, path, device="cuda"):
        """A local transformers model folder (e.g. a download of Intel/dpt-large or Intel/dpt-hybrid-midas): config.json, preprocessor_config.json
        (optional) and model.safetensors or pytorch_model.bin.  A missing file raises K2Error naming it."""
        what = "DPTDepthEstimator.from_pretrained"
        stem = "pytorch_model" if os.path.exists(os.path.join(path, "pytorch_model.bin")) else "model"
        return cls.from_transformers(load_weights(path, (f"{stem}.safetensors", f"{stem}.bin"), what),
                                     read_json(path, "config.json", what),
                                     read_json(path, "preprocessor_config.json", what, required=False), device)

    def _pack(self):
        """fp16 GEMM weights (the patch embedding as pack_patch_embed's [H, Kp]), fp32 biases and LayerNorm parameters, the
        fp16 position embedding at the input's patch grid with the patch convolution's bias folded into the patch rows."""
        c, dev, sd = self.cfg, self.device, self.sd
        F = c["fusion_hidden_size"]
        w = lambda name: ops.pack_conv_weight(sd[name].detach().to(dev))  # noqa: E731
        pk = {"layers": pack_layers(lambda i, name: sd[f"layers.{i}.{name}"], c["backbone_out_indices"][-1] + 1, dev)}
        if self.hybrid:
            pk.update(self._pack_bit())
        else:
            pos = resize_pos_embed(sd["position_embedding"].detach().cpu(), self.grid)
            pos[1:] += sd["patch_embedding.bias"].detach().cpu().float()   # the patch conv's bias, on the patch rows only
            pk.update(embed=pack_patch_embed(sd["patch_embedding.weight"], sd["cls_token"], c["kp"], dev),
                      pos=pos.to(dev).half().contiguous())
        rs = "neck.reassemble_stage."
        for i, (C, f) in enumerate(zip(c["neck_hidden_sizes"], c["reassemble_factors"])):
            pk[f"neck_conv.{i}"] = w(f"neck.convs.{i}.weight")
            fp = f"neck.fusion_stage.layers.{i}."
            pk[f"fusion_proj.{i}"] = (w(fp + "projection.weight"), f32(sd[fp + "projection.bias"], dev))
            for u in ((1, 2) if i else (2,)):
                p = f"{fp}residual_layer{u}."
                c2 = w(p + "convolution2.weight")
                if u == 1:   # + the running map as a 1x1 source with an identity block: running + unit1(stage) in one epilogue
                    eye = torch.zeros(F, c2.shape[1] // 9, dtype=torch.float16, device=dev)
                    eye[:, :F] = torch.eye(F, dtype=torch.float16, device=dev)
                    c2 = torch.cat([c2, eye], 1).contiguous()
                pk[f"unit{u}.{i}"] = ((w(p + "convolution1.weight"), f32(sd[p + "convolution1.bias"], dev)),
                                      (c2, f32(sd[p + "convolution2.bias"], dev)))
            if self.hybrid and i < 2:   # the BiT stage maps go straight into neck.convs.0 / 1
                continue
            pk[f"readout.{i}"] = (w(f"{rs}readout_projects.{i}.0.weight"), f32(sd[f"{rs}readout_projects.{i}.0.bias"], dev))
            pk[f"proj.{i}"] = (w(f"{rs}layers.{i}.projection.weight"), f32(sd[f"{rs}layers.{i}.projection.bias"], dev))
            rw, rb = sd.get(f"{rs}layers.{i}.resize.weight"), sd.get(f"{rs}layers.{i}.resize.bias")
            if f > 1:   # ConvTranspose2d weight [in, out, a, b] -> GEMM rows (a s + b) C + out over K = in
                s = int(f)
                g = rw.detach().to(dev).permute(2, 3, 1, 0).reshape(s * s * C, C)
                pk[f"resize.{i}"] = (ops.pack_conv_weight(g), f32(rb, dev).repeat(s * s))
            elif f < 1:
                pk[f"resize.{i}"] = (ops.pack_conv_weight(rw.detach().to(dev)), f32(rb, dev))
        pk["head"] = [(w("head.head.0.weight"), f32(sd["head.head.0.bias"], dev)),
                      (w("head.head.2.weight"), f32(sd["head.head.2.bias"], dev)),
                      (ops.pad_rows(w("head.head.4.weight"), 16), f32(sd["head.head.4.bias"], dev))]
        return pk

    def _pack_bit(self):
        """The hybrid's backbone: each BiT convolution's weight standardised in float64 and rounded once (the stem's
        [64, 3 * 49] padded to 192 columns for k2_im2col_f16's rows), GroupNorm gamma / beta fp32; the token projection as one
        GEMM weight [H, kp]: the 1x1 projection in columns [0, C3), the CLS token in column C3 (the token rows hold a 1
        there on the CLS row); the position embedding stays on the host (fp32, projection bias on the patch rows) and is
        resized per input size by the plan."""
        c, dev, sd = self.cfg, self.device, self.sd
        b, H = c["bit"], c["hidden_size"]
        ws = lambda name: ops.pack_conv_weight(standardize_weight(sd[name]).to(dev))  # noqa: E731
        gn = lambda name: (f32(sd[name + ".weight"], dev), f32(sd[name + ".bias"], dev))  # noqa: E731
        stem = standardize_weight(sd["bit.embedder.convolution.weight"]).reshape(b["stem"], -1)
        pk = {"stem": (ops.pack_conv_weight(stem.to(dev)), *gn("bit.embedder.norm")), "stages": []}
        for s, depth in enumerate(b["depths"]):
            blocks = []
            for l in range(depth):
                lp = f"bit.encoder.stages.{s}.layers.{l}."
                blk = {f"conv{k}": (ws(f"{lp}conv{k}.weight"), *gn(f"{lp}norm{k}")) for k in (1, 2, 3)}
                if l == 0:
                    blk["down"] = (ws(f"{lp}downsample.conv.weight"), *gn(f"{lp}downsample.norm"))
                blocks.append(blk)
            pk["stages"].append(blocks)
        C3 = b["channels"][2]
        we = torch.zeros(H, c["kp"], dtype=torch.float16, device=dev)
        we[:, :C3] = sd["projection.weight"].detach().to(dev).reshape(H, C3).half()
        we[:, C3] = sd["cls_token"].detach().to(dev).half()
        pk["embed"] = we
        pk["pos_host"] = sd["position_embedding"].detach().cpu().float()
        pk["proj_bias_host"] = sd["projection.bias"].detach().cpu().float()
        return pk

    def _new_plan(self, B, h=None, w=None):
        return _HybridPlan(self, B, h, w) if self.hybrid else _DepthPlan(self, B)

    def attend(self, qkv, out):
        """The layers' attention: k2_attention_d64 over the tokens (per-head [q | k | v], scale 1/8)."""
        return ops.attention_d64(qkv, self.cfg["num_attention_heads"], scale=0.125, out=out)

    def preprocess(self, images):
        """PIL image(s) -> fp32 pixel_values [B, 3, S, S] on the CPU (preprocess_images with this estimator's settings)."""
        return preprocess_images(images, self.proc, self.size)

    @torch.no_grad()
    def predicted_depth(self, pixel_values, use_graph=True):
        """pixel_values fp32 [B, 3, S, S] -> DPTForDepthEstimation's predicted_depth, fp32 [B, S', S'] on the device (S' = S for
        an even patch grid).  The hybrid takes any [B, 3, H, W] with H and W multiples of 16 (one plan per (B, H, W)).  One CUDA graph replay of the batch size's launch plan (use_graph=False: the same launches one
        by one)."""
        S = self.size
        if self.hybrid:
            shp = tuple(pixel_values.shape)
            if pixel_values.dim() != 4 or shp[1] != 3 or shp[2] % 16 or shp[3] % 16 or min(shp[2:]) <= 0:
                raise K2Error(f"DPT-Hybrid: pixel_values must be [B, 3, H, W] with H and W multiples of 16, got {list(shp)}")
            if (shp[2] // 16) % 2 != (shp[3] // 16) % 2:
                raise K2Error(f"DPT-Hybrid: pixel_values {list(shp)}: patch grids with one odd and one even side are not "
                              "implemented")
            plan = self._plan(shp[0], shp[2], shp[3])
        elif pixel_values.dim() != 4 or tuple(pixel_values.shape[1:]) != (3, S, S):
            raise K2Error(f"DPT: pixel_values must be [B, 3, {S}, {S}], got {list(pixel_values.shape)}")
        else:
            plan = self._plan(pixel_values.shape[0])
        plan.pix.copy_(pixel_values)
        plan.run(use_graph)
        return plan.out.clone()

    def depth(self, images):
        """PIL image(s) -> a list of PIL "L" depth images, each of its image's size (depth_image of predicted_depth)."""
        from PIL import Image
        if isinstance(images, Image.Image):
            images = [images]
        pred = self.predicted_depth(self.preprocess(images).to(self.device)).cpu()
        return [depth_image(p, img.size[1], img.size[0]) for p, img in zip(pred, images)]


class _DepthPlan(LaunchPlan):
    """The estimator at B images as one static launch list over fixed buffers (replayed as one CUDA graph); see the module
    docstring.  self.out is predicted_depth, fp32 [B, S', S']."""

    def __init__(self, est, B):
        super().__init__(est.device, B)
        self.e, self.B = est, B
        self.pix = torch.zeros(B, 3, est.size, est.size, device=self.dev, dtype=torch.float32)
        self.pos = est._packed["pos"].expand(B, *est._packed["pos"].shape).contiguous()
        self._build()

    def _conv3(self, x, wb, cout, residual=None, extra=None):
        """3x3 convolution (+ bias) (+ residual) of x fp16 NHWC; extra: a second source read as a 1x1 term."""
        B, Hs, Ws, C = x.shape
        out = self._new(B, Hs, Ws, cout)
        srcs = [(x, 9)] + ([(extra, 1)] if extra is not None else [])
        K = 9 * C + (extra.shape[-1] if extra is not None else 0)
        w, b = wb if isinstance(wb, tuple) else (wb, None)
        self._conv(srcs, w, cout, out, 2 * B * Hs * Ws * K * cout, bias=b, residual=residual, want_stats=False, kind="conv")
        return out

    def _relu(self, x):
        y = self._new(*x.shape)
        self._add(lambda: ops.relu_f16(x, out=y), "relu")
        return y

    def _bilinear(self, x, size, align):
        y = self._new(x.shape[0], size[0], size[1], x.shape[-1])
        self._add(lambda: ops.bilinear_f16(x, size, align, out=y), "bilinear")
        return y

    def _unit(self, x, units, extra=None):
        """DPTPreActResidualLayer: conv3x3(relu(conv3x3(relu(x)))) + x (+ extra through the identity block)."""
        (w1, b1), (w2, b2) = units
        F = w1.shape[0]
        a = self._conv3(self._relu(x), (w1, b1), F)
        self._add(lambda: ops.relu_f16(a), "relu")
        return self._conv3(a, (w2, b2), F, residual=x, extra=extra)

    def _build(self):
        e, pk, B = self.e, self.e._packed, self.B
        c = e.cfg
        G, H, P = e.grid, c["hidden_size"], c["patch_size"]
        T, heads, eps = G * G + 1, c["num_attention_heads"], c["layer_norm_eps"]
        h = record_patch_embed(self, self.pix, pk["embed"], self.pos, P, c["kp"])
        hidden, start = [], 0
        for idx in c["backbone_out_indices"]:
            h = record_layers(self, h, pk["layers"][start:idx + 1], e.attend, 4 * B * heads * T * T * 64, eps)
            hidden.append(h)
            start = idx + 1
        self._fuse_head([self._reassemble(i, hs, (G, G)) for i, hs in enumerate(hidden)])

    def _reassemble(self, i, hs, grid):
        """Neck stage i of the hidden state hs [B, 1 + gh gw, H]: readout, projection, resize, then neck.convs.i."""
        e, pk, B, A = self.e, self.e._packed, self.B, self._add
        c = e.cfg
        (gh, gw), H, F = grid, c["hidden_size"], c["fusion_hidden_size"]
        C, f, M = c["neck_hidden_sizes"][i], c["reassemble_factors"][i], B * gh * gw
        ro, r, p = self._new(B, gh, gw, 2 * H), self._new(B, gh, gw, H), self._new(B, gh, gw, C)
        A(lambda: ops.readout_rows_f16(hs, out=ro.view(B, gh * gw, 2 * H)), "readout")
        self._gemm(ro, pk[f"readout.{i}"][0], H, r, 2 * M * 2 * H * H, bias=pk[f"readout.{i}"][1])
        A(lambda: ops.gelu_f16_(r), "gelu")
        self._gemm(r, pk[f"proj.{i}"][0], C, p, 2 * M * H * C, bias=pk[f"proj.{i}"][1])
        if f > 1:
            s = int(f)
            g, y = self._new(B, gh, gw, s * s * C), self._new(B, s * gh, s * gw, C)
            self._gemm(p, pk[f"resize.{i}"][0], s * s * C, g, 2 * M * C * s * s * C, bias=pk[f"resize.{i}"][1])
            A(lambda: ops.depth_to_space_f16(g, s, C, out=y), "depth_to_space")
        elif f < 1:
            full, Go = self._conv3(p, pk[f"resize.{i}"], C), ((gh + 1) // 2, (gw + 1) // 2)
            if gh % 2 == 0 and gw % 2 == 0:
                y = self._new(B, *Go, C)
                A(lambda: ops.subsample2(full, 0, 0, out=y), "subsample")
            else:   # align_corners from G to (G + 1) / 2 samples: source index 2i exactly, weights 1 and 0
                y = self._bilinear(full, Go, True)
        else:
            y = p
        return self._conv3(y, pk[f"neck_conv.{i}"], F)

    def _fuse_head(self, feats):
        """The fusion stage over the neck maps feats (shallow to deep), then the head -> self.out fp32 [B, S'h, S'w]."""
        pk, B, A, F = self.e._packed, self.B, self._add, self.e.cfg["fusion_hidden_size"]
        run = None
        for j, fe in enumerate(reversed(feats)):   # fusion layer j (its packed weights' key) takes the stage from the deep end
            if run is None:
                x = fe
            else:
                if fe.shape[1:3] != run.shape[1:3]:
                    fe = self._bilinear(fe, tuple(run.shape[1:3]), False)
                x = self._unit(fe, pk[f"unit1.{j}"], extra=run)
            x = self._unit(x, pk[f"unit2.{j}"])
            up = self._bilinear(x, (2 * x.shape[1], 2 * x.shape[2]), True)
            run = self._new(*up.shape)
            wp, bp = pk[f"fusion_proj.{j}"]
            self._gemm(up, wp, F, run, 2 * up.numel() * F, bias=bp)
        (w0, b0), (w2, b2), (w4, b4) = pk["head"]
        a = self._conv3(run, (w0, b0), F // 2)
        a = self._bilinear(a, (2 * a.shape[1], 2 * a.shape[2]), True)
        a = self._conv3(a, (w2, b2), 32)
        A(lambda: ops.relu_f16(a), "relu")
        Sh, Sw = a.shape[1:3]
        out = torch.empty(B, 1, Sh, Sw, device=self.dev, dtype=torch.float32)
        self._conv([(a, 1)], w4, 1, out, 2 * B * Sh * Sw * 32, bias=b4, want_stats=False, out_mode=1, kind="conv")
        A(lambda: ops.relu_f32(out), "relu")
        self.out = out.view(B, Sh, Sw)


class _HybridPlan(_DepthPlan):
    """The hybrid estimator at B images of h x w (multiples of 16) as one static launch list; the neck stages 2 / 3, fusion
    and head are _DepthPlan's.  The BiT backbone:
        stem      k2_im2col_f16 (7x7 stride 2, TF-SAME: 2 before, 3 after on an even side) -> ONE k2_conv_gemm over the
                  [B, h/2, w/2, 192] rows with fused GroupNorm partials -> k2_gn_act_f16 (GN + ReLU) -> k2_maxpool_f16
                  (3x3 stride 2, pads 0 before, 1 after, pad value 0);
        stages    bottlenecks: 1x1 conv -> GN + ReLU -> 3x3 conv -> GN + ReLU -> 1x1 conv -> k2_gn_act_f16(GN + shortcut,
                  ReLU), the shortcut the input or, in a stage's first block, GN(1x1 conv(input)) normalised inside the same
                  launch.  Stride 2 (the first block of stages 2 and 3): the 3x3 convolution at stride 1, pad 1, then
                  k2_subsample2_nhwc(1, 1) (TF-SAME pads 0 before, 1 after on an even side); the 1x1 downsample
                  subsamples (0, 0) first.  GroupNorm statistics come from the convolutions' fused partials
                  (k2_gn_finalize) or a k2_gn_stats pass, as LaunchPlan._stats picks.
    The last stage-3 block writes straight into the token rows [B, 1 + gh gw, kp] (CLS row: a 1 in column C3), and ONE GEMM
    with the [projection | CLS] weight and the resized position embedding (+ projection bias on the patch rows) as its
    residual gives the tokens; then the ViT layers in segments ending at backbone_out_indices[2] and [3]."""

    def __init__(self, est, B, h, w):
        LaunchPlan.__init__(self, est.device, B)
        self.e, self.B, self.h, self.w = est, B, h, w
        self.pix = torch.zeros(B, 3, h, w, device=self.dev, dtype=torch.float32)
        pk, gh, gw = est._packed, h // 16, w // 16
        pos = resize_pos_embed(pk["pos_host"], (gh, gw))
        pos[1:] += pk["proj_bias_host"]
        self.pos = pos.to(self.dev).half().expand(B, *pos.shape).contiguous()
        self._build()

    def _conv1(self, x, wb, cout):
        out = self._new(*x.shape[:3], cout)
        self._conv([(x, 1)], wb[0], cout, out, 2 * x.shape[0] * x.shape[1] * x.shape[2] * x.shape[-1] * cout)
        return out

    def _gn_act(self, x, wb, relu=True, r=None, r_norm=None, out=None):
        st = self._stats(x, None, BIT_GN_EPS)
        y = self._new(*x.shape) if out is None else out
        self._add(lambda: ops.gn_act_f16(x, st, wb[1], wb[2], r=r, r_norm=r_norm, relu=relu, out=y), "gn_act")
        return y

    def _bottleneck(self, x, blk, stride2, out=None):
        mid, cout = blk["conv1"][0].shape[0], blk["conv3"][0].shape[0]
        r, r_norm = x, None
        if "down" in blk:
            xs = x
            if stride2:
                xs = self._new(x.shape[0], x.shape[1] // 2, x.shape[2] // 2, x.shape[3])
                self._add(lambda: ops.subsample2(x, 0, 0, out=xs), "subsample")
            r = self._conv1(xs, blk["down"], cout)
            r_norm = (self._stats(r, None, BIT_GN_EPS), blk["down"][1], blk["down"][2])
        a = self._gn_act(self._conv1(x, blk["conv1"], mid), blk["conv1"])
        B, Hs, Ws, _ = a.shape
        c2 = self._new(B, Hs, Ws, mid)
        self._conv([(a, 9)], blk["conv2"][0], mid, c2, 2 * B * Hs * Ws * 9 * mid * mid, want_stats=not stride2,
                   kind="conv_stride2_at_1" if stride2 else "conv_gemm")
        if stride2:
            full, c2 = c2, self._new(B, Hs // 2, Ws // 2, mid)
            self._add(lambda: ops.subsample2(full, 1, 1, out=c2), "subsample")
        a = self._gn_act(c2, blk["conv2"])
        return self._gn_act(self._conv1(a, blk["conv3"], cout), blk["conv3"], r=r, r_norm=r_norm, out=out)

    def _build(self):
        e, pk, B, A = self.e, self.e._packed, self.B, self._add
        c = e.cfg
        b, H, h, w = c["bit"], c["hidden_size"], self.h, self.w
        gh, gw = h // 16, w // 16
        T, heads, eps = gh * gw + 1, c["num_attention_heads"], c["layer_norm_eps"]
        kst = pk["stem"][0].shape[1]
        rows = self._new(B, h // 2, w // 2, kst)
        A(lambda: ops.im2col_f16(self.pix, 7, 2, (2, 2), (h // 2, w // 2), kst, out=rows), "im2col")
        s0 = self._new(B, h // 2, w // 2, b["stem"])
        self._conv([(rows, 1)], pk["stem"][0], b["stem"], s0, 2 * B * (h // 2) * (w // 2) * 147 * b["stem"], kind="conv")
        a0 = self._gn_act(s0, pk["stem"])
        pooled = self._new(B, h // 4, w // 4, b["stem"])
        A(lambda: ops.maxpool_f16(a0, (0, 0), (h // 4, w // 4), out=pooled), "maxpool")
        # the token rows: the CLS row holds a 1 in column C3, the patch rows' columns >= C3 stay 0; set once here
        C3 = b["channels"][2]
        self.tok_rows = self._new(B, T, c["kp"])
        self.tok_rows.zero_()
        self.tok_rows[:, 0, C3] = 1
        patch_view = self.tok_rows.as_strided((B, gh, gw, C3), (T * c["kp"], gw * c["kp"], c["kp"], 1), c["kp"])
        maps, x = [], pooled
        for s, blocks in enumerate(pk["stages"]):
            for l, blk in enumerate(blocks):
                last = s == 2 and l == len(blocks) - 1
                x = self._bottleneck(x, blk, stride2=(s > 0 and l == 0), out=patch_view if last else None)
            maps.append(x)
        self.bit_maps = maps
        emb = self._new(B, T, H)
        self._gemm(self.tok_rows, pk["embed"], H, emb, 2 * B * T * c["kp"] * H, residual=self.pos)
        idx = c["backbone_out_indices"]
        h1 = record_layers(self, emb, pk["layers"][:idx[2] + 1], e.attend, 4 * B * heads * T * T * 64, eps)
        h2 = record_layers(self, h1, pk["layers"][idx[2] + 1:idx[3] + 1], e.attend, 4 * B * heads * T * T * 64, eps)
        self.vit_hidden = (h1, h2)
        F = c["fusion_hidden_size"]
        feats = [self._conv3(maps[0], pk["neck_conv.0"], F), self._conv3(maps[1], pk["neck_conv.1"], F),
                 self._reassemble(2, h1, (gh, gw)), self._reassemble(3, h2, (gh, gw))]
        self._fuse_head(feats)
