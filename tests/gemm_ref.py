"""Shared by tests/test_gpu_gemm_float64.py, tests/test_gpu_linear_float64.py and tests/test_cpu_gemm_geometry.py: the GEMM
geometry every model builds (derived from the model code and configs, not chosen here), exact integer operands, and the exact
checker.

Exact operands: small integers in fp16 / fp32 (weights of every other output column times a power of two, so that many sums
exceed 2048, where fp16 spacing is 2 and more), integer bias and residual, every partial sum below 2^24 in magnitude.  fp32
accumulation of such operands is exact in any order, on any tile, split or K chunk, so the expected output is the rounding of
the exact float64 sum: fp16_rn for fp16 outputs, the value itself for fp32 outputs.  The check is bit equality."""
import inspect
import math
from dataclasses import dataclass

import torch

EXACT_MAX = 2.0 ** 24   # fp32 represents every integer below this: no accumulation order can round


# ------------------------------------------------------------------------------------------------------------------------------
# exact operands and the exact checker (CPU or GPU)
# ------------------------------------------------------------------------------------------------------------------------------
def ints(g, shape, lim=4, device="cpu", dtype=torch.float16):
    """Uniform integers in [-lim, lim]."""
    return torch.randint(-lim, lim + 1, tuple(shape), generator=g, device=device).to(dtype)


def exact_scale(k_terms):
    """Power of two for the weights of every other output column: sums of k_terms products of [-4, 4] x [-4, 4] (std
    6.7 sqrt(k)) then reach a std of about 1500, so a good share of them lies above 2048."""
    return 2.0 ** max(0, round(math.log2(1500.0 / (6.67 * math.sqrt(k_terms)))))


def scale_odd_rows(w, s):
    """w [N, ...] with rows 1, 3, 5, ... multiplied by s (exact: s is a power of two and |w| s stays small)."""
    w = w.clone()
    w[1::2] *= s
    return w


def exact_expected(acc64, out_dtype):
    """The rounding of an exact float64 result to the kernel's output type; refuses a result fp32 cannot hold exactly."""
    big = acc64.abs().max().item() if acc64.numel() else 0.0
    assert big < EXACT_MAX, f"exact-operand sum {big} is not below 2^24: fp32 accumulation would not be exact"
    out = acc64.float()
    if out_dtype == torch.float16:
        assert big < 65504, f"exact-operand result {big} overflows fp16"
        out = out.half()
    return out


def check_exact(y, want, what):
    """Bit equality of y and want (fp16 or fp32, any shape); the message names the first differing element."""
    assert y.shape == want.shape and y.dtype == want.dtype, (what, y.shape, want.shape, y.dtype, want.dtype)
    it = torch.int16 if y.dtype == torch.float16 else torch.int32
    yb, wb = y.contiguous().view(it), want.contiguous().view(it)
    if torch.equal(yb, wb):
        return
    bad = (yb != wb).nonzero()
    i = tuple(bad[0].tolist())
    raise AssertionError(f"{what}: {bad.shape[0]} of {y.numel()} elements differ from the exact result; first at {i}: "
                         f"got {y[i].item()!r}, want {want[i].item()!r}")


# ------------------------------------------------------------------------------------------------------------------------------
# geometry, derived from the model code and configs
# ------------------------------------------------------------------------------------------------------------------------------
@dataclass(frozen=True)
class Gemm:
    """One k2_conv_gemm launch of a model.  geom = output (NB, H, W) (a flat-row GEMM: (1, 1, M)); srcs = ((C, taps), ...);
    rows: launched through ops.gemm_rows; stem = (Cx, C2, C3, mul23): the single source is k2_stem_im2col's patch rows of
    cat(x, x2 (* x3), x3) with C = Kpad; w_rows: packed weight rows (0 = cout, 16 for the padded output heads)."""
    name: str
    geom: tuple
    srcs: tuple
    cout: int
    residual: bool = False
    out_mode: int = 0
    w_rows: int = 0
    rows: bool = False
    stem: tuple = None

    @property
    def ktot(self):
        return sum(t * ((c + 63) // 64 * 64) for c, t in self.srcs)

    @property
    def k_terms(self):
        """Products per output element (zero padding excluded)."""
        if self.stem:
            return 9 * sum(self.stem[:3])
        return sum(t * c for c, t in self.srcs)

    @property
    def m(self):
        return self.geom[0] * self.geom[1] * self.geom[2]


TOWER_ROWS = (1, 2, 8)
_RESIDUAL = ("attn.proj", "mlp.fc2")   # encoder.record_layers: the out-proj and fc2 GEMMs add the residual stream


def _layer_gemms(tower, H, I, T):
    from kandinsky2.model.encoder import layer_shapes
    out = []
    for name, shape in layer_shapes(H, I).items():
        if name.endswith(".weight") and len(shape) == 2:
            layer = name[:-len(".weight")]
            for r in TOWER_ROWS:
                out.append(Gemm(f"{tower}:{layer}:rows{r}", (1, 1, r * T), ((shape[1], 1),), shape[0],
                                residual=layer in _RESIDUAL, rows=True))
    return out


def _prior_meta(cfg):
    from kandinsky2.model.prior import PriorTransformer
    return PriorTransformer(**dict(cfg, xf_layers=1), device="meta")


def tower_gemms():
    """The transformer towers' Linear layers as flat-row GEMMs at rows x tokens output rows, rows in TOWER_ROWS."""
    from kandinsky2.model.clip_text import text_tower_config
    from kandinsky2.model.clip_vision import tower_config
    from kandinsky2.model.text_encoders import XLMRobertaTokenizer, xlmr_config
    from oracle.prior_oracle import CONFIG_PRIOR
    from tests import clip_text_oracle, clip_vision_oracle, xlmr_oracle
    from tests.prior22_oracle import CONFIG_PRIOR22
    out = []
    for ver, cfg in (("2.1", CONFIG_PRIOR), ("2.2", CONFIG_PRIOR22)):
        p = _prior_meta(cfg)
        T = p.text_ctx + p.ext_len
        blk = p.transformer.resblocks[0]
        if ver == "2.1":   # the 2.2 prior's layers have the same shapes
            out += _layer_gemms("prior", p.xf_width, blk.mlp.c_fc.weight.shape[0], T)
        n, k = p.text_enc_proj.weight.shape
        out += [Gemm(f"prior{ver}:text_enc_proj:rows{r}", (1, 1, r * p.text_ctx), ((k, 1),), n, rows=True) for r in TOWER_ROWS]
    c = text_tower_config(clip_text_oracle.CONFIG_BIGG)
    out += _layer_gemms("clip_text", c["hidden_size"], c["intermediate_size"], c["max_position_embeddings"])
    c = tower_config(clip_vision_oracle.CONFIG_BIGG)
    out += _layer_gemms("clip_vision", c["hidden_size"], c["intermediate_size"], c["tokens"])
    out += [Gemm(f"clip_vision:patch_embed:rows{r}", (1, 1, r * c["tokens"]), ((c["kp"], 1),), c["hidden_size"],
                 residual=True, rows=True) for r in TOWER_ROWS]
    c = xlmr_config(xlmr_oracle.CONFIG_LARGE)
    T = inspect.signature(XLMRobertaTokenizer).parameters["model_max_length"].default
    out += _layer_gemms("xlmr", c["hidden_size"], c["intermediate_size"], T)
    return out


UNET_GEOM = (8, 96, 96)    # bench.py's cfg-2: UNet batch 8 (4 images under CFG) at a 96 x 96 latent
MOVQ_LATENT = (2, 96, 96)  # two images decoded from 96 x 96 latents (768 x 768 pixels)
HINT_ROWS = 2              # the ControlNet hint stem runs once per generation on the CFG rows of one image


def unet_gemms():
    """Each attention level's qkv and encoder_kv GEMMs (flat rows; 2.1 and 2.2 encoder-token counts) and proj_out + residual
    (a 1x1 conv over the level's NHWC geometry)."""
    import bench
    from tests.test_gpu_attention_float64 import _encoder_tokens, _unet_attention_levels
    N, h, w = UNET_GEOM
    md = bench.UNET_CFG["model_dim"]
    out = []
    for ds, heads in _unet_attention_levels():
        C, hh, ww = 64 * heads, h // ds, w // ds
        out.append(Gemm(f"unet:qkv:ds{ds}", (1, 1, N * hh * ww), ((C, 1),), 3 * C, rows=True))
        for ver, tc in sorted(_encoder_tokens().items()):
            out.append(Gemm(f"unet:encoder_kv{ver}:ds{ds}", (1, 1, N * tc), ((md, 1),), 2 * C, rows=True))
        out.append(Gemm(f"unet:proj_out:ds{ds}", (N, hh, ww), ((C, 1),), C, residual=True))
    return out


def _movq_dd():
    from kandinsky2 import configs
    return configs.CONFIG_2_2["image_enc_params"]["params"]["ddconfig"]


def movq_gemms():
    """The AttnBlock's qkv GEMM and proj + residual at the latent, and the ResBlock whose nin_shortcut runs as a second K
    segment (3x3 of h + 1x1 of x) at the smallest image size with a channel change."""
    from kandinsky2.vqgan.autoencoder import _enc_topology, _topology
    from tests.test_gpu_attention_float64 import _movq_attention
    dd = _movq_dd()
    B, h, w = MOVQ_LATENT
    out = []
    for T, C in sorted(_movq_attention(dd, h, w)):
        if T != h * w:   # an attention block above the latent scale: same GEMM widths, more rows
            continue
        out.append(Gemm(f"movq:qkv:T{T}", (1, 1, B * T), ((C, 1),), 3 * C, rows=True))
        out.append(Gemm(f"movq:proj:T{T}", (B, h, w), ((C, 1),), C, residual=True))
    changes = []   # (pixels, name, cin, cout, size)
    _, levels = _topology(dd)
    s = 1
    for lv in levels:
        changes += [(s * s, "decoder", ci, co, s) for ci, co in lv["blocks"] if ci != co]
        s *= 2 if lv["up"] else 1
    elv = _enc_topology(dd)
    s = 2 ** (len(elv) - 1)
    for lv in elv:
        changes += [(s * s, "encoder", ci, co, s) for ci, co in lv["blocks"] if ci != co]
        s //= 2 if lv["down"] else 1
    _, where, ci, co, s = min(changes)
    out.append(Gemm(f"movq:{where}_resblock_nin:{ci}to{co}", (B, h * s, w * s), ((co, 9), (ci, 1)), co))
    return out


def _hint_convs():
    """[(index, Cin, Cout, output size)] of the ControlNet hint stem's convolutions (stride-2 ones run as 'same' convs)."""
    from kandinsky2.model.unet import _HINT_STEM
    _, h, _ = UNET_GEOM
    size, out = 8 * h, []
    for i, (ci, co, stride) in enumerate(_HINT_STEM):
        out.append((i, ci, co, size))
        size //= stride
    return out


def head_gemms():
    """The fp32 NCHW output heads (out_mode 1; packed weight rows padded to 16): UNet out, MoVQ decoder and encoder conv_out,
    the hint stem's last conv."""
    import bench
    from kandinsky2.model.unet import _topology as unet_topology
    from kandinsky2.vqgan.autoencoder import _enc_topology
    cfg = bench.UNET_CFG
    inp, _, _ = unet_topology(cfg["in_channels"], cfg["model_channels"], tuple(cfg["channel_mult"]), cfg["num_res_blocks"],
                              tuple(cfg["attention_resolutions"]))
    dd = _movq_dd()
    B, h, w = MOVQ_LATENT
    s = 2 ** (len(dd["ch_mult"]) - 1)
    zc = dd["z_channels"] * (2 if dd["double_z"] else 1)
    i, ci, co, size = _hint_convs()[-1]
    return [Gemm("unet:out", UNET_GEOM, ((inp[0][0][2], 9),), cfg["out_channels"], out_mode=1, w_rows=16),
            Gemm("movq:decoder_conv_out", (B, h * s, w * s), ((dd["ch"] * dd["ch_mult"][0], 9),), dd["out_ch"], out_mode=1,
                 w_rows=16),
            Gemm("movq:encoder_conv_out", (B, h, w), ((dd["ch"] * dd["ch_mult"][-1], 9),), zc, out_mode=1, w_rows=16),
            Gemm(f"hint:conv{i}", (HINT_ROWS, size, size), ((ci, 9),), co, out_mode=1, w_rows=16)]


def generic_epilogue_gemms():
    """Launches whose output width takes the per-row fallback of the epilogue: the hint stem's 3x3 convs with Cout % 64 != 0
    (the first one is a stem, in stem_gemms), and split-K with Cout % 32 != 0 (no model layer has it: an ABI edge)."""
    out = [Gemm(f"hint:conv{i}", (HINT_ROWS, size, size), ((ci, 9),), co, w_rows=16)
           for i, ci, co, size in _hint_convs()[1:-1] if co % 64]
    out += [Gemm(f"abi:splitk_cout{n}", (1, 1, 1000), ((2048, 1),), n, residual=True, rows=True) for n in (72, 200)]
    return out


def stem_gemms():
    """k2_stem_im2col + GEMM at each call site: the UNet (plain, inpainting, ControlNet), the hint stem's first conv and the
    MoVQ decoder / encoder conv_in."""
    import bench
    from kandinsky2.model.unet import _topology as unet_topology
    cfg = bench.UNET_CFG
    lat = cfg["in_channels"]
    co = unet_topology(lat, cfg["model_channels"], tuple(cfg["channel_mult"]), cfg["num_res_blocks"],
                       tuple(cfg["attention_resolutions"]))[0][0][0][2]
    dd = _movq_dd()
    B, h, w = MOVQ_LATENT
    s = 2 ** (len(dd["ch_mult"]) - 1)
    i, ci, hco, size = _hint_convs()[0]
    sites = [("unet", UNET_GEOM, (lat, 0, 0, 0), co),
             ("unet_inpaint", UNET_GEOM, (lat, lat, 1, 1), co),           # cat(x, image * mask, mask): InpaintText2ImUNet
             ("unet_controlnet", UNET_GEOM, (lat, 4, 0, 0), co),          # cat(x, 4 hint feature channels)
             (f"hint:conv{i}", (HINT_ROWS, size, size), (ci, 0, 0, 0), hco),
             ("movq:decoder_conv_in", (B, h, w), (dd["z_channels"], 0, 0, 0), dd["ch"] * dd["ch_mult"][-1]),
             ("movq:encoder_conv_in", (B, h * s, w * s), (dd["in_channels"], 0, 0, 0), dd["ch"])]
    out = []
    for name, geom, st, cout in sites:
        kpad = (9 * sum(st[:3]) + 63) // 64 * 64
        out.append(Gemm(f"stem:{name}", geom, ((kpad, 1),), cout, stem=st, w_rows=16 if cout < 16 else 0))
    return out


def all_gemms():
    return tower_gemms() + unet_gemms() + movq_gemms() + head_gemms() + generic_epilogue_gemms() + stem_gemms()


def film_total():
    """Output width of the UNet's FiLM linear (all emb_layers of bench.py's UNet as one weight): 2 Cout per ResBlock."""
    import bench
    from kandinsky2.model.unet import _topology
    cfg = bench.UNET_CFG
    inp, mid, out = _topology(cfg["in_channels"], cfg["model_channels"], tuple(cfg["channel_mult"]), cfg["num_res_blocks"],
                              tuple(cfg["attention_resolutions"]))
    layers = [x for blk in inp for x in blk] + list(mid) + [x for blk in out for x in blk]
    return sum(2 * x[2] for x in layers if x[0] == "res")
