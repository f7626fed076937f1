"""H100-native MOVQ: `decode` (latents -> image) through the C-ABI kernels; reference module boundary.

Drop-in for kandinsky2/vqgan/autoencoder.py:160-201 (class MOVQ; ctor (ddconfig, n_embed, embed_dim); decode :182-185)
with the decoder of kandinsky2/vqgan/movq_modules.py:228-357.  state_dict keys/shapes equal the reference's for
`decoder.*`, `post_quant_conv.*` and `quantize.embedding.weight` (the encoder / quant_conv halves of a reference
checkpoint are accepted and ignored: the image->latent direction is SURVEY.md 8f rank 1, not on this path).

decode / encode at a fixed geometry are static launch plans (kandinsky2/launch_plan.py) over pre-allocated buffers, replayed as
ONE CUDA graph; nothing loops over images on the host.  Kernel program (activations NHWC fp16, fp32 accumulate):
  SpatialNorm + swish      statistics from partial sums the producing conv's epilogue wrote (k2_gn_finalize, no read of the
                           tensor) + k2_sn_apply: GroupNorm and the two 4 -> C latent modulations folded into 10 coefficients
                           per channel held in registers (movq_modules.py:61-68: no conv_y / conv_b tensors, no interpolate)
  conv3x3 / nin_shortcut   k2_conv_gemm (shortcut folded in as extra K segment / epilogue residual)
  AttnBlock (1 head, d=C)  q,k,v in one GEMM; scores = q k^T as ONE batched GEMM (image n's k rows are its B operand);
                           row softmax in place; P V as one batched GEMM against the transposed values; proj GEMM + residual
                           (movq_modules.py:201-225)
  Upsample                 no upsampled tensor: conv3x3(nearest_2x(h)) = four 2x2 phase convolutions over h itself
                           (k2_conv_gemm taps = 4, 2.25x fewer MACs; movq_modules.py:93-97)
"""
import os

import torch
import torch.nn as nn

from .. import ops
from .._native import K2Error
from ..launch_plan import LaunchPlan


# MoVQ AttnBlock (one head, C = 512): fused flash-attention kernel (k2_attention_d512) instead of two batched GEMMs around a
# materialised [T, T] score matrix
_FUSED_ATTN = os.environ.get("K2_MOVQ_FUSED_ATTN", "1") != "0"


class _Node(nn.Module):
    pass


def _enc_topology(dd):
    ch, mult, nrb = dd["ch"], tuple(dd["ch_mult"]), dd["num_res_blocks"]
    curr = dd["resolution"]
    in_mult = (1,) + mult
    levels = []
    for i in range(len(mult)):
        bi, bo = ch * in_mult[i], ch * mult[i]
        blocks = []
        for _ in range(nrb):
            blocks.append((bi, bo))
            bi = bo
        levels.append(dict(level=i, blocks=blocks, attn=curr in tuple(dd["attn_resolutions"]), down=i != len(mult) - 1, ch=bo))
        if i != len(mult) - 1:
            curr //= 2
    return levels


def _topology(dd):
    ch, mult, nrb = dd["ch"], tuple(dd["ch_mult"]), dd["num_res_blocks"]
    nres = len(mult)
    block_in = ch * mult[-1]
    curr = dd["resolution"] // 2 ** (nres - 1)
    levels, bi = [], block_in
    for lvl in reversed(range(nres)):
        bo = ch * mult[lvl]
        blocks = []
        for _ in range(nrb + 1):
            blocks.append((bi, bo))
            bi = bo
        levels.append(dict(level=lvl, blocks=blocks, attn=curr in tuple(dd["attn_resolutions"]), up=lvl != 0, ch=bo))
        if lvl != 0:
            curr *= 2
    return block_in, levels


class MOVQ(nn.Module):
    def __init__(self, ddconfig, n_embed, embed_dim, device=None, param_dtype=torch.float32):
        super().__init__()
        self.ddconfig = dict(ddconfig)
        self.n_embed, self.embed_dim = n_embed, embed_dim
        self._packed = None
        self._plans = {}
        self.use_cuda_graph = True
        dd = self.ddconfig
        kw = dict(device=device, dtype=param_dtype)
        zc = embed_dim

        def P(path, *shape):
            node = self
            parts = path.split(".")
            for name in parts[:-1]:
                if name not in node._modules:
                    node.add_module(name, _Node())
                node = node._modules[name]
            node.register_parameter(parts[-1], nn.Parameter(torch.zeros(*shape, **kw), requires_grad=False))

        def SN(p, c):
            P(p + "norm_layer.weight", c); P(p + "norm_layer.bias", c)
            P(p + "conv_y.weight", c, zc, 1, 1); P(p + "conv_y.bias", c)
            P(p + "conv_b.weight", c, zc, 1, 1); P(p + "conv_b.bias", c)

        def RES(p, cin, cout):
            SN(p + "norm1.", cin)
            P(p + "conv1.weight", cout, cin, 3, 3); P(p + "conv1.bias", cout)
            SN(p + "norm2.", cout)
            P(p + "conv2.weight", cout, cout, 3, 3); P(p + "conv2.bias", cout)
            if cin != cout:
                P(p + "nin_shortcut.weight", cout, cin, 1, 1); P(p + "nin_shortcut.bias", cout)

        def ATT(p, c):
            SN(p + "norm.", c)
            for n in ("q", "k", "v", "proj_out"):
                P(p + n + ".weight", c, c, 1, 1); P(p + n + ".bias", c)

        # ---- encoder (image -> latent; vqgan_blocks.py:253-367) -- plain GroupNorm(32, eps 1e-6), no SpatialNorm
        def ERES(p, cin, cout):
            P(p + "norm1.weight", cin); P(p + "norm1.bias", cin)
            P(p + "conv1.weight", cout, cin, 3, 3); P(p + "conv1.bias", cout)
            P(p + "norm2.weight", cout); P(p + "norm2.bias", cout)
            P(p + "conv2.weight", cout, cout, 3, 3); P(p + "conv2.bias", cout)
            if cin != cout:
                P(p + "nin_shortcut.weight", cout, cin, 1, 1); P(p + "nin_shortcut.bias", cout)

        def EATT(p, c):
            P(p + "norm.weight", c); P(p + "norm.bias", c)
            for n in ("q", "k", "v", "proj_out"):
                P(p + n + ".weight", c, c, 1, 1); P(p + n + ".bias", c)

        self.enc_levels = _enc_topology(dd)
        P("encoder.conv_in.weight", dd["ch"], dd["in_channels"], 3, 3); P("encoder.conv_in.bias", dd["ch"])
        for lv in self.enc_levels:
            p = f"encoder.down.{lv['level']}."
            for bi, (cin, cout) in enumerate(lv["blocks"]):
                ERES(p + f"block.{bi}.", cin, cout)
            if lv["attn"]:
                for bi in range(len(lv["blocks"])):
                    EATT(p + f"attn.{bi}.", lv["ch"])
            if lv["down"]:
                P(p + "downsample.conv.weight", lv["ch"], lv["ch"], 3, 3); P(p + "downsample.conv.bias", lv["ch"])
        ce = self.enc_levels[-1]["ch"]
        ERES("encoder.mid.block_1.", ce, ce)
        EATT("encoder.mid.attn_1.", ce)
        ERES("encoder.mid.block_2.", ce, ce)
        zc_out = dd["z_channels"] * (2 if dd.get("double_z") else 1)
        P("encoder.norm_out.weight", ce); P("encoder.norm_out.bias", ce)
        P("encoder.conv_out.weight", zc_out, ce, 3, 3); P("encoder.conv_out.bias", zc_out)

        self.block_in, self.levels = _topology(dd)
        P("decoder.conv_in.weight", self.block_in, dd["z_channels"], 3, 3); P("decoder.conv_in.bias", self.block_in)
        RES("decoder.mid.block_1.", self.block_in, self.block_in)
        ATT("decoder.mid.attn_1.", self.block_in)
        RES("decoder.mid.block_2.", self.block_in, self.block_in)
        for lv in sorted(self.levels, key=lambda l: l["level"]):
            p = f"decoder.up.{lv['level']}."
            for bi, (cin, cout) in enumerate(lv["blocks"]):
                RES(p + f"block.{bi}.", cin, cout)
            if lv["attn"]:
                for bi in range(len(lv["blocks"])):
                    ATT(p + f"attn.{bi}.", lv["ch"])
            if lv["up"]:
                P(p + "upsample.conv.weight", lv["ch"], lv["ch"], 3, 3); P(p + "upsample.conv.bias", lv["ch"])
        c_last = self.levels[-1]["ch"]
        SN("decoder.norm_out.", c_last)
        P("decoder.conv_out.weight", dd["out_ch"], c_last, 3, 3); P("decoder.conv_out.bias", dd["out_ch"])
        P("quantize.embedding.weight", n_embed, embed_dim)
        P("quant_conv.weight", embed_dim, dd["z_channels"], 1, 1); P("quant_conv.bias", embed_dim)
        P("post_quant_conv.weight", dd["z_channels"], embed_dim, 1, 1); P("post_quant_conv.bias", dd["z_channels"])

    # ------------------------------------------------------------------------------------------
    def load_state_dict(self, state_dict, strict=True, assign=False):
        """Same keys as the reference's MOVQ (autoencoder.py:167-174); training-only `loss.*` entries are dropped."""
        sd = {k: v for k, v in state_dict.items() if not k.startswith("loss.")}
        self._packed, self._plans = None, {}
        return super().load_state_dict(sd, strict=strict, assign=assign)

    @classmethod
    def from_diffusers(cls, state_dict, config, device="cuda", param_dtype=torch.float16):
        """From a diffusers `VQModel` state dict and its config.json dict (norm_type "spatial": the Kandinsky 2.2 decoder
        folders' `movq/`), through diffusers_compat.movq_config and checkpoints.diffusers_movq_to_k2; the weights are cast to
        param_dtype (fp16, the dtype the 2.2 pipelines load the MoVQ in).  The 2.2 pipelines' movq.decode(latents,
        force_not_quantize=True) is decode here, and movq.encode(x).latents is encode."""
        from ..checkpoints import diffusers_movq_to_k2
        from ..diffusers_compat import movq_config
        dd, n_embed, embed_dim = movq_config(config)
        m = cls(dd, n_embed, embed_dim, device=device, param_dtype=param_dtype)
        m.load_state_dict(diffusers_movq_to_k2(state_dict, dd))
        return m

    @classmethod
    def from_pretrained(cls, path, device="cuda", param_dtype=torch.float16):
        """A local diffusers `VQModel` folder (e.g. the `movq/` of kandinsky-2-2-decoder): config.json and
        diffusion_pytorch_model{,.fp16}.{safetensors,bin}.  A missing file raises K2Error naming it."""
        from ..checkpoints import load_weights, read_json
        from ..diffusers_compat import WEIGHT_FILES
        what = "MOVQ.from_pretrained"
        config = read_json(path, "config.json", what)
        return cls.from_diffusers(load_weights(path, WEIGHT_FILES, what), config, device, param_dtype)

    def _apply(self, fn, recurse=True):
        self._packed, self._plans = None, {}
        return super()._apply(fn, recurse)

    @torch.no_grad()
    def init_synthetic_(self, seed=0):
        dev = self._get("post_quant_conv.weight").device
        g = torch.Generator(device=dev).manual_seed(seed)
        for name, prm in self.named_parameters():
            if name.endswith("bias"):
                prm.normal_(0.0, 0.05, generator=g)
            elif prm.dim() == 1:
                prm.normal_(0.0, 0.1, generator=g).add_(1.0)
            elif name == "quantize.embedding.weight":
                prm.normal_(0.0, 1.0, generator=g)
            else:
                prm.normal_(0.0, prm[0].numel() ** -0.5, generator=g)
        self._packed, self._plans = None, {}
        return self

    def _get(self, key):
        node = self
        for name in key.split("."):
            node = node._modules[name] if name in node._modules else node._parameters[name]
        return node

    def finalize(self):
        dev = self._get("post_quant_conv.weight").device
        if dev.type != "cuda":
            raise K2Error("MOVQ must live on a CUDA sm_90 device; there is no CPU path")
        f32 = lambda k: self._get(k).detach().to(torch.float32).contiguous()
        pk = {}

        def sn(p):
            c = self._get(p + "norm_layer.weight").shape[0]
            w = torch.cat([f32(p + "conv_y.weight").reshape(c, -1), f32(p + "conv_y.bias")[:, None],
                           f32(p + "conv_b.weight").reshape(c, -1), f32(p + "conv_b.bias")[:, None]], 1).contiguous()
            return dict(g=f32(p + "norm_layer.weight"), b=f32(p + "norm_layer.bias"), w=w)

        def res(p, cin, cout):
            d = dict(n1=sn(p + "norm1."), n2=sn(p + "norm2."), w1=ops.pack_conv_weight(self._get(p + "conv1.weight")),
                     c1=f32(p + "conv1.bias"), c2=f32(p + "conv2.bias"))
            w2 = ops.pack_conv_weight(self._get(p + "conv2.weight"))
            if cin != cout:
                w2 = torch.cat([w2, ops.pack_conv_weight(self._get(p + "nin_shortcut.weight"))], 1).contiguous()
                d["c2"] = d["c2"] + f32(p + "nin_shortcut.bias")
            d["w2"] = w2
            return d

        def att_common(p):
            pc = ops.pack_conv_weight
            return dict(wqkv=torch.cat([pc(self._get(p + n + ".weight")) for n in ("q", "k", "v")], 0).contiguous(),
                        bqkv=torch.cat([f32(p + n + ".bias") for n in ("q", "k", "v")]).contiguous(),
                        wp=pc(self._get(p + "proj_out.weight")), bp=f32(p + "proj_out.bias"))

        def att(p):
            d = att_common(p)
            d["n"] = sn(p + "norm.")
            return d

        pk["pq_w"] = f32("post_quant_conv.weight").reshape(self.ddconfig["z_channels"], self.embed_dim).contiguous()
        pk["pq_b"] = f32("post_quant_conv.bias")
        pk["in_w"] = ops.pack_stem_weight(self._get("decoder.conv_in.weight"))
        pk["in_b"] = f32("decoder.conv_in.bias")
        pk["mid1"] = res("decoder.mid.block_1.", self.block_in, self.block_in)
        pk["mida"] = att("decoder.mid.attn_1.")
        pk["mid2"] = res("decoder.mid.block_2.", self.block_in, self.block_in)
        for lv in self.levels:
            p = f"decoder.up.{lv['level']}."
            for bi, (cin, cout) in enumerate(lv["blocks"]):
                pk[p + f"block.{bi}"] = res(p + f"block.{bi}.", cin, cout)
                if lv["attn"]:
                    pk[p + f"attn.{bi}"] = att(p + f"attn.{bi}.")
            if lv["up"]:
                pk[p + "up_w"] = ops.pack_conv_weight_up2(self._get(p + "upsample.conv.weight"))
                pk[p + "up_b"] = f32(p + "upsample.conv.bias")
        # ---- encoder
        def gn(p):
            return dict(g=f32(p + "weight"), b=f32(p + "bias"))

        def eres(p, cin, cout):
            d = dict(n1=gn(p + "norm1."), n2=gn(p + "norm2."), w1=ops.pack_conv_weight(self._get(p + "conv1.weight")),
                     c1=f32(p + "conv1.bias"), c2=f32(p + "conv2.bias"))
            w2 = ops.pack_conv_weight(self._get(p + "conv2.weight"))
            if cin != cout:
                w2 = torch.cat([w2, ops.pack_conv_weight(self._get(p + "nin_shortcut.weight"))], 1).contiguous()
                d["c2"] = d["c2"] + f32(p + "nin_shortcut.bias")
            d["w2"] = w2
            return d

        def eatt(p):
            d = att_common(p)
            d["n"] = gn(p + "norm.")
            return d

        pk["e_in_w"] = ops.pack_stem_weight(self._get("encoder.conv_in.weight"))
        pk["e_in_b"] = f32("encoder.conv_in.bias")
        for lv in self.enc_levels:
            p = f"encoder.down.{lv['level']}."
            for bi, (cin, cout) in enumerate(lv["blocks"]):
                pk[p + f"block.{bi}"] = eres(p + f"block.{bi}.", cin, cout)
                if lv["attn"]:
                    pk[p + f"attn.{bi}"] = eatt(p + f"attn.{bi}.")
            if lv["down"]:
                pk[p + "down_w"] = ops.pack_conv_weight(self._get(p + "downsample.conv.weight"))
                pk[p + "down_b"] = f32(p + "downsample.conv.bias")
        ce = self.enc_levels[-1]["ch"]
        pk["e_mid1"] = eres("encoder.mid.block_1.", ce, ce)
        pk["e_mida"] = eatt("encoder.mid.attn_1.")
        pk["e_mid2"] = eres("encoder.mid.block_2.", ce, ce)
        pk["e_out_n"] = gn("encoder.norm_out.")
        pk["e_out_w"] = ops.pad_rows(ops.pack_conv_weight(self._get("encoder.conv_out.weight")), 16)
        pk["e_out_b"] = f32("encoder.conv_out.bias")
        pk["qc_w"] = f32("quant_conv.weight").reshape(self.embed_dim, -1).contiguous()
        pk["qc_b"] = f32("quant_conv.bias")
        pk["out_n"] = sn("decoder.norm_out.")
        pk["out_w"] = ops.pad_rows(ops.pack_conv_weight(self._get("decoder.conv_out.weight")), 16)
        pk["out_b"] = f32("decoder.conv_out.bias")
        pk["codebook"] = f32("quantize.embedding.weight")
        self._packed = pk
        self._plans = {}
        return self

    # ------------------------------------------------------------------------------------------
    def _plan(self, mode, B, H, W):
        if self._packed is None:
            self.finalize()
        key = (mode, B, H, W)
        if key not in self._plans:
            self._plans[key] = _MovqPlan(self, mode, B, H, W)
        return self._plans[key]

    @torch.no_grad()
    def decode(self, quant, out_dtype=None):
        """quant [B, z_channels, h, w] -> image [B, out_ch, H, W] (autoencoder.py:182-185). Output dtype follows
        the input (the reference decodes in fp16 when the pipeline is fp16) unless out_dtype is given."""
        if not quant.is_cuda:
            raise K2Error("k2b200 MOVQ.decode: input must be a CUDA tensor (no CPU fallback)")
        plan = self._plan("decode", quant.shape[0], quant.shape[2], quant.shape[3])
        plan.x_in.copy_(quant)
        plan.run(self.use_cuda_graph)
        dt = out_dtype or (quant.dtype if quant.is_floating_point() else torch.float32)
        return plan.out.clone() if dt == torch.float32 else plan.out.to(dt)

    @torch.no_grad()
    def encode(self, x):
        """image [B, 3, H, W] in [-1, 1] -> latent fp32 [B, embed_dim, H/8, W/8], no quantisation (autoencoder.py:176-180:
        quant_conv(Encoder(x))).  The stride-2 Downsample conv (pad (0,1,0,1), vqgan_blocks.py:109-126) is evaluated as
        the stride-1 'same' conv on tensor cores followed by taking the odd pixels."""
        if not x.is_cuda:
            raise K2Error("k2b200 MOVQ.encode: input must be a CUDA tensor (no CPU fallback)")
        plan = self._plan("encode", x.shape[0], x.shape[2], x.shape[3])
        plan.x_in.copy_(x)
        plan.run(self.use_cuda_graph)
        return plan.out.clone()

    @torch.no_grad()
    def decode_to_uint8(self, quant, crop_h=None, crop_w=None):
        """decode + process_images (kandinsky2/utils.py:57-70) fused on the device -> uint8 NHWC (cropped)."""
        if not quant.is_cuda:
            raise K2Error("k2b200 MOVQ.decode: input must be a CUDA tensor (no CPU fallback)")
        plan = self._plan("decode", quant.shape[0], quant.shape[2], quant.shape[3])
        plan.x_in.copy_(quant)
        plan.run(self.use_cuda_graph)
        return ops.images_to_u8(plan.out, crop_h or plan.out.shape[2], crop_w or plan.out.shape[3])

    @torch.no_grad()
    def quantize_indices(self, z):
        """Nearest-codebook indices of z [B, e_dim, h, w] (quntize.py:80-99): int64 [B*h*w], ties -> lowest index."""
        if self._packed is None:
            self.finalize()
        zf = ops.nchw_to_nhwc_f32(z.float().contiguous()).reshape(-1, self.embed_dim)
        return ops.vq_argmin(zf, self._packed["codebook"])


class _MovqPlan(LaunchPlan):
    """Launch plan of MOVQ.decode (mode "decode": H, W = latent size) or MOVQ.encode ("encode": H, W = image size) for B
    images.  x_in (fp32 NCHW) is the static input, out (fp32 NCHW) the static output."""
    EPS = 1e-6  # GroupNorm eps of the VQGAN blocks (movq_modules.py:48, vqgan_blocks.py:34)

    def __init__(self, model, mode, B, H, W):
        pk = model._packed
        super().__init__(pk["pq_w"].device, B)
        self.m, self.mode, self.B = model, mode, B
        self._flip = 0
        f32 = dict(device=self.dev, dtype=torch.float32)
        dd = model.ddconfig
        if mode == "decode":
            self.x_in = torch.zeros(B, dd["z_channels"], H, W, **f32)
            s = 2 ** (len(model.levels) - 1)
            self.out = torch.empty(B, dd["out_ch"], H * s, W * s, **f32)
            self._build_decode(H, W)
        else:
            self.x_in = torch.zeros(B, dd["in_channels"], H, W, **f32)
            self._build_encode(H, W)

    # blocks ------------------------------------------------------------------------------------
    def _x(self, *shape):
        """Block outputs alternate between two buffers per shape (a block's input is dead once the next block has run)."""
        self._flip ^= 1
        return self._tmp(f"x{self._flip}", *shape)

    def _sn(self, x, zq, n, act, y):
        """SpatialNorm (decoder: zq given) or plain GroupNorm(32, eps 1e-6) (encoder: zq None), optional swish."""
        st = self._stats(x, None, self.EPS)
        if zq is None:
            self._add(lambda: ops.gn_apply(x, None, st, n["g"], n["b"], act=act, y=y), "gn_apply")
        else:
            self._add(lambda: ops.sn_apply(x, st, n["g"], n["b"], zq, n["w"], act=act, y=y), "sn_apply")

    def _res(self, x, zq, d):
        B, H, W, cin = x.shape
        cout = d["c1"].shape[0]
        hn = self._tmp("hn", B, H, W, cin)
        self._sn(x, zq, d["n1"], 1, hn)
        h = self._tmp("h", B, H, W, cout)
        self._conv([(hn, 9)], d["w1"], cout, h, 2 * B * H * W * cout * 9 * cin, bias=d["c1"], part_slot="part_h")
        hn2 = self._tmp("hn", B, H, W, cout)
        self._sn(h, zq, d["n2"], 1, hn2)
        o = self._x(B, H, W, cout)
        if cin == cout:
            self._conv([(hn2, 9)], d["w2"], cout, o, 2 * B * H * W * cout * 9 * cout, bias=d["c2"], residual=x)
        else:
            self._conv([(hn2, 9), (x, 1)], d["w2"], cout, o, 2 * B * H * W * cout * (9 * cout + cin), bias=d["c2"])
        return o

    def _attn(self, x, zq, d):
        """AttnBlock (movq_modules.py:201-225 / vqgan_blocks.py:186-240): one head of width C over T = H*W tokens."""
        B, H, W, C = x.shape
        T = H * W
        if T % 64:
            raise K2Error("MoVQ attention needs h*w to be a multiple of 64 (latents are multiples of 8 px)")
        hn = self._tmp("hn", B, H, W, C)
        self._sn(x, zq, d["n"], 0, hn)
        qkv = self._tmp("qkv", B, T, 3 * C)
        self._gemm(hn.view(B, T, C), d["wqkv"], 3 * C, qkv, 2 * B * T * 3 * C * C, bias=d["bqkv"])
        if C == 512 and _FUSED_ATTN:
            # fused flash kernel: no [T, T] score matrix (680 MB for four 768 x 768 images) in HBM
            o = self._tmp("att", B, T, C)
            self._add(lambda: ops.attention_d512(qkv, C ** -0.5, out=o), "attention", 4 * B * T * T * C)
            out = self._x(B, H, W, C)
            self._conv([(o.view(B, H, W, C), 1)], d["wp"], C, out, 2 * B * T * C * C, bias=d["bp"], residual=x)
            return out
        vT = self._tmp("vT", B, C, T)
        self._add(lambda: ops.transpose_f16(qkv[:, :, 2 * C:], out=vT), "transpose")
        scores = self._tmp("scores", B, T, T)
        q, k = qkv[:, :, :C], qkv[0, :, C:2 * C]
        # scores[n] = q[n] k[n]^T: A rows = q (row stride 3C), B operand of image n = its k rows (batch stride T * 3C)
        self._conv([(q.unsqueeze(1), 1)], k, T, scores.view(B, 1, T, T), 2 * B * T * T * C, want_stats=False,
                   w_batch_stride=T * 3 * C, kind="attn_gemm")
        self._add(lambda: ops.softmax_rows(scores.view(B * T, T), C ** -0.5, out=scores.view(B * T, T)), "softmax")
        o = self._tmp("att", B, T, C)
        self._conv([(scores.view(B, 1, T, T), 1)], vT[0], C, o.view(B, 1, T, C), 2 * B * T * T * C, want_stats=False,
                   w_batch_stride=C * T, kind="attn_gemm")
        out = self._x(B, H, W, C)
        self._conv([(o.view(B, H, W, C), 1)], d["wp"], C, out, 2 * B * T * C * C, bias=d["bp"], residual=x)
        return out

    # programs ----------------------------------------------------------------------------------
    def _build_decode(self, h, w):
        m, pk, B, S = self.m, self.m._packed, self.B, self._add
        f32 = dict(device=self.dev, dtype=torch.float32)
        zc = m.ddconfig["z_channels"]
        zq = torch.empty(B, h, w, m.embed_dim, **f32)
        z2 = torch.empty(B, zc, h, w, **f32)
        S(lambda: ops.nchw_to_nhwc_f32(self.x_in, out=zq), "misc")
        S(lambda: ops.pointwise_nchw_f32(self.x_in, pk["pq_w"], pk["pq_b"], out=z2), "misc")
        kpad = (9 * zc + 63) // 64 * 64
        patches = self._new(B, h, w, kpad)
        S(lambda: ops.stem_im2col(z2, kpad=kpad, out=patches), "stem_im2col")
        x = self._x(B, h, w, m.block_in)
        self._conv([(patches, 1)], pk["in_w"], m.block_in, x, 2 * B * h * w * m.block_in * 9 * zc, bias=pk["in_b"])
        x = self._res(x, zq, pk["mid1"])
        x = self._attn(x, zq, pk["mida"])
        x = self._res(x, zq, pk["mid2"])
        for lv in m.levels:
            p = f"decoder.up.{lv['level']}."
            for bi in range(len(lv["blocks"])):
                x = self._res(x, zq, pk[p + f"block.{bi}"])
                if lv["attn"]:
                    x = self._attn(x, zq, pk[p + f"attn.{bi}"])
            if lv["up"]:
                _, H, W, C = x.shape
                o = self._x(B, 2 * H, 2 * W, C)
                self._conv([(x, 4)], pk[p + "up_w"], C, o, 2 * B * 4 * H * W * C * C * 9, bias=pk[p + "up_b"])
                x = o
        _, H, W, C = x.shape
        hn = self._tmp("hn", B, H, W, C)
        self._sn(x, zq, pk["out_n"], 1, hn)
        oc = m.ddconfig["out_ch"]
        self._conv([(hn, 9)], pk["out_w"], oc, self.out, 2 * B * H * W * oc * 9 * C, bias=pk["out_b"], out_mode=1,
                   want_stats=False)

    def _build_encode(self, H, W):
        m, pk, B, S = self.m, self.m._packed, self.B, self._add
        dd = m.ddconfig
        cin = dd["in_channels"]
        kpad = (9 * cin + 63) // 64 * 64
        patches = self._new(B, H, W, kpad)
        S(lambda: ops.stem_im2col(self.x_in, kpad=kpad, out=patches), "stem_im2col")
        x = self._x(B, H, W, dd["ch"])
        self._conv([(patches, 1)], pk["e_in_w"], dd["ch"], x, 2 * B * H * W * dd["ch"] * 9 * cin, bias=pk["e_in_b"])
        for lv in m.enc_levels:
            p = f"encoder.down.{lv['level']}."
            for bi in range(len(lv["blocks"])):
                x = self._res(x, None, pk[p + f"block.{bi}"])
                if lv["attn"]:
                    x = self._attn(x, None, pk[p + f"attn.{bi}"])
            if lv["down"]:
                _, h, w, C = x.shape
                full = self._tmp("h", B, h, w, C)
                self._conv([(x, 9)], pk[p + "down_w"], C, full, 2 * B * h * w * C * C * 9, bias=pk[p + "down_b"],
                           want_stats=False)
                o = self._x(B, h // 2, w // 2, C)
                S(lambda full=full, o=o: ops.subsample2(full, 1, 1, out=o), "misc")
                self._parts.pop(o.data_ptr(), None)
                x = o
        x = self._res(x, None, pk["e_mid1"])
        x = self._attn(x, None, pk["e_mida"])
        x = self._res(x, None, pk["e_mid2"])
        _, h, w, C = x.shape
        hn = self._tmp("hn", B, h, w, C)
        self._sn(x, None, pk["e_out_n"], 1, hn)
        zc_out = pk["e_out_b"].shape[0]
        z = torch.empty(B, zc_out, h, w, device=self.dev, dtype=torch.float32)
        self._conv([(hn, 9)], pk["e_out_w"], zc_out, z, 2 * B * h * w * zc_out * 9 * C, bias=pk["e_out_b"], out_mode=1,
                   want_stats=False)
        self.out = torch.empty(B, m.embed_dim, h, w, device=self.dev, dtype=torch.float32)
        S(lambda: ops.pointwise_nchw_f32(z, pk["qc_w"], pk["qc_b"], out=self.out), "misc")
