"""The pre-LayerNorm transformer layer stack shared by the diffusion prior (model/prior.py) and the two CLIP towers
(model/clip_text.py, model/clip_vision.py): how one layer's weights are named, checked and packed, and the launches one layer
records in a LaunchPlan:
    LayerNorm -> qkv GEMM -> attention -> out-proj GEMM + residual -> LayerNorm -> fc1 GEMM -> GELU -> fc2 GEMM + residual.
The attention launch is the caller's; everything else is the same for all the models (the 2.1 ViT-L/14 towers of
model/clip_vitl14.py record QuickGELU instead of GELU: record_layers(act="quick_gelu")).  record_layers(post_ln=True)
records the post-LayerNorm layer of the 2.1 text encoder (model/text_encoders.py, XLM-RoBERTa) over the same packed names.

Around the stack: Tower, the shell of every tower that runs as graph-replayed launch plans (the CLIP towers, XLM-R, DPT):
the state-dict check, the packed weights, the plan cache, the token-id check and the distinct-prompt encode; the ViT patch
embedding the image towers share (pack_patch_embed, record_patch_embed); the f32 / f16 device packers; and the part of the
transformers CLIP config both CLIP towers read."""
import torch

from .. import ops
from .._native import K2Error

_NORMS = ("ln_1", "ln_2")
_GEMMS = ("attn.qkv", "attn.proj", "mlp.fc1", "mlp.fc2")
# the MLP activations a layer can record, by name (the name is also the launch's kind): the exact GELU of the prior, the bigG
# towers and XLM-R, and OpenAI CLIP's QuickGELU x * sigmoid(1.702 x) of the Kandinsky 2.1 ViT-L/14 towers
ACTIVATIONS = {"gelu": ops.gelu_f16_, "quick_gelu": ops.quick_gelu_f16_}


def layer_shapes(H, I):
    """{name: shape} of one layer's parameters in this package's names, at width H and MLP width I."""
    return {"ln_1.weight": (H,), "ln_1.bias": (H,), "ln_2.weight": (H,), "ln_2.bias": (H,),
            "attn.qkv.weight": (3 * H, H), "attn.qkv.bias": (3 * H,), "attn.proj.weight": (H, H), "attn.proj.bias": (H,),
            "mlp.fc1.weight": (I, H), "mlp.fc1.bias": (I,), "mlp.fc2.weight": (H, I), "mlp.fc2.bias": (H,)}


def f32(t, dev):
    """t as a contiguous fp32 tensor on dev."""
    return t.detach().to(dev, torch.float32).contiguous()


def f16(t, dev):
    """t as a contiguous fp16 tensor on dev."""
    return t.detach().to(dev, torch.float16).contiguous()


def pack_layers(get, L, dev):
    """L layers packed on `dev` once: a list of dicts with "ln_1" / "ln_2" -> (fp32 gain, fp32 bias) and "attn.qkv",
    "attn.proj", "mlp.fc1", "mlp.fc2" -> (fp16 [N, K] GEMM weight, ops.pack_conv_weight; fp32 bias).  get(i, name) returns
    layer i's parameter `name` (a layer_shapes key)."""
    layers = []
    for i in range(L):
        p = {n: (f32(get(i, n + ".weight"), dev), f32(get(i, n + ".bias"), dev)) for n in _NORMS}
        for n in _GEMMS:
            p[n] = (ops.pack_conv_weight(get(i, n + ".weight").detach().to(dev)), f32(get(i, n + ".bias"), dev))
        layers.append(p)
    return layers


def record_layers(plan, h, layers, attend, attn_flops, eps, post_ln=False, act="gelu"):
    """Record the layers (pack_layers) into `plan` over h fp16 [rows, tokens, C]; returns the last layer's output.  The
    buffers are [rows, tokens, C] views so that the GEMM tuner counts rows * tokens output rows.  attend(qkv, out) launches
    the attention of qkv [rows, tokens, 3C] into out [rows, tokens, C]; attn_flops is what one such launch computes.  The
    first layer reads h as its residual input; the stream then alternates between two buffers.  post_ln=True records the
    post-LayerNorm layer of BERT / XLM-RoBERTa instead (_record_post_ln).  act: the MLP activation, an ACTIVATIONS name."""
    rows, tokens, C = h.shape
    if act not in ACTIVATIONS:
        raise K2Error(f"encoder layers: activation {act!r} is not implemented (only {sorted(ACTIVATIONS)})")
    if not layers:
        return h
    if post_ln:
        return _record_post_ln(plan, h, layers, attend, attn_flops, eps, act)
    gelu = ACTIVATIONS[act]
    I, M, S = layers[0]["mlp.fc1"][0].shape[0], rows * tokens, plan._add
    y, att, hA, hB = (plan._new(rows, tokens, C) for _ in range(4))
    qkv, f = plan._new(rows, tokens, 3 * C), plan._new(rows, tokens, I)
    for L in layers:
        S(lambda h=h, L=L: ops.layernorm_f16(h, *L["ln_1"], eps=eps, out=y), "layernorm")
        plan._gemm(y, L["attn.qkv"][0], 3 * C, qkv, 2 * M * C * 3 * C, bias=L["attn.qkv"][1])
        S(lambda: attend(qkv, att), "attention", attn_flops)
        plan._gemm(att, L["attn.proj"][0], C, hA, 2 * M * C * C, bias=L["attn.proj"][1], residual=h)
        S(lambda L=L: ops.layernorm_f16(hA, *L["ln_2"], eps=eps, out=y), "layernorm")
        plan._gemm(y, L["mlp.fc1"][0], I, f, 2 * M * C * I, bias=L["mlp.fc1"][1])
        S(lambda: gelu(f), act)
        plan._gemm(f, L["mlp.fc2"][0], C, hB, 2 * M * I * C, bias=L["mlp.fc2"][1], residual=hA)
        h = hB
    return h


def _record_post_ln(plan, h, layers, attend, attn_flops, eps, act):
    """The post-LayerNorm layer (transformers' XLMRobertaLayer), eight launches:
        qkv GEMM -> attention -> out-proj GEMM + residual -> LayerNorm ln_1 (attention.output.LayerNorm) -> fc1 GEMM -> GELU
        -> fc2 GEMM + residual (ln_1's output) -> LayerNorm ln_2 (output.LayerNorm), whose output is the next layer's input.
    The first layer reads h; the stream then lives in one buffer that every layer overwrites last."""
    rows, tokens, C = h.shape
    I, M, S = layers[0]["mlp.fc1"][0].shape[0], rows * tokens, plan._add
    gelu = ACTIVATIONS[act]
    att, hA, y, hB, out = (plan._new(rows, tokens, C) for _ in range(5))
    qkv, f = plan._new(rows, tokens, 3 * C), plan._new(rows, tokens, I)
    for L in layers:
        plan._gemm(h, L["attn.qkv"][0], 3 * C, qkv, 2 * M * C * 3 * C, bias=L["attn.qkv"][1])
        S(lambda: attend(qkv, att), "attention", attn_flops)
        plan._gemm(att, L["attn.proj"][0], C, hA, 2 * M * C * C, bias=L["attn.proj"][1], residual=h)
        S(lambda L=L: ops.layernorm_f16(hA, *L["ln_1"], eps=eps, out=y), "layernorm")
        plan._gemm(y, L["mlp.fc1"][0], I, f, 2 * M * C * I, bias=L["mlp.fc1"][1])
        S(lambda: gelu(f), act)
        plan._gemm(f, L["mlp.fc2"][0], C, hB, 2 * M * I * C, bias=L["mlp.fc2"][1], residual=y)
        S(lambda L=L: ops.layernorm_f16(hB, *L["ln_2"], eps=eps, out=out), "layernorm")
        h = out
    return h


def pack_patch_embed(weight, cls, kp, dev):
    """The ViT patch embedding as one fp16 GEMM weight [H, kp] on dev: the patch convolution's weight [H, 3, P, P] in columns
    [0, 3 P^2), the class embedding [H] in column 3 P^2 (k2_clip_patchify's CLS row holds a 1 there), zeros after."""
    H, K = weight.shape[0], weight[0].numel()
    we = torch.zeros(H, kp, dtype=torch.float16, device=dev)
    we[:, :K] = weight.detach().to(dev).reshape(H, K).half()
    we[:, K] = cls.detach().to(dev).half()
    return we


def record_patch_embed(plan, pix, embed, pos, patch, kp):
    """Record the ViT embedding into `plan`: k2_clip_patchify of pix fp32 [B, 3, S, S] into [CLS | patch] rows of width kp,
    then ONE GEMM with pack_patch_embed's weight and pos fp16 [B, T, H] as the epilogue residual.  Returns the fp16
    embeddings [B, T, H]."""
    B, T, H = pos.shape
    rows = plan._new(B, T, kp)
    plan._add(lambda: ops.clip_patchify(pix, patch, kp, out=rows), "patchify")
    emb = plan._new(B, T, H)
    plan._gemm(rows, embed, H, emb, 2 * B * T * kp * H, residual=pos)
    return emb


class Tower:
    """The shell of a tower that runs as graph-replayed launch plans: the state-dict check, the weights packed on the device
    once, one plan per input geometry built on demand, the token-id check and the distinct-prompt encode.  A subclass sets
    `what` (the name its K2Error messages start with) and `device`, calls _take(sd, want) from its constructor, and
    implements _pack() (the packed dict, read by its plans as tower._packed) and _new_plan(*key) (its LaunchPlan)."""

    what = "tower"

    def _take(self, sd, want):
        """Keep the state dict sd after checking it against want {name: shape}: K2Error names the keys missing or of another
        shape and the unknown keys.  Nothing is packed yet: finalize() does that, or the first _plan()."""
        bad = [k for k, s in want.items() if k not in sd or tuple(sd[k].shape) != s]
        extra = sorted(set(sd) - set(want))
        if bad or extra:
            raise K2Error(f"{self.what}: keys missing or of the wrong shape for the config {bad}, unknown keys {extra}")
        self.sd, self._packed, self._plans = sd, None, {}

    def finalize(self):
        """Pack the weights on the device once (_pack); plans built on earlier weights are dropped."""
        self._packed, self._plans = self._pack(), {}
        return self

    def _plan(self, *key):
        """The launch plan for `key`, built (and the weights packed) on first use."""
        if self._packed is None:
            self.finalize()
        if key not in self._plans:
            self._plans[key] = self._new_plan(*key)
        return self._plans[key]

    def _check_ids(self, input_ids, max_tokens):
        """K2Error unless input_ids is an integer [n, T] tensor with n > 0, 0 < T <= max_tokens and every id in
        [0, cfg["vocab_size"]); checked before anything is copied to the device."""
        if input_ids.dim() != 2 or not 0 < input_ids.shape[1] <= max_tokens or input_ids.shape[0] == 0:
            raise K2Error(f"{self.what}: input_ids must be [n, T] with 0 < T <= {max_tokens}, got {list(input_ids.shape)}")
        if input_ids.is_floating_point() or input_ids.is_complex() or input_ids.dtype == torch.bool:
            raise K2Error(f"{self.what}: input_ids must be integers, got {input_ids.dtype}")
        lo, hi, V = int(input_ids.min()), int(input_ids.max()), self.cfg["vocab_size"]
        if lo < 0 or hi >= V:
            raise K2Error(f"{self.what}: token ids must lie in [0, {V}), got [{lo}, {hi}]")

    def _encode_distinct(self, prompts, encode):
        """encode(distinct prompts) -> device tensors with one row per distinct prompt, in order; returns them with the rows
        gathered back to one per prompt, so that each distinct prompt is tokenized and encoded once."""
        distinct = list(dict.fromkeys(prompts))
        outs = encode(distinct)
        idx = torch.tensor([distinct.index(p) for p in prompts], device=self.device)
        return tuple(t[idx] for t in outs)


def clip_config(config, required, what, head_dim):
    """The part of a transformers CLIP{Text,Vision}Config dict both towers read: the `required` integer keys, hidden_act and
    layer_norm_eps (transformers' defaults "quick_gelu" and 1e-5 when absent), checked against what this package implements
    (exact GELU, heads of head_dim); K2Error naming the `what` tower otherwise."""
    missing = [k for k in required if k not in config]
    if missing:
        raise K2Error(f"CLIP {what} config: missing {missing}")
    c = {k: int(config[k]) for k in required}
    c["hidden_act"] = config.get("hidden_act", "quick_gelu")
    c["layer_norm_eps"] = float(config.get("layer_norm_eps", 1e-5))
    if c["hidden_act"] != "gelu":
        raise K2Error(f"CLIP {what} tower: hidden_act {c['hidden_act']!r} is not implemented (only the exact 'gelu' of "
                      "ViT-bigG/14; the 2.1 tower's quick_gelu is not)")
    H, heads = c["hidden_size"], c["num_attention_heads"]
    if H % heads or H // heads != head_dim:
        raise K2Error(f"CLIP {what} tower: head width {H / heads:g} is not implemented (only {head_dim})")
    c["head_dim"] = head_dim
    return c
