"""float64 restatements of the launches the transformer towers record through model/encoder.py's record_layers, each carrying a
first-order bound on what the plan's own arithmetic may leave.  The pattern is tests/plan_blocks_ref.py's: a value is V(v, e),
v the float64 result of the launch on the plan's own fp16 inputs with the fp32 weights of the state dict the tower was loaded
from (never the packed fp16 tensors, so that a packing or remap error shows), e a bound on |plan - v|.  The terms:
  fp16 weights          max(2^-11 |W|, 2^-25) per GEMM weight, carried with |x|;
  fp32 accumulation     K 2^-23 sum |products| over the K products, bias and residual included (test_gpu_conv_float64.py);
  fp16 storage          2^-11 |v| + 2^-25 at every GEMM output the plan stores in fp16;
  LayerNorm             one fp16 ulp of v plus 2^-20 (|gamma x_hat| + |beta|) (test_gpu_prior_kernels.py, layernorm_f16);
  GELU / QuickGELU      one fp16 ulp of v (test_gpu_prior_kernels.py / test_gpu_clip_vitl14_kernels.py, every fp16 input);
  attention             attention_ref.ref_attention's allowance for the fused kernels (attention_d64, attention_heads),
                        attention_ref.ref_attention_small's for attention_small, each plus one fp16 ulp of v;
  around the stack      the embeds' fp16 tables (xlmr_embed also carries them through its LayerNorm), clip_patchify's
                        fp16 pixels, the patch-embedding GEMM's fp16 position rows, prior_tokens' three roundings,
                        k2_linear's and k2_timestep_embedding's bounds as plan_blocks_ref states them, masked_mean_f16's
                        fp32 sum; clip_text_pool and the fp32 widening are exact.
Products of error terms are dropped; SLACK = 1.1 on the bound (plan_blocks_ref.share) is the only slack.

The q, k and v of the reference are the state dict's own per-head projections: the qkv GEMM's reference weight is assembled
here in the layout the attention kernels read (per head [q_h | k_h | v_h]), independently of checkpoints.pack_heads, and the
attention reference splits the plan's qkv snapshot by that same kernel contract.

Every launch is checked on the plan's own snapshot of its input (layer(..., snap=)): a launch's bound is its own arithmetic.
Mode(em=True) evaluates the same launches as an emulated plan instead (fp16 weights, fp16 rounding at every storage point,
float64 elsewhere): the CPU self-test holds it to the bound.  Mode(mut=...) applies one wiring error of MUTATIONS; such a value
must fall outside the bound.  The LayerNorm eps mutation (1e-5 instead of DPT's 1e-12) is not listed: at the towers' activation
scales it moves x_hat by about 1e-5 / (2 var), below an fp16 ulp of the output, so no bound on fp16 results can see it."""
import math

import torch

from tests.attention_ref import U, _ulp16, ref_attention, ref_attention_small
from tests.plan_blocks_ref import EPS32, EXACT, SLACK, TINY, TS_C, U16, Mode, V, _linear, share  # noqa: F401

MUTATIONS = {
    "ln_2_neighbour": "the next layer's ln_2 parameters",
    "fc2_bias_neighbour": "the next layer's mlp.fc2.bias",
    "pre_ln_residual_from_ln": "the pre-LN out-proj residual taken from the LayerNorm output instead of the layer input",
    "post_ln_fc2_residual_from_hA": "the post-LN fc2 residual taken from hA instead of ln_1's output",
    "qk_swap_head": "q and k exchanged in head 0",
    "v_next_head": "head 0's v taken from head 1",
    "scale_eighth": "the attention scale 1/8 instead of head_dim^-0.5",
    "act_swapped": "GELU and QuickGELU swapped",
    "mask_one_longer": "the key mask one token longer",
    "causal_off": "the causal mask off",
    "pos_shift": "XLM-R position rows shifted by one (counted from padding_idx instead of padding_idx + 1)",
    "time_token_to_image_row": "the prior's time token written to the image-token row",
}

# the launches of one layer in record_layers' order, and the stage names they write
PRE_LN = ("ln_1", "qkv", "att", "proj", "ln_2", "fc1", "act", "fc2")
POST_LN = ("qkv", "att", "proj", "ln_1", "fc1", "act", "fc2", "ln_2")


# ------------------------------------------------------------------------------------------------------------------------------
# the towers' source state dicts: layer i's parameters by role, fp32
# ------------------------------------------------------------------------------------------------------------------------------
_CLIP = dict(ln_1="layer_norm1", q="self_attn.q_proj", k="self_attn.k_proj", v="self_attn.v_proj", proj="self_attn.out_proj",
             ln_2="layer_norm2", fc1="mlp.fc1", fc2="mlp.fc2")
_FORMATS = {
    "clip_text": ("text_model.encoder.layers.{}.", _CLIP),
    "clip_vision": ("vision_model.encoder.layers.{}.", _CLIP),
    "mclip": ("transformer.encoder.layer.{}.",
              dict(q="attention.self.query", k="attention.self.key", v="attention.self.value", proj="attention.output.dense",
                   ln_1="attention.output.LayerNorm", fc1="intermediate.dense", fc2="output.dense", ln_2="output.LayerNorm")),
    "dpt": ("dpt.encoder.layer.{}.",
            dict(ln_1="layernorm_before", q="attention.attention.query", k="attention.attention.key",
                 v="attention.attention.value", proj="attention.output.dense", ln_2="layernorm_after", fc1="intermediate.dense",
                 fc2="output.dense")),
    "openai_text": ("transformer.resblocks.{}.",
                    dict(ln_1="ln_1", proj="attn.out_proj", ln_2="ln_2", fc1="mlp.c_fc", fc2="mlp.c_proj")),
    "openai_vision": ("visual.transformer.resblocks.{}.",
                      dict(ln_1="ln_1", proj="attn.out_proj", ln_2="ln_2", fc1="mlp.c_fc", fc2="mlp.c_proj")),
    "prior21": ("transformer.resblocks.{}.", dict(ln_1="ln_1", proj="attn.c_proj", ln_2="ln_2", fc1="mlp.c_fc", fc2="mlp.c_proj")),
    "prior22": ("transformer_blocks.{}.",
                dict(ln_1="norm1", q="attn1.to_q", k="attn1.to_k", v="attn1.to_v", proj="attn1.to_out.0", ln_2="norm3",
                     fc1="ff.net.0.proj", fc2="ff.net.2")),
}


def layer_params(fmt, sd, i):
    """{role: (fp32 weight, fp32 bias)} of layer i of a source state dict: ln_1, q, k, v, proj, ln_2, fc1, fc2 (ln_1 / ln_2 in
    the package's meaning: for the post-LN stack attention.output.LayerNorm / output.LayerNorm)."""
    prefix, names = _FORMATS[fmt]
    p = prefix.format(i)
    g = lambda n: (sd[p + n + ".weight"].float(), sd[p + n + ".bias"].float())  # noqa: E731
    out = {role: g(n) for role, n in names.items()}
    if fmt == "prior21":   # the reference's c_qkv is already per head [q_h | k_h | v_h] (QKVMultiheadAttention's split)
        w, b = sd[p + "attn.c_qkv.weight"].float(), sd[p + "attn.c_qkv.bias"].float()
        H = w.shape[1]
        ws, bs = w.reshape(H // 64, 3, 64, H).unbind(1), b.reshape(H // 64, 3, 64).unbind(1)
        out.update({r: (wr.reshape(H, H), br.reshape(H)) for r, wr, br in zip("qkv", ws, bs)})
    elif "q" not in names:   # OpenAI's fused in_proj [q; k; v]
        ws, bs = sd[p + "attn.in_proj_weight"].float().chunk(3), sd[p + "attn.in_proj_bias"].float().chunk(3)
        out.update({r: (w, b) for r, w, b in zip("qkv", ws, bs)})
    return out


def qkv_weight(P, hd):
    """(weight [3 H, K], bias [3 H]) of the qkv GEMM in the attention kernels' layout: per head [q_h | k_h | v_h]."""
    (wq, bq), (wk, bk), (wv, bv) = P["q"], P["k"], P["v"]
    H, K = wq.shape
    w = torch.stack([t.reshape(H // hd, hd, K) for t in (wq, wk, wv)], 1).reshape(3 * H, K)
    b = torch.stack([t.reshape(H // hd, hd) for t in (bq, bk, bv)], 1).reshape(3 * H)
    return w, b


# ------------------------------------------------------------------------------------------------------------------------------
# launches
# ------------------------------------------------------------------------------------------------------------------------------
def layernorm(x, w, b, eps, M=EXACT):
    """layernorm_f16 of fp16 rows x (V, exact input) with fp32 gain / bias."""
    xv = x.v
    mu = xv.mean(-1, keepdim=True)
    xhat = (xv - mu) / torch.sqrt(xv.var(-1, unbiased=False, keepdim=True) + eps)
    gd, bd = w.double(), b.double()
    v = xhat * gd + bd
    if M.em:
        return V(v.half().double())
    if not M.bound:
        return V(v)
    return V(v, _ulp16(v) + 2.0 ** -20 * ((gd * xhat).abs() + bd.abs()))


def gemm(x, w, b, M=EXACT, res=None):
    """gemm_rows: fp16 x [..., K] (V, exact input) @ fp16(W)^T + fp32 bias (+ fp16 residual, V exact), fp32 accumulation,
    stored in fp16."""
    Wd = w.double()
    Wv = w.half().double() if M.em else Wd
    v = x.v @ Wv.T + b.double()
    if res is not None:
        v = v + res.v
    if M.em:
        return V(v.half().double())
    if not M.bound:
        return V(v)
    Wa, xa = Wd.abs(), x.v.abs()
    A = xa @ Wa.T + b.double().abs() + (res.v.abs() if res is not None else 0)
    K = w.shape[1] + 1 + (res is not None)
    e = xa @ (U16 * Wa).clamp(min=TINY).T + K * EPS32 * A + U16 * v.abs() + TINY
    return V(v, e)


def activation(x, act, M=EXACT):
    """gelu_f16_ (exact GELU) or quick_gelu_f16_ (x sigmoid(1.702 x)) of fp16 x (V, exact input)."""
    if M.mut == "act_swapped":
        act = "gelu" if act == "quick_gelu" else "quick_gelu"
    xv = x.v
    v = 0.5 * xv * torch.special.erfc(-xv / 2.0 ** 0.5) if act == "gelu" else xv * torch.sigmoid(1.702 * xv)
    if M.em:
        return V(v.half().double())
    return V(v, _ulp16(v)) if M.bound else V(v)


def one_longer(keep):
    """The key mask one token longer: each row's first masked token kept (the prior's always-kept extension tokens stay)."""
    keep = keep.clone()
    masked = keep == 0
    rows = masked.any(1).nonzero().flatten()
    keep[rows, masked.int().argmax(1)[rows]] = 1
    return keep


def _split_heads(qkv, heads, hd, M):
    """qkv [B, T, heads * 3 hd] -> q, k, v [B, T, heads, hd] by the kernels' layout, with the head mutations applied."""
    B, T = qkv.shape[:2]
    q, k, v = qkv.reshape(B, T, heads, 3, hd).unbind(3)
    if M.mut == "qk_swap_head":
        q, k = q.clone(), k.clone()
        q[:, :, 0], k[:, :, 0] = k[:, :, 0].clone(), q[:, :, 0].clone()
    elif M.mut == "v_next_head":
        v = v.clone()
        v[:, :, 0] = v[:, :, 1]
    return q, k, v


def attention(qkv, t, M=EXACT, keep=None):
    """The tower's attention launch over the fp16 qkv snapshot (V, exact input): t["attn"] "small" (attention_small, key mask
    `keep` [B, T] and t["causal"]) or "fused" (attention_d64 / attention_heads, no mask); scale t["scale"]."""
    heads, hd = t["heads"], t["hd"]
    scale = 0.125 if M.mut == "scale_eighth" else t["scale"]
    q, k, v = _split_heads(qkv.v, heads, hd, M)
    B, T = q.shape[:2]
    if t["attn"] == "small":
        causal = t["causal"] and M.mut != "causal_off"
        if keep is not None and M.mut == "mask_one_longer":
            keep = one_longer(keep)
        o, allow = ref_attention_small(torch.stack([q, k, v], 3).reshape(B, T, -1), heads, keep, causal, scale)
        o, allow = o.reshape(B, T, heads * hd), allow.reshape(B, T, heads * hd)
    else:
        outs = [ref_attention(q[b], k[b], v[b], scale) for b in range(B)]
        o = torch.stack([x[0] for x in outs]).reshape(B, T, heads * hd)
        allow = torch.stack([x[1] for x in outs]).reshape(B, T, heads * hd)
    if M.em:
        return V(o.half().double())
    return V(o, allow + _ulp16(o)) if M.bound else V(o)


# ------------------------------------------------------------------------------------------------------------------------------
# one layer of record_layers
# ------------------------------------------------------------------------------------------------------------------------------
def layer(P, Pn, h, t, M=EXACT, snap=None, keep=None):
    """Layer with parameters P (layer_params; Pn: the next layer's, read by the neighbour mutations) over its input h (V) ->
    {stage: V} in launch order (PRE_LN / POST_LN).  snap {stage: V}: the plan's own output of a stage, which the next stage
    reads instead of the computed value, so that each stage's bound is its own launch's arithmetic.
    t: the tower's traits -- heads, hd, scale, eps, act ("gelu" / "quick_gelu"), post_ln, attn ("small" / "fused"), causal."""
    S = {}

    def nx(key, val):
        S[key] = val
        return snap[key] if snap is not None and key in snap else val

    eps, mut = t["eps"], M.mut
    ln_2 = Pn["ln_2"] if mut == "ln_2_neighbour" else P["ln_2"]
    fc2_b = Pn["fc2"][1] if mut == "fc2_bias_neighbour" else P["fc2"][1]
    wq, bq = qkv_weight(P, t["hd"])
    if not t["post_ln"]:
        y = nx("ln_1", layernorm(h, *P["ln_1"], eps, M))
        qkv = nx("qkv", gemm(y, wq, bq, M))
        att = nx("att", attention(qkv, t, M, keep))
        hA = nx("proj", gemm(att, *P["proj"], M, res=y if mut == "pre_ln_residual_from_ln" else h))
        y2 = nx("ln_2", layernorm(hA, *ln_2, eps, M))
        f = nx("fc1", gemm(y2, *P["fc1"], M))
        g = nx("act", activation(f, t["act"], M))
        S["fc2"] = gemm(g, P["fc2"][0], fc2_b, M, res=hA)
        return S
    qkv = nx("qkv", gemm(h, wq, bq, M))
    att = nx("att", attention(qkv, t, M, keep))
    hA = nx("proj", gemm(att, *P["proj"], M, res=h))
    y = nx("ln_1", layernorm(hA, *P["ln_1"], eps, M))
    f = nx("fc1", gemm(y, *P["fc1"], M))
    g = nx("act", activation(f, t["act"], M))
    hB = nx("fc2", gemm(g, P["fc2"][0], fc2_b, M, res=hA if mut == "post_ln_fc2_residual_from_hA" else y))
    S["ln_2"] = layernorm(hB, *ln_2, eps, M)
    return S


def _eq(a, b, what):
    assert a.shape == b.shape and torch.equal(a, b), what


def check_wiring(layers, post_ln, name):
    """layers: per layer {stage: recorded call with "ins" / "out" snapshots}.  Each launch read exactly the bits its producer
    in the layer order wrote; returns the last layer's output."""
    h = layers[0][POST_LN[0] if post_ln else PRE_LN[0]]["ins"]["x"]
    for i, c in enumerate(layers):
        w = lambda s: f"{name} layer {i}: {s}"  # noqa: E731
        if not post_ln:
            _eq(c["ln_1"]["ins"]["x"], h, w("ln_1 does not read the layer input"))
            _eq(c["qkv"]["ins"]["x"], c["ln_1"]["out"], w("the qkv GEMM does not read ln_1's output"))
            _eq(c["proj"]["ins"]["res"], h, w("the out-proj residual is not the layer input"))
            _eq(c["ln_2"]["ins"]["x"], c["proj"]["out"], w("ln_2 does not read the out-proj output"))
            _eq(c["fc1"]["ins"]["x"], c["ln_2"]["out"], w("fc1 does not read ln_2's output"))
            _eq(c["fc2"]["ins"]["res"], c["proj"]["out"], w("the fc2 residual is not the out-proj output"))
            last = "fc2"
        else:
            _eq(c["qkv"]["ins"]["x"], h, w("the qkv GEMM does not read the layer input"))
            _eq(c["proj"]["ins"]["res"], h, w("the out-proj residual is not the layer input"))
            _eq(c["ln_1"]["ins"]["x"], c["proj"]["out"], w("ln_1 does not read the out-proj output"))
            _eq(c["fc1"]["ins"]["x"], c["ln_1"]["out"], w("fc1 does not read ln_1's output"))
            _eq(c["fc2"]["ins"]["res"], c["ln_1"]["out"], w("the fc2 residual is not ln_1's output"))
            _eq(c["ln_2"]["ins"]["x"], c["fc2"]["out"], w("ln_2 does not read fc2's output"))
            last = "ln_2"
        _eq(c["att"]["ins"]["qkv"], c["qkv"]["out"], w("attention does not read the qkv GEMM's output"))
        _eq(c["proj"]["ins"]["x"], c["att"]["out"], w("the out-proj does not read the attention output"))
        _eq(c["act"]["ins"]["x"], c["fc1"]["out"], w("the activation does not read fc1's output"))
        _eq(c["fc2"]["ins"]["x"], c["act"]["out"], w("fc2 does not read the activation's output"))
        h = c[last]["out"]
    return h


def mutations(t):
    """The MUTATIONS that apply to a tower with traits t."""
    out = ["ln_2_neighbour", "fc2_bias_neighbour", "qk_swap_head", "v_next_head", "act_swapped"]
    out.append("post_ln_fc2_residual_from_hA" if t["post_ln"] else "pre_ln_residual_from_ln")
    if t["hd"] != 64:
        out.append("scale_eighth")
    if t.get("masked"):
        out.append("mask_one_longer")
    if t["attn"] == "small" and t["causal"]:
        out.append("causal_off")
    return out


def stage_shares(got, ref):
    """got {stage: plan tensor}, ref {stage: V with bound} -> {stage: (worst, median) share of the bound}."""
    return {k: share(got[k], ref[k]) for k in ref if k in got}


def rejection(mutated, ref):
    """How far a mutated restatement lies outside the bound: the largest |mutated - v| / (SLACK e) over the stages."""
    return max(share(mutated[k].v, ref[k])[0] for k in ref if k in mutated)


def stack(Ps, h, t, M=EXACT, keep=None, at=None, mut=None):
    """The whole layer stack chained in float64 from the input h (V) without snapshots -> the last layer's output value;
    mut applied at layer `at` only.  For the end-to-end effect of a mutation."""
    x = h
    for i, P in enumerate(Ps):
        Pn = Ps[i + 1] if i + 1 < len(Ps) else Ps[i - 1]
        Mi = Mode(bound=False, mut=mut if i == at else None)
        x = V(layer(P, Pn, x, t, Mi, keep=keep)[PRE_LN[-1] if not t["post_ln"] else POST_LN[-1]].v)
    return x.v


def rel_l2(a, b):
    return ((a - b).norm() / b.norm()).item()



# ------------------------------------------------------------------------------------------------------------------------------
# what the towers record before and after the stack
# ------------------------------------------------------------------------------------------------------------------------------
def _ln_of(s, es, w, b, eps):
    """LayerNorm of float64 rows s carrying an input error es (first order: d x_hat = rstd (dx - d mean - x_hat
    mean(x_hat (dx - d mean)))), plus layernorm's own allowance."""
    mu = s.mean(-1, keepdim=True)
    rstd = 1.0 / torch.sqrt(s.var(-1, unbiased=False, keepdim=True) + eps)
    xhat = (s - mu) * rstd
    gd, bd = w.double(), b.double()
    v = xhat * gd + bd
    dx = rstd * (es + es.mean(-1, keepdim=True) + xhat.abs() * (xhat.abs() * es).mean(-1, keepdim=True))
    return V(v, gd.abs() * dx + _ulp16(v) + 2.0 ** -20 * ((gd * xhat).abs() + bd.abs()))


def xlmr_positions(ids, pad_id, M=EXACT):
    """transformers' create_position_ids_from_input_ids: padding_idx + the count of non-pad ids up to t, padding_idx on a pad."""
    m = (ids != pad_id).long()
    p = torch.cumsum(m, 1) * m + pad_id
    return p - m if M.mut == "pos_shift" else p


def xlmr_embed(ids, word, pos, type0, gamma, beta, pad_id, eps, M=EXACT):
    """xlmr_embed: LayerNorm(word[id] + type + pos[p]) from fp32 tables the plan holds in fp16, an fp32 sum, float64
    statistics, one rounding.  Bound: the tables' fp16 rounding and the two fp32 additions through the LayerNorm."""
    p = xlmr_positions(ids, pad_id, M)
    a, t, q = word.double()[ids], type0.double()[None, None], pos.double()[p]
    s = a + t + q
    if M.em:
        s16 = a.float().half().double() + t.float().half().double() + q.float().half().double()
        return V(_ln_of(s16, torch.zeros_like(s16), gamma, beta, eps).v.half().double())
    mag = a.abs() + t.abs() + q.abs()
    es = U16 * mag + 3 * TINY + 2 * EPS32 * mag
    out = _ln_of(s, es, gamma, beta, eps)
    return out if M.bound else V(out.v)


def patchify(pix, P, kp):
    """clip_patchify: [CLS | patches] rows of width kp: the CLS row a one-hot at column 3 P^2, each patch's pixels in
    (c, ky, kx) order rounded to fp16, zeros after."""
    B, _, S, _ = pix.shape
    G = S // P
    p = pix.double().reshape(B, 3, G, P, G, P).permute(0, 2, 4, 1, 3, 5).reshape(B, G * G, 3 * P * P)
    rows = torch.zeros(B, G * G + 1, kp, dtype=torch.float64, device=pix.device)
    rows[:, 0, 3 * P * P] = 1
    rows[:, 1:, :3 * P * P] = p
    return V(rows, U16 * rows.abs() + TINY * (rows != 0))


def patch_embed(rows, wconv, cls, pos, kp, M=EXACT, bias=None):
    """The patch-embedding GEMM: rows (V, exact) @ [conv weight | class embedding | 0]^T + the position rows the plan holds in
    fp16 (pos fp32 [T, H]; bias: the patch convolution's, folded into the patch rows)."""
    H = wconv.shape[0]
    K3 = wconv[0].numel()
    w = torch.zeros(H, kp, dtype=torch.float32, device=wconv.device)
    w[:, :K3] = wconv.reshape(H, K3).float()
    w[:, K3] = cls.reshape(H).float()
    pv = pos.double().clone()
    if bias is not None:
        pv[1:] += bias.double()
    B = rows.v.shape[0]
    res = pv.expand(B, *pv.shape)
    if M.em:
        return gemm(rows, w, torch.zeros(H), M, res=V(res.float().half().double()))
    out = gemm(rows, w, torch.zeros(H, dtype=torch.float32, device=w.device), M, res=V(res))
    return V(out.v, out.e + U16 * res.abs() + TINY) if M.bound else out


def masked_mean(h, keep, M=EXACT):
    """masked_mean_f16: the kept rows' fp32 sum in ascending t over the count, fp32 out (h V exact [B, T, H])."""
    if M.mut == "mask_one_longer":
        keep = one_longer(keep)
    k = keep.double()[..., None]
    n = k.sum(1)
    v = (h.v * k).sum(1) / n
    if M.em:
        return V(v.float().double())
    e = (n + 2) * EPS32 * (h.v.abs() * k).sum(1) / n + U * v.abs()
    return V(v, e) if M.bound else V(v)


def pool_rows(h, index):
    """clip_text_pool: the hidden row at each sequence's pooled position, widened exactly."""
    v = h.v[torch.arange(h.v.shape[0], device=h.v.device), index]
    return V(v, torch.zeros_like(v))


def projection(x, W, b, M=EXACT, silu_in=False):
    """k2_linear with fp32 weights (test_gpu_linear_float64.py's bound): x (V, exact fp32 input) @ W^T + b."""
    b = torch.zeros(W.shape[0], dtype=W.dtype, device=W.device) if b is None else b
    return _linear(V(x.v, torch.zeros_like(x.v) if x.e is None else x.e), W, b, M, silu_in=silu_in)


def timestep_embedding(t, dim, M=EXACT):
    """k2_timestep_embedding: [cos | sin] of t f, f = 10000^(-i / half); the kernel's argument error (TS_C) through cos / sin
    and their own 2 ulps, as plan_blocks_ref.film_chain bounds them."""
    half = dim // 2
    f = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float64, device=t.device) / half)
    arg = t.double()[:, None] * f[None]
    v = torch.cat([torch.cos(arg), torch.sin(arg)], 1)
    if M.em:
        return V(v.float().double())
    return V(v, TS_C * EPS32 * torch.cat([arg, arg], 1).abs() + 2 * EPS32 * v.abs()) if M.bound else V(v)


def prior_token(x, pos):
    """prior_tokens: fp16(fp16(x) + fp16(pos)) of the fp32 row x (V, exact) and the fp32 position row: its three roundings."""
    v = x.v + pos.double()
    return V(v, U16 * (x.v.abs() + pos.double().abs() + v.abs()) + 3 * TINY)
