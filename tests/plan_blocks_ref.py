"""float64 restatements of the UNet and MoVQ blocks as their launch plans compute them, each carrying a first-order bound on
what the plan's own arithmetic may leave, derived term by term.

A value is V(v, e): v the float64 result of the block's operations on the plan's fp16 inputs with the fp32 state-dict
weights (never the packed fp16 weights, so that a packing error shows), e a bound on |plan - v|.  The terms:
  fp16 weights            max(2^-11 |W|, 2^-25) per weight; the up2 path's phase sums (ops.pack_conv_weight_up2) add
                          3 fp32 roundings of the summed magnitudes before that rounding;
  fp16 storage            2^-11 |v| + 2^-25 at every tensor the plan stores in fp16 (h1 / h2 / h3, hn / h / hn2, qkv, the
                          attention output, scores and P on the unfused route), 2^-24 |v| at the fp32 NCHW heads;
  fp32 accumulation       K 2^-23 sum |products| (K products, bias and residual included), as in test_gpu_conv_float64.py;
  input errors            carried through convolutions with |W|;
  GroupNorm               the kernels' own allowance (test_gpu_groupnorm_float64.py: fp32 affine 2^-20 of its terms, the
                          statistics' format for both gn_stats and conv partials) plus the perturbation of the statistics by
                          the input error: |d mean| <= mean_g e, |d rstd| / rstd <= rstd^2 mean_g(|x - mean| e);
  SiLU                    slope <= 1.1 on the carried error, plus its own 2^-20 + 2^-23 |t| relative;
  attention               tests/attention_ref.py's kernel allowance (fused) or the softmax_rows allowance of
                          test_gpu_attention_float64.py with its fp16 scores and P (unfused), plus the input errors: a score
                          error eta_ts = scale (e_q |k| + |q| e_k) moves the output by <= sum_s p_ts eta_ts (|v_s| + |o_t|),
                          a value error by sum_s p_ts e_v;
  FiLM chain              k2_timestep_embedding's argument error and k2_linear's FMA chains as test_gpu_linear_float64.py
                          bounds them, fp16 FiLM weights as above.
Products of two error terms are dropped; SLACK = 1.1 on the final bound stands for them, the only slack allowed.

Blocks are checked stage by stage, split at the storage points a launch plan leaves behind (the stage keys of each block
function): every stage reads the plan's own snapshot of its input, so a stage's bound is its own arithmetic.  Carried with |W|
through a whole block, the first-order bound grows by about sqrt(K) per convolution -- on CONFIG_TINY's first ResBlock it
reaches 0.9 of |v| after two 3x3 convolutions -- and no longer separates a wiring error from rounding.

Mode(em=True) evaluates the same blocks as an emulated plan instead (fp16 weights, fp16 rounding at every storage point,
float64 elsewhere, no bound): the CPU self-test holds that emulation to the bound.  Mode(mut=...) applies one wiring error
(MUTATIONS) to the value; such a value must fall outside the bound."""
import math

import torch
import torch.nn.functional as F

from tests.attention_ref import U, ref_attention
from tests.test_gpu_groupnorm_float64 import CHAIN_PARTIAL, SILU_SLOPE, _ref_stats, _silu64, _silu_allow, _stats_allowance

U16 = 2.0 ** -11   # fp16 rounding to nearest, relative
EPS32 = 2.0 ** -23  # fp32 add, rounding or truncating, relative
TINY = 2.0 ** -25   # half the fp16 subnormal step
SLACK = 1.1         # the dropped second-order terms: every product of two relative errors above is < 2^-8

MUTATIONS = {
    "film_neighbour": "the neighbouring ResBlock's FiLM rows",
    "film_scale": "scale instead of 1 + scale",
    "gn_first_source": "GroupNorm statistics of h alone instead of the concat [h | skip]",
    "res_unresampled": "the residual taken from the un-resampled input",
    "zq_offset": "zq resized with a one-pixel offset",
    "no_enc": "the encoder tokens dropped from the UNet attention",
    "no_scale": "the MoVQ attention without its C^-0.5 scale",
    "up2_plain": "plain 3x3 weights on the up2 path (one kernel tap per phase tap, no pre-sum)",
    "film_packed_neighbour": "the first ResBlock's emb_layers packed in its same-width neighbour's place in the FiLM GEMM",
    "emb_no_xf_proj": "the time embedding without the conditioning's xf_proj",
    "film_no_silu_in": "the FiLM GEMM without SiLU on its input",
}
TS_C = 21   # k2_timestep_embedding's argument error in units of |t f| 2^-23 (test_gpu_linear_float64.py)


class Mode:
    def __init__(self, em=False, bound=None, mut=None):
        self.em = em
        self.bound = (not em and mut is None) if bound is None else bound
        self.mut = mut


EXACT = Mode()


class V:
    __slots__ = ("v", "e")

    def __init__(self, v, e=None):
        self.v, self.e = v, e


def inp(x):
    """A plan tensor read as an exact block input: NHWC fp16 [n, H, W, C] -> NCHW float64 with zero error."""
    v = x.double().permute(0, 3, 1, 2).contiguous()
    return V(v, torch.zeros_like(v))


def share(got, ref):
    """(worst, median) of |got - v| / (SLACK e) over all elements (0 where both are 0: exact copies); got NCHW (any float
    dtype).  NaN in got fails as an infinite share."""
    err = (got.double() - ref.v).abs()
    r = torch.where(err == 0, torch.zeros_like(err), err / (SLACK * ref.e)).nan_to_num(nan=float("inf")).flatten()
    return r.max().item(), r.median().item()


def check_stages(got, ref):
    """got {stage: tensor}, ref {stage: V} -> (worst share over the stages, median share of the output, {stage: worst})."""
    per = {k: share(got[k], ref[k])[0] for k in ref if k in got}
    return max(per.values()), share(got["out"], ref["out"])[1], per


# ------------------------------------------------------------------------------------------------------------------------------
# storage points
# ------------------------------------------------------------------------------------------------------------------------------
def r16(x, M):
    if M.em:
        return V(x.v.half().double())
    if not M.bound:
        return x
    return V(x.v, x.e + U16 * x.v.abs() + TINY)


def _pool(t):
    return F.avg_pool2d(t, 2)


def pool16(x, M):
    """2 x 2 average of fp16 activations (each rounded before the fp32 average), stored in fp16."""
    if M.em:
        return V(_pool(x.v.half().double()).half().double())
    v = _pool(x.v)
    if not M.bound:
        return V(v)
    return V(v, _pool(x.e + U16 * x.v.abs() + TINY) + 4 * U * _pool(x.v.abs()) + U16 * v.abs() + TINY)


def up2x(x):
    up = lambda t: t.repeat_interleave(2, 2).repeat_interleave(2, 3)  # noqa: E731
    return V(up(x.v), None if x.e is None else up(x.e))


# ------------------------------------------------------------------------------------------------------------------------------
# convolutions
# ------------------------------------------------------------------------------------------------------------------------------
# up2: output row 2y + a reads upsampled rows 2y + a + ky - 1, i.e. source row y + ty + a - 1 with these kernel rows per ty
_PHASE_ROWS = {0: ((0,), (1, 2)), 1: ((0, 1), (2,))}


def _phase_w(W, a, b, first=False):
    k = W.new_zeros(W.shape[0], W.shape[1], 2, 2)
    for ty in (0, 1):
        for tx in (0, 1):
            rows, cols = _PHASE_ROWS[a][ty], _PHASE_ROWS[b][tx]
            if first:
                k[:, :, ty, tx] = W[:, :, rows[0], cols[0]]
            else:
                k[:, :, ty, tx] = W[:, :, list(rows)][:, :, :, list(cols)].sum((2, 3))
    return k


def _up2(x, W, first=False, em=False):
    """3x3 conv over the nearest-2x upsampling of x as four 2x2 phase convolutions over x itself.  em: phase weights summed in
    fp32 and rounded to fp16 once (pack_conv_weight_up2)."""
    n, _, H, Wd = x.shape
    out = x.new_zeros(n, W.shape[0], 2 * H, 2 * Wd)
    xp = F.pad(x, (1, 1, 1, 1))
    for a in (0, 1):
        for b in (0, 1):
            k = _phase_w(W.float(), a, b, first).half().double() if em else _phase_w(W, a, b, first)
            out[:, :, a::2, b::2] = F.conv2d(xp, k)[:, :, a:a + H, b:b + Wd]
    return out


def _lin(x, W, kind, first=False, em=False):
    if kind == "3x3":
        return F.conv2d(x, W, padding=1)
    if kind == "1x1":
        return F.conv2d(x, W.reshape(W.shape[0], W.shape[1], 1, 1))
    return _up2(x, W, first, em)


_K = {"3x3": 9, "1x1": 1, "up2": 4}


def conv(parts, biases, M, res=None, out16=True):
    """parts [(V x NCHW, fp32 weight [Cout, Cin, kh, kw] or [Cout, Cin(, 1)], kind '3x3' | '1x1' | 'up2')]; biases: fp32
    vectors the plan sums in fp32 (c2 + skip bias); res: V added in the epilogue.  Output rounded to fp16 (out16) or fp32."""
    first = M.mut == "up2_plain"
    v = 0
    for x, W, kind in parts:
        Wv = W.half().double() if M.em else W.double()
        v = v + _lin(x.v, Wv, kind, first and kind == "up2", M.em)
    bsum = sum(b.double() for b in biases)
    v = v + bsum[None, :, None, None]
    if res is not None:
        v = v + res.v
    if M.em:
        return V(v.half().double() if out16 else v.float().double())
    if not M.bound:
        return V(v)
    A = sum(b.double().abs() for b in biases)[None, :, None, None] + (res.v.abs() if res is not None else 0)
    e = (res.e if res is not None else 0) + (U * A if len(biases) > 1 else 0)
    K = len(biases) + (res is not None)
    for x, W, kind in parts:
        Wa = W.double().abs()
        ew = ((U16 + (3 * U if kind == "up2" else 0)) * Wa).clamp(min=TINY)
        xa = x.v.abs()
        A = A + _lin(xa, Wa, kind)
        e = e + _lin(x.e, Wa, kind) + _lin(xa, ew, kind)
        K += _K[kind] * x.v.shape[1]
    e = e + K * EPS32 * A
    e = e + (U16 * v.abs() + TINY if out16 else U * v.abs())
    return V(v, e)


# ------------------------------------------------------------------------------------------------------------------------------
# GroupNorm (+FiLM | SpatialNorm modulation) (+SiLU), before the storage rounding
# ------------------------------------------------------------------------------------------------------------------------------
def _group_stats(x, first_c=None):
    """Per (image, group) mean / biased variance of NCHW x.  first_c: the mutation's statistics -- 32 groups over the first
    source's first_c channels alone (finalize fed only the first source's partials), applied by group index to the concat."""
    n = x.shape[0]
    if first_c is not None:
        x = x[:, :first_c]
    xg = x.reshape(n, 32, -1)
    return xg.mean(-1), xg.var(-1, unbiased=False)


def sn_mod(sd, p, zq, H, W, M):
    """SpatialNorm modulation (my, mb, |my| terms, |mb| terms) [n, C, H, W] of the fp32 latent zq [n, 4, h, w] nearest-resized
    to H x W (the plan reads the plan input x_in itself)."""
    zu = F.interpolate(zq.double(), size=(H, W), mode="nearest")
    if M.mut == "zq_offset":
        zu = torch.cat([zu[:, :, :, :1], zu[:, :, :, :-1]], 3)
    wy, by = sd[p + "conv_y.weight"].double().flatten(1), sd[p + "conv_y.bias"].double()
    wb, bb = sd[p + "conv_b.weight"].double().flatten(1), sd[p + "conv_b.bias"].double()
    e = lambda z, w, b: torch.einsum("nzhw,cz->nchw", z, w) + b[None, :, None, None]  # noqa: E731
    return e(zu, wy, by), e(zu, wb, bb), e(zu.abs(), wy.abs(), by.abs()), e(zu.abs(), wb.abs(), bb.abs())


def norm(srcs, gamma, beta, eps, act, M, film=None, mod=None):
    """GroupNorm32 of the channel concat of srcs (V NCHW), affine, FiLM rows film [n, 2C] (fp32 plan side input, exact) or
    SpatialNorm modulation mod, optional SiLU.  Not yet rounded."""
    x = torch.cat([s.v for s in srcs], 1)
    n, C, H, W = x.shape
    cpg = C // 32
    first_c = srcs[0].v.shape[1] if M.mut == "gn_first_source" and len(srcs) > 1 else None
    mean, var = _group_stats(x, first_c)
    rstd = 1.0 / torch.sqrt(var + eps)
    bc = lambda t: t.repeat_interleave(cpg, 1)[:, :, None, None]  # noqa: E731
    mu, rho = bc(mean), bc(rstd)
    xc = x - mu
    gd, bd = gamma.double()[None, :, None, None], beta.double()[None, :, None, None]
    if mod is None:
        if film is not None:
            s = film[:, :C].double()[:, :, None, None]
            sc = s if M.mut == "film_scale" else 1 + s
            sh = film[:, C:2 * C].double()[:, :, None, None]
        else:
            sc, sh = torch.ones_like(gd), torch.zeros_like(gd)
        A = gd * rho * sc
        t = xc * A + bd * sc + sh
    else:
        my, mb, my_abs, mb_abs = mod
        A = gd * rho
        t = (xc * A + bd) * my + mb
    o = _silu64(t) if act else t
    if not M.bound:
        return V(o)
    ex = torch.cat([s.e for s in srcs], 1)
    # the statistics' perturbation by the input error
    em_in = ex.reshape(n, 32, -1).mean(-1)
    er_in = rstd ** 2 * (xc.abs() * ex).reshape(n, 32, -1).mean(-1)
    # the kernels' own statistics allowance, whichever path (gn_stats or conv partials) the plan took
    ek, rk = [], []
    chain_stats = -(-H * W // 16) + 16   # gn_stats' chain is at most this (test_gpu_groupnorm_float64._stats_chain)
    for i in range(n):
        rs = _ref_stats(x[i].permute(1, 2, 0), 32)
        m1, r1 = _stats_allowance("partials", rs, eps, CHAIN_PARTIAL)
        m2, r2 = _stats_allowance("stats", rs, eps, chain_stats)
        ek.append(torch.maximum(m1, m2))
        rk.append(torch.maximum(r1, r2))
    em, er = bc(em_in + torch.stack(ek)), bc(er_in + torch.stack(rk))
    if mod is None:
        terms = (x * A).abs() + (mu * A).abs() + (bd * sc).abs() + sh.abs()
        scal = A.abs()
    else:
        terms = ((x * A).abs() + (mu * A).abs() + bd.abs()) * my_abs + mb_abs
        scal = (A * my).abs()
    e = scal * (ex + em) + (xc * scal).abs() * er + 2.0 ** -20 * terms
    if act:
        e = SILU_SLOPE * e + _silu_allow(t)
    return V(o, e)


# ------------------------------------------------------------------------------------------------------------------------------
# attention, one image: q [T, H, D], k / v [S, H, D] as V
# ------------------------------------------------------------------------------------------------------------------------------
def attend(q, k, v, scale, M, fused=True):
    """softmax(q k^T scale) v -> V [T, H, D], not yet rounded.  fused: one kernel with fp32 scores (attention_d64 /
    attention_d512); else the MoVQ's unfused route: fp16 scores of a GEMM, softmax_rows to fp16 P, a P V GEMM."""
    T, H, D = q.v.shape
    S = k.v.shape[0]
    if M.em:
        s = torch.einsum("thc,shc->hts", q.v, k.v)
        if not fused:
            s = s.half().double()
        p = torch.softmax(s * scale, -1)
        if not fused:
            p = p.half().double()
        return V(torch.einsum("hts,shc->thc", p, v.v))
    if not M.bound:
        return V(torch.einsum("hts,shc->thc", torch.softmax(torch.einsum("thc,shc->hts", q.v, k.v) * scale, -1), v.v))
    ka, va = k.v.abs(), v.v.abs()
    if fused:
        o, allow = ref_attention(q.v, k.v, v.v, scale)
    outs, errs = [], []
    rows = max(1, 2 ** 24 // (H * S))
    for t0 in range(0, T, rows):
        qc, eqc = q.v[t0:t0 + rows], q.e[t0:t0 + rows]
        s = torch.einsum("thc,shc->hts", qc, k.v)
        es = torch.einsum("thc,shc->hts", eqc, ka) + torch.einsum("thc,shc->hts", qc.abs(), k.e)
        if not fused:  # the scores GEMM: D-term fp32 chain, fp16 store
            es += D * EPS32 * torch.einsum("thc,shc->hts", qc.abs(), ka) + U16 * s.abs() + TINY
        z = s * scale
        p = torch.softmax(z, -1)
        pe = p * (scale * es)
        if fused:
            oc = o[t0:t0 + rows]
            ec = (torch.einsum("hts,shc->thc", p, v.e) + torch.einsum("hts,shc->thc", pe, va)
                  + pe.sum(-1).transpose(0, 1)[..., None] * oc.abs() + allow[t0:t0 + rows])
        else:
            eta = 2.0 ** -22 * (z.abs() + z.amax(-1, keepdim=True).abs()) + 2.0 ** -21
            ep = (p * (eta + (p * eta).sum(-1, keepdim=True) + (S / 256 + 16) * U)
                  + pe + p * pe.sum(-1, keepdim=True) + U16 * p + TINY)
            oc = torch.einsum("hts,shc->thc", p, v.v)
            ec = (torch.einsum("hts,shc->thc", ep, va) + torch.einsum("hts,shc->thc", p, v.e)
                  + S * EPS32 * torch.einsum("hts,shc->thc", p, va))
        outs.append(oc)
        errs.append(ec)
    return V(torch.cat(outs), torch.cat(errs))


def _img_heads(x, i, heads, width, parts):
    """Image i of NCHW [n, heads * parts * width, H, W] -> `parts` V tensors [T, heads, width]."""
    def one(t):
        return t[i].reshape(heads, parts, width, -1).permute(1, 3, 0, 2)
    vv = one(x.v)
    ee = one(x.e) if x.e is not None else [None] * parts
    return [V(vv[j], ee[j]) for j in range(parts)]


def _stack_heads(outs, H, W):
    """[V [T, heads, D]] per image -> V NCHW [n, heads * D, H, W]."""
    f = lambda t: t.reshape(H, W, -1).permute(2, 0, 1)  # noqa: E731
    v = torch.stack([f(o.v) for o in outs])
    e = torch.stack([f(o.e) for o in outs]) if outs[0].e is not None else None
    return V(v, e)


# ------------------------------------------------------------------------------------------------------------------------------
# UNet blocks (oracle/unet_oracle.py _res / _attn; kandinsky2/model/unet.py _Plan._layer)
# ------------------------------------------------------------------------------------------------------------------------------
def _stages(snap):
    """Stage outputs of one block, and the input each next stage reads: the plan's snapshot of that storage point when one is
    given (the block is checked stage by stage, each from the plan's own fp16 input), else the computed value."""
    S = {}

    def nx(key, val):
        S[key] = val
        return snap[key] if snap is not None and key in snap else val
    return S, nx


def unet_res(sd, p, a, b, film, updown, M=EXACT, snap=None):
    """ResBlock over a (and the up path's skip b): film = this block's FiLM rows [n, 2 cout] (plan.film).  -> {stage: V}:
    h1 (h1s on the up path), xres (resampling blocks), h2, h3, out."""
    w = lambda k: sd[p + k]  # noqa: E731
    S, nx = _stages(snap)
    srcs = [a] + ([b] if b is not None else [])
    h = norm(srcs, w("in_layers.0.weight"), w("in_layers.0.bias"), 1e-5, 1, M)
    W1, c1 = w("in_layers.2.weight"), w("in_layers.2.bias")
    xres = None
    if updown is None:
        h1 = nx("h1", r16(h, M))
        h2 = nx("h2", r16(conv([(h1, W1, "3x3")], [c1], M), M))
    elif updown == "down":
        xres = nx("xres", pool16(a, M))
        h1 = nx("h1", pool16(h, M))
        h2 = nx("h2", r16(conv([(h1, W1, "3x3")], [c1], M), M))
    else:
        xres = nx("xres", up2x(a))
        h1 = nx("h1s", r16(h, M))
        h2 = nx("h2", r16(conv([(h1, W1, "up2")], [c1], M), M))
    h3 = nx("h3", r16(norm([h2], w("out_layers.0.weight"), w("out_layers.0.bias"), 1e-5, 1, M, film=film), M))
    W2, c2 = w("out_layers.3.weight"), w("out_layers.3.bias")
    if (p + "skip_connection.weight") not in sd:
        res = xres if xres is not None else a
        if M.mut == "res_unresampled" and xres is not None:
            Ho, Wo = h3.v.shape[2:]
            iy = torch.arange(Ho, device=a.v.device) % a.v.shape[2]
            ix = torch.arange(Wo, device=a.v.device) % a.v.shape[3]
            res = V(a.v[:, :, iy][:, :, :, ix])
        S["out"] = conv([(h3, W2, "3x3")], [c2], M, res=res)
        return S
    x = V(torch.cat([s.v for s in srcs], 1), torch.cat([s.e for s in srcs], 1) if a.e is not None else None)
    S["out"] = conv([(h3, W2, "3x3"), (x, w("skip_connection.weight"), "1x1")], [c2, w("skip_connection.bias")], M)
    return S


def unet_attn(sd, p, a, enc, M=EXACT, snap=None):
    """AttentionBlock over a with the encoder K / V enc [n, ctx, 2C] (the plan's enc_kv buffer: per head k | v).
    -> {stage: V}: xn, qkv, att, out."""
    w = lambda k: sd[p + k]  # noqa: E731
    S, nx = _stages(snap)
    n, C, H, W = a.v.shape
    heads = C // 64
    xn = nx("xn", r16(norm([a], w("norm.weight"), w("norm.bias"), 1e-5, 0, M), M))
    qkv = nx("qkv", r16(conv([(xn, w("qkv.weight"), "1x1")], [w("qkv.bias")], M), M))
    outs = []
    for i in range(n):
        q, k, v = _img_heads(qkv, i, heads, 64, 3)
        if M.mut != "no_enc" and enc is not None and enc.shape[1]:
            ek, ev = enc[i].double().reshape(-1, heads, 2, 64).unbind(2)
            z = torch.zeros_like(ek)
            k = V(torch.cat([ek, k.v]), None if k.e is None else torch.cat([z, k.e]))
            v = V(torch.cat([ev, v.v]), None if v.e is None else torch.cat([z, v.e]))
        outs.append(attend(q, k, v, 0.125, M, fused=True))
    att = nx("att", r16(_stack_heads(outs, H, W), M))
    S["out"] = conv([(att, w("proj_out.weight"), "1x1")], [w("proj_out.bias")], M, res=a)
    return S


def _linear(x, W, b, M, silu_in=False, silu_out=False, add=None, half_w=False):
    """k2_linear: fp32 x [n, K] (V) @ W^T + b (+ add), fp32 out; half_w: the plan holds W in fp16.  Bound as
    test_gpu_linear_float64.py: (K + 8) 2^-24 sum |products| for the fp32 FMA chain, SiLU's own error on the input or the
    output (slope 1.1 on what it carries), one rounding of the added row; plus the input error through |W| and, for fp16
    weights, max(2^-11 |W|, 2^-25)."""
    xin = _silu64(x.v) if silu_in else x.v
    Wv = W.half().double() if half_w and M.em else W.double()
    v = xin @ Wv.T + b.double()
    o = _silu64(v) if silu_out else v
    if add is not None:
        o = o + add.double()
    if M.em:
        return V(o.float().double())
    if not M.bound:
        return V(o)
    Wa = W.double().abs()
    acc = (W.shape[1] + 8) * U * (xin.abs() @ Wa.T + b.double().abs()) + (SILU_SLOPE * x.e if silu_in else x.e) @ Wa.T
    if silu_in:
        acc = acc + _silu_allow(x.v) @ Wa.T
    if half_w:
        acc = acc + xin.abs() @ (U16 * Wa).clamp(min=TINY).T
    e = SILU_SLOPE * acc + _silu_allow(v) if silu_out else acc
    if add is not None:
        e = e + U * o.abs()
    return V(o, e)


def film_chain(sd, lay, t, xf_proj, M=EXACT, snap=None):
    """The UNet plan's forked conditioning branch: e0 = timestep_embedding(t), e1 = silu(time_embed.0(e0)),
    emb = time_embed.2(e1) + xf_proj, film = every ResBlock's emb_layers.1(silu(emb)) as one fp16-weight GEMM in the plan's
    row order (lay = film_layout).  t, xf_proj: the plan's fp32 inputs t_in / xf_proj.  -> {stage: V}: e0, e1, emb, out (the
    whole plan.film)."""
    S, nx = _stages(snap)
    mc = sd["time_embed.0.weight"].shape[1]
    half = mc // 2
    f = torch.exp(-math.log(10000.0) * torch.arange(half, dtype=torch.float64, device=t.device) / half)
    arg = t.double()[:, None] * f[None]
    e0 = torch.cat([torch.cos(arg), torch.sin(arg)], 1)
    if M.em:
        e0 = V(e0.float().double())
    elif M.bound:   # the kernel's argument error (TS_C) through cos / sin (slope <= 1), and their own 2 ulps
        e0 = V(e0, TS_C * EPS32 * torch.cat([arg, arg], 1).abs() + 2 * EPS32 * e0.abs())
    else:
        e0 = V(e0)
    e0 = nx("e0", e0)
    e1 = nx("e1", _linear(e0, sd["time_embed.0.weight"], sd["time_embed.0.bias"], M, silu_out=True))
    emb = nx("emb", _linear(e1, sd["time_embed.2.weight"], sd["time_embed.2.bias"], M,
                            add=None if M.mut == "emb_no_xf_proj" else xf_proj))
    order = list(lay)
    if M.mut == "film_packed_neighbour":
        i, j = 0, order.index(film_neighbour(lay, order[0]))
        order[i], order[j] = order[j], order[i]
    Wf = torch.cat([sd[p + "emb_layers.1.weight"] for p in order])
    bf = torch.cat([sd[p + "emb_layers.1.bias"] for p in order])
    S["out"] = _linear(emb, Wf, bf, M, silu_in=M.mut != "film_no_silu_in", half_w=True)
    return S


def _f32_in(x):
    """An fp32 plan input: exact, but allowed one fp32 rounding (the inpainting stem's product img * mask)."""
    v = x.double()
    return V(v, U * v.abs())


def unet_stem(sd, x_in, M=EXACT):
    """conv_in over the fp32 NCHW stem input (inpainting: already concatenated [x, img * mask, mask]), its 3x3 patches rounded
    to fp16 (stem_im2col)."""
    return conv([(r16(_f32_in(x_in), M), sd["input_blocks.0.0.weight"], "3x3")], [sd["input_blocks.0.0.bias"]], M)


def unet_head(sd, h, M=EXACT):
    hn = r16(norm([h], sd["out.0.weight"], sd["out.0.bias"], 1e-5, 1, M), M)
    return conv([(hn, sd["out.2.weight"], "3x3")], [sd["out.2.bias"]], M, out16=False)


def unet_enc_kv(sd, p, xf16, M=EXACT):
    """encoder_kv of the fp16 conditioning tokens xf16 [n, ctx, model_dim] -> V [n, 2C, ctx, 1] (plan layout: transpose)."""
    x = xf16.double().permute(0, 2, 1)[..., None]
    return conv([(V(x, torch.zeros_like(x)), sd[p + "encoder_kv.weight"], "1x1")], [sd[p + "encoder_kv.bias"]], M)


def unet_block_table(cfg):
    """[(prefix, layer, c0)] in the plan's order; c0 = channels of the block input's first source (the up path's h)."""
    from oracle import unet_oracle as uo
    inp, mid, out = uo.unet_topology(cfg)
    table = []
    ch = inp[0][0][2]
    for bi, blk in enumerate(inp[1:], start=1):
        for li, layer in enumerate(blk):
            table.append((f"input_blocks.{bi}.{li}.", layer, ch))
            ch = layer[2] if layer[0] == "res" else ch
    for li, layer in enumerate(mid):
        table.append((f"middle_block.{li}.", layer, ch))
    for bi, blk in enumerate(out):
        for li, layer in enumerate(blk):
            table.append((f"output_blocks.{bi}.{li}.", layer, ch))
            ch = layer[2] if layer[0] == "res" else ch
    return table


def film_layout(cfg):
    """{prefix: (offset, cout)} of every ResBlock's rows in the plan's one FiLM GEMM, and the prefixes in order."""
    lay, off = {}, 0
    for p, layer, _ in unet_block_table(cfg):
        if layer[0] == "res":
            lay[p] = (off, layer[2])
            off += 2 * layer[2]
    return lay


def film_neighbour(lay, p):
    """The nearest other ResBlock with the same width: its rows are what an off-by-one FiLM offset would read."""
    order = list(lay)
    i = order.index(p)
    for j in sorted(range(len(order)), key=lambda j: (abs(j - i), j)):
        if j != i and lay[order[j]][1] == lay[p][1]:
            return order[j]
    raise AssertionError(p)


# ------------------------------------------------------------------------------------------------------------------------------
# MoVQ blocks (oracle/movq_oracle.py _res / _attn / _enc_res / _enc_attn; kandinsky2/vqgan/autoencoder.py _MovqPlan)
# ------------------------------------------------------------------------------------------------------------------------------
def _movq_norm(sd, p, x, zq, act, M):
    if zq is None:
        return norm([x], sd[p + "weight"], sd[p + "bias"], 1e-6, act, M)
    H, W = x.v.shape[2:]
    return norm([x], sd[p + "norm_layer.weight"], sd[p + "norm_layer.bias"], 1e-6, act, M, mod=sn_mod(sd, p, zq, H, W, M))


def movq_res(sd, p, x, zq, M=EXACT, snap=None):
    """ResnetBlock (decoder: SpatialNorm over zq; encoder: zq None, GroupNorm eps 1e-6).  -> {stage: V}: hn, h, hn2, out."""
    S, nx = _stages(snap)
    hn = nx("hn", r16(_movq_norm(sd, p + "norm1.", x, zq, 1, M), M))
    h = nx("h", r16(conv([(hn, sd[p + "conv1.weight"], "3x3")], [sd[p + "conv1.bias"]], M), M))
    hn2 = nx("hn2", r16(_movq_norm(sd, p + "norm2.", h, zq, 1, M), M))
    if (p + "nin_shortcut.weight") not in sd:
        S["out"] = conv([(hn2, sd[p + "conv2.weight"], "3x3")], [sd[p + "conv2.bias"]], M, res=x)
    else:
        S["out"] = conv([(hn2, sd[p + "conv2.weight"], "3x3"), (x, sd[p + "nin_shortcut.weight"], "1x1")],
                        [sd[p + "conv2.bias"], sd[p + "nin_shortcut.bias"]], M)
    return S


def movq_attn(sd, p, x, zq, fused, M=EXACT, snap=None):
    """AttnBlock: one head of width C, scale C^-0.5; fused = attention_d512, else the GEMM / softmax_rows / GEMM route (its fp16
    scores and P are carried inside the att stage).  -> {stage: V}: hn, qkv (q | k | v, the plan's layout), att, out."""
    S, nx = _stages(snap)
    n, C, H, W = x.v.shape
    hn = nx("hn", r16(_movq_norm(sd, p + "norm.", x, zq, 0, M), M))
    qkv = [r16(conv([(hn, sd[p + c + ".weight"], "1x1")], [sd[p + c + ".bias"]], M), M) for c in ("q", "k", "v")]
    qkv = nx("qkv", V(torch.cat([t.v for t in qkv], 1), None if qkv[0].e is None else torch.cat([t.e for t in qkv], 1)))
    scale = 1.0 if M.mut == "no_scale" else C ** -0.5
    outs = []
    for i in range(n):
        q, k, v = _img_heads(qkv, i, 1, C, 3)
        outs.append(attend(q, k, v, scale, M, fused=fused))
    att = nx("att", r16(_stack_heads(outs, H, W), M))
    S["out"] = conv([(att, sd[p + "proj_out.weight"], "1x1")], [sd[p + "proj_out.bias"]], M, res=x)
    return S


def movq_upconv(sd, p, x, M=EXACT):
    """Upsample: 3x3 over the nearest-2x upsampling (the plan's taps = 4 phase convolution)."""
    return conv([(x, sd[p + "upsample.conv.weight"], "up2")], [sd[p + "upsample.conv.bias"]], M)


def movq_downconv(sd, p, x, M=EXACT):
    """Downsample (pad (0, 1, 0, 1), 3x3 stride 2): the 'same' conv stored in fp16, then its odd pixels (subsample2(1, 1))."""
    o = conv([(x, sd[p + "downsample.conv.weight"], "3x3")], [sd[p + "downsample.conv.bias"]], M)
    return V(o.v[:, :, 1::2, 1::2], None if o.e is None else o.e[:, :, 1::2, 1::2])


def movq_dec_stem(sd, x_in, M=EXACT):
    """post_quant_conv (fp32 1x1 over the fp32 latent), its 3x3 patches rounded to fp16, conv_in.  The bound charges the fp32
    pointwise kernel an fp16 weight rounding it does not have (an over-count of 2^-11 of a 4-term sum)."""
    z2 = conv([(_f32_in(x_in), sd["post_quant_conv.weight"], "1x1")], [sd["post_quant_conv.bias"]], M, out16=False)
    if M.em:  # the emulation keeps the 1x1's fp32 weights, as the plan's pointwise kernel does
        z2 = V(F.conv2d(x_in.double(), sd["post_quant_conv.weight"].double(),
                        sd["post_quant_conv.bias"].double()).float().double())
    return conv([(r16(z2, M), sd["decoder.conv_in.weight"], "3x3")], [sd["decoder.conv_in.bias"]], M)


def movq_dec_head(sd, x, zq, M=EXACT):
    hn = r16(_movq_norm(sd, "decoder.norm_out.", x, zq, 1, M), M)
    return conv([(hn, sd["decoder.conv_out.weight"], "3x3")], [sd["decoder.conv_out.bias"]], M, out16=False)


def movq_enc_stem(sd, x_in, M=EXACT):
    return conv([(r16(_f32_in(x_in), M), sd["encoder.conv_in.weight"], "3x3")], [sd["encoder.conv_in.bias"]], M)


def movq_enc_head(sd, x, M=EXACT):
    """norm_out + swish, conv_out to fp32 NCHW, then quant_conv (fp32 1x1)."""
    hn = r16(_movq_norm(sd, "encoder.norm_out.", x, None, 1, M), M)
    z = conv([(hn, sd["encoder.conv_out.weight"], "3x3")], [sd["encoder.conv_out.bias"]], M, out16=False)
    if M.em:
        return V(F.conv2d(z.v, sd["quant_conv.weight"].double(), sd["quant_conv.bias"].double()).float().double())
    return conv([(z, sd["quant_conv.weight"], "1x1")], [sd["quant_conv.bias"]], M, out16=False)


def downsample_oracle(sd, p, h):
    """The oracle's own Downsample (movq_oracle.movq_encode), for the CPU test that the plan's restatement equals it."""
    return F.conv2d(F.pad(h, (0, 1, 0, 1)), sd[p + "downsample.conv.weight"].double(), sd[p + "downsample.conv.bias"].double(),
                    stride=2)


def log2_share(s):
    return math.log2(max(s, 1e-300))
