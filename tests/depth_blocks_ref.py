"""float64 restatements of the depth estimators' launches outside the ViT layers -- the DPT neck, fusion and head, the hybrid's
BiT backbone and token GEMM -- and of the ControlNet hint stem, each carrying a first-order bound on what the launch's own
arithmetic may leave.  The pattern is tests/plan_blocks_ref.py's: a value is V(v, e), v the float64 result of the launch on
its input with the fp32 weights of the transformers / diffusers state dict (never the packed fp16 tensors, so that a packing
error shows), e a bound on |plan - v|.  The terms:
  fp16 weights          max(2^-11 |W|, 2^-25) per weight (plan_blocks_ref.conv, tower_layers_ref.gemm); a BiT weight is
                        standardised here in float64 and its one fp16 rounding is the weight term;
  fp32 accumulation     K 2^-23 sum |products|, bias, residual and identity-block terms included;
  fp16 storage          2^-11 |v| + 2^-25 at every fp16 output, 2^-24 |v| at the fp32 NCHW outputs;
  GELU                  tower_layers_ref.activation (one fp16 ulp);
  SiLU                  test_gpu_groupnorm_float64's _silu_allow, before the storage rounding;
  bilinear              one fp16 ulp of v plus the fp32 index / weight error test_gpu_depth_kernels.py derives
                        (4 max(Hi, Wi) 2^-23 2 max|x| + 4 2^-24 max|x|);
  GroupNorm             plan_blocks_ref.norm: exact statistics of the input, the statistics' format (gn_stats or conv
                        partials, whichever is larger) and the fp32 affine 2^-20 of its terms; one more 2^-20 term for the
                        shortcut a gn_act launch adds.  A statistics launch itself is held to _stats_allowance of the
                        producer's output;
  exact copies          readout rows, depth_to_space, subsample, ReLU, max pool, im2col (one fp16 rounding of fp32 pixels):
                        bound 0, checked bit for bit.
Products of error terms are dropped; SLACK = 1.1 on the bound (plan_blocks_ref.share) is the only slack.

Walk runs the launches in the plan's order.  With snap (the plan's own output of every launch, in order) each launch reads
those snapshots, so its bound is its own arithmetic (the GPU test; the CPU test with an emulated plan).  Without snap it
chains its own values: Mode(em=True) is the emulated plan (fp16 weights, fp16 rounding at every storage point, float64
elsewhere), pure EXACT mode the model in float64, which the CPU test ties to the oracles.  Mode(mut=...) applies one wiring
error of MUTATIONS at the launches it concerns; such a value must fall outside the bound."""
import torch
import torch.nn.functional as F

from tests import tower_layers_ref as R
from tests.attention_ref import U, _ulp16
from tests.plan_blocks_ref import EPS32, EXACT, TINY, U16, Mode, V, conv, norm, r16, share  # noqa: F401
from tests.test_gpu_groupnorm_float64 import CHAIN_PARTIAL, _ref_stats, _silu64, _silu_allow, _stats_allowance

MIN_REJECT = 4.0
GN_EPS = 1e-5

MUTATIONS = {
    "resize_taps_transposed": "the neck's ConvTranspose2d taps (a, b) transposed",
    "d2s_swapped": "depth_to_space with the sub-pixel order (b, a) for (a, b)",
    "readout_no_cls": "the readout rows without their CLS half",
    "readout_other_cls": "the readout rows with the other image's CLS",
    "neck_sub11": "the neck's factor-0.5 subsample at (1, 1)",
    "bit_sub00": "the BiT stride-2 subsample at (0, 0)",
    "im2col_pads_32": "the BiT stem im2col padded (3, 2) instead of (2, 3)",
    "fusion_no_running": "the fusion sum without the running map",
    "unit1_on_running": "unit1 applied to the running map instead of the stage",
    "bilinear_align": "the fusion bilinear with the other align_corners",
    "head_relu_dropped": "the head's ReLU dropped",
    "down_no_gn": "the downsample shortcut without its GroupNorm",
    "ws_off": "a BiT convolution's weight not standardised",
    "pos_shift": "the position residual shifted by one row",
    "hint_no_silu": "the hint stem without SiLU after one convolution",
}


def _nchw(t):
    return t.permute(0, 3, 1, 2)


def _nhwc(t):
    return t.permute(0, 2, 3, 1)


def _map(x, fn):
    return V(fn(x.v), None if x.e is None else fn(x.e))


def _exact(v, M):
    """An exact copy's value: bound 0 where a bound is kept."""
    return V(v, torch.zeros_like(v)) if M.bound else V(v)


def _pure(M):
    return not M.em and not M.bound and M.mut is None


def standardized(w, M=EXACT):
    """WeightStandardizedConv2d's weight in float64 from the fp32 weight: per output channel (w - mean) / sqrt(var + 1e-8)."""
    w = w.double()
    if M.mut == "ws_off":
        return w
    flat = w.reshape(w.shape[0], -1)
    mean = flat.mean(1, keepdim=True)
    var = ((flat - mean) ** 2).mean(1, keepdim=True)
    return ((flat - mean) / torch.sqrt(var + 1e-8)).reshape(w.shape)


# ------------------------------------------------------------------------------------------------------------------------------
# launches (NHWC values unless stated)
# ------------------------------------------------------------------------------------------------------------------------------
def conv3(x, W, b, M, out16=True):
    """k2_conv_gemm 3x3, pad 1 (+ bias): plan_blocks_ref.conv on the NHWC value; out16 False: fp32 NCHW out (out_mode 1)."""
    bias = b if b is not None else torch.zeros(W.shape[0], dtype=torch.float64, device=W.device)
    o = conv([(_map(x, _nchw), W, "3x3")], [bias], M, out16=out16)
    return _map(o, _nhwc) if out16 else o


def gemm(x, W, b, M, res=None):
    """gemm_rows / a 1x1 conv_gemm over the rows: tower_layers_ref.gemm with W [Cout, Cin(, 1, 1)]."""
    W = W.reshape(W.shape[0], -1)
    b = b if b is not None else torch.zeros(W.shape[0], dtype=torch.float64, device=W.device)
    return R.gemm(x, W, b, M, res=res)


def conv_fused(a, W, b, x, run, M):
    """The fusion unit's last conv_gemm: conv3x3(a) + b + the residual x (+ the running map run as a second 1x1 source with an
    identity weight): 9 C products and C identity products, the bias and the residual in one fp32 sum, one fp16 rounding."""
    ac, xc = _nchw(a.v), _nchw(x.v)
    Wd = W.double()
    Wv = W.half().double() if M.em else Wd
    v = F.conv2d(ac, Wv, padding=1) + b.double()[None, :, None, None] + xc
    if run is not None:
        v = v + _nchw(run.v)
    if M.em:
        return V(_nhwc(v).half().double())
    if not M.bound:
        return V(_nhwc(v))
    Wa = Wd.abs()
    A = F.conv2d(ac.abs(), Wa, padding=1) + b.double().abs()[None, :, None, None] + xc.abs()
    K = 9 * ac.shape[1] + 2
    if run is not None:
        A = A + _nchw(run.v).abs()
        K += run.v.shape[-1]
    e = F.conv2d(ac.abs(), (U16 * Wa).clamp(min=TINY), padding=1) + K * EPS32 * A + U16 * v.abs() + TINY
    return V(_nhwc(v), _nhwc(e))


def bilinear(x, size, align, M):
    """k2_bilinear_f16: torch's bilinear interpolate of the NCHW view in float64, one rounding."""
    if M.mut == "bilinear_align":
        align = not align
    v = _nhwc(F.interpolate(_nchw(x.v), size=size, mode="bilinear", align_corners=align))
    if M.em:
        return V(v.half().double())
    if not M.bound:
        return V(v)
    amax = x.v.abs().amax()
    e = _ulp16(v) + 4 * max(x.v.shape[1:3]) * 2.0 ** -23 * 2 * amax + 4 * U * amax
    return V(v, e)


def gn_act(x, gamma, beta, M, r=None, rn=None, relu=True):
    """k2_gn_act_f16: [relu](GN(x) gamma + beta + s), s = the fp16 shortcut r, or GN(r) with rn = (gamma, beta)."""
    t = norm([_map(x, _nchw)], gamma, beta, GN_EPS, 0, M)
    if r is not None:
        rc = _map(r, _nchw)
        s = norm([rc], rn[0], rn[1], GN_EPS, 0, M) if rn is not None and M.mut != "down_no_gn" else rc
        if M.bound:
            t = V(t.v + s.v, t.e + s.e + 2.0 ** -20 * s.v.abs())
        else:
            t = V(t.v + s.v)
    if relu:
        t = V(t.v.clamp_min(0), t.e)
    return r16(_map(t, _nhwc), M)


def gn_stats_ref(x, M):
    """The statistics launch (k2_gn_stats or k2_gn_finalize) of the producer's output x: (mean, rstd) [NB, 32] in float64 and
    the larger of the two formats' allowances."""
    xs = x.v
    NB, H, W, _ = xs.shape
    chain_stats = -(-H * W // 16) + 16
    out = []
    for n in range(NB):
        rs = _ref_stats(xs[n], 32)
        m1, r1 = _stats_allowance("partials", rs, GN_EPS, CHAIN_PARTIAL)
        m2, r2 = _stats_allowance("stats", rs, GN_EPS, chain_stats)
        out.append((rs[0], 1.0 / torch.sqrt(rs[1] + GN_EPS), torch.maximum(m1, m2), torch.maximum(r1, r2),
                    (rs[0].abs() / rs[1].sqrt().clamp_min(1e-300)).max()))
    return [torch.stack(t) for t in zip(*out)]


class Stats:
    """A statistics launch's reference; share() compares the plan's [NB, 32, 2] (mean, rstd)."""

    def __init__(self, x, M):
        self.mean, self.rstd, self.em, self.er, self.ratio = gn_stats_ref(x, M)
        self.v = torch.stack([self.mean, self.rstd], -1)

    def share(self, got):
        dm = (got[..., 0].double() - self.mean).abs() / self.em
        dr = (got[..., 1].double() - self.rstd).abs() / (self.rstd * self.er)
        r = torch.cat([dm.flatten(), dr.flatten()]).nan_to_num(nan=float("inf"))
        return r.max().item(), r.median().item()


def readout(hs, grid, M):
    """k2_readout_rows_f16: [token | CLS] rows of hs [B, T, H], each image's own CLS -> [B, gh, gw, 2 H]."""
    B, T, H = hs.v.shape
    tok = hs.v[:, 1:]
    cls = hs.v[:, :1].expand_as(tok)
    if M.mut == "readout_no_cls":
        cls = torch.zeros_like(tok)
    elif M.mut == "readout_other_cls":
        if B < 2:
            return None
        cls = cls.roll(1, 0)
    return _exact(torch.cat([tok, cls], -1).reshape(B, *grid, 2 * H), M)


def conv_transpose(p, W, b, s, M):
    """The resize of factor s (ConvTranspose2d, kernel = stride = s) in float64 of the GEMM's input p: F.conv_transpose2d, bound
    for its C + 1 term fp32 sum, the fp16 weights and the storage rounding."""
    pc = _nchw(p.v)
    Wd = W.double()
    if M.mut == "resize_taps_transposed":
        Wd = Wd.transpose(2, 3)
    Wv = Wd.half().double() if M.em else Wd
    v = F.conv_transpose2d(pc, Wv, b.double(), stride=s)
    if M.em:
        return V(_nhwc(v).half().double())
    if not M.bound:
        return V(_nhwc(v))
    Wa = Wd.abs()
    A = F.conv_transpose2d(pc.abs(), Wa, b.double().abs(), stride=s)
    e = (F.conv_transpose2d(pc.abs(), (U16 * Wa).clamp(min=TINY), stride=s) + (pc.shape[1] + 1) * EPS32 * A
         + U16 * v.abs() + TINY)
    return V(_nhwc(v), _nhwc(e))


def space_to_depth(y, s):
    """[B, s gh, s gw, C] -> the GEMM rows depth_to_space reads: column (a s + b) C + c of pixel (i, j) = y[s i + a, s j + b, c]."""
    B, Hs, Ws, C = y.shape
    return y.reshape(B, Hs // s, s, Ws // s, s, C).permute(0, 1, 3, 2, 4, 5).reshape(B, Hs // s, Ws // s, s * s * C)


def depth_to_space(g, s, C, M):
    B, gh, gw, _ = g.v.shape
    t = g.v.reshape(B, gh, gw, s, s, C)
    t = t.permute(0, 1, 4, 2, 3, 5) if M.mut == "d2s_swapped" else t.permute(0, 1, 3, 2, 4, 5)
    return _exact(t.reshape(B, s * gh, s * gw, C), M)


def stride2(full, ref_v, off, M, mut):
    """A stride-2 convolution done at stride 1 (full, V) then subsampled at off: the value of the stride-2 convolution itself
    (ref_v, computed by F.conv2d(stride=2) of the same input), carrying the stride-1 bound at the kept pixels."""
    if M.mut == mut:
        v = full.v[:, 1 - off::2, 1 - off::2]
        return V(v) if v.shape == ref_v.shape else None   # an odd grid: the mutation does not apply
    if not M.bound:
        return V(ref_v) if not M.em else V(full.v[:, off::2, off::2])
    return V(ref_v, full.e[:, off::2, off::2])


# ------------------------------------------------------------------------------------------------------------------------------
# the walk
# ------------------------------------------------------------------------------------------------------------------------------
class Walk:
    """The restated launches in the plan's order.  Each launch: op (the ops entry point, or a set of them), label, checks =
    [(label, V reference, {mutation: value})] against the launch's output (none: checked at a later launch, `at`), reads =
    {input snapshot name: producer launch index, or a tensor the input must equal}."""

    def __init__(self, M, snap=None, muts=True):
        self.M, self.snap, self.muts, self.launches, self.vals = M, snap, muts, [], []

    def add(self, op, label, f, reads=None, muts=(), also=(), at=None):
        """f(M) -> V, the launch's output; also: [(label, f2, muts)] further references of the same output.  Returns (value the
        next launches read, this launch's index)."""
        i = len(self.launches)
        M = self.M
        val = f(M)
        checks = []
        if M.bound and at is None:
            for lab, g, ms in [(label, f, muts)] + list(also):
                ref = val if g is f else g(M)
                mv = {}
                if self.muts:
                    for m in ms:
                        x = g(Mode(mut=m))
                        if x is not None:
                            mv[m] = x.v
                checks.append((lab, ref, mv))
        self.launches.append(dict(op=op, label=label, checks=checks, reads=reads or {}, at=at))
        self.vals.append(val)
        if self.snap is not None:
            s = self.snap[i]
            return V(s, torch.zeros_like(s)), i
        return (V(val.v) if not isinstance(val, Stats) else val), i

    # ---------------------------------------------------------------- DPT neck, fusion, head
    def reassemble(self, sd, c, i, hs, grid):
        """_DepthPlan._reassemble of stage i over the hidden state hs (V [B, T, H])."""
        rs = "neck.reassemble_stage."
        H, C, f = c["hidden_size"], c["neck_hidden_sizes"][i], float(c["reassemble_factors"][i])
        ro, iro = self.add("readout_rows_f16", "readout", lambda M: readout(hs, grid, M),
                           muts=("readout_no_cls", "readout_other_cls"))
        wr, br = sd[f"{rs}readout_projects.{i}.0.weight"], sd[f"{rs}readout_projects.{i}.0.bias"]
        r, ir = self.add("gemm_rows", "readout gemm", lambda M: gemm(ro, wr, br, M), {"x": iro})
        g, ig = self.add("gelu_f16_", "gelu", lambda M: R.activation(r, "gelu", M), {"x": ir})
        wp, bp = sd[f"{rs}layers.{i}.projection.weight"], sd[f"{rs}layers.{i}.projection.bias"]
        p, ip = self.add("gemm_rows", "projection", lambda M: gemm(g, wp, bp, M), {"x": ig})
        if f > 1:
            s = int(f)
            wt, bt = sd[f"{rs}layers.{i}.resize.weight"], sd[f"{rs}layers.{i}.resize.bias"]
            q, iq = self.add("gemm_rows", "resize gemm", lambda M: V(space_to_depth(conv_transpose(p, wt, bt, s, M).v, s)),
                             {"x": ip}, at="depth_to_space")
            y, iy = self.add("depth_to_space_f16", "depth_to_space", lambda M: depth_to_space(q, s, C, M), {"x": iq},
                             muts=("d2s_swapped",),
                             also=[("resize x%d (conv_transpose2d)" % s, lambda M: conv_transpose(p, wt, bt, s, M),
                                    ("resize_taps_transposed",))])
        elif f < 1:
            wt, bt = sd[f"{rs}layers.{i}.resize.weight"], sd[f"{rs}layers.{i}.resize.bias"]
            full, ifull = self.add("conv_gemm", "resize conv3x3 (stride 1)", lambda M: conv3(p, wt, bt, M), {"srcs": [ip]})
            gh, gw = grid
            ref2 = lambda M: _nhwc(F.conv2d(_nchw(p.v), wt.double(), bt.double(), stride=2, padding=1))  # noqa: E731
            chk = ("resize /2 (conv2d stride 2)",
                   lambda M: stride2(conv3(p, wt, bt, M) if (M.bound or M.em) else full, ref2(M), 0, M, "neck_sub11"),
                   ("neck_sub11",))
            copy = lambda M: _exact(full.v[:, ::2, ::2], M)  # noqa: E731
            if gh % 2 == 0 and gw % 2 == 0:
                y, iy = self.add("subsample2", "subsample", copy, {"x": ifull}, also=[chk])
            else:
                y, iy = self.add("bilinear_f16", "bilinear halving (every second pixel)", copy, {"x": ifull}, also=[chk])
        else:
            y, iy = p, ip
        return self.add("conv_gemm", "neck conv3x3", lambda M: conv3(y, sd[f"neck.convs.{i}.weight"], None, M),
                        {"srcs": [iy]})

    def _relu(self, x, ix, label, mut=None):
        return self.add("relu_f16", label, lambda M: _exact(x.v if mut and M.mut == mut else x.v.clamp_min(0), M), {"x": ix},
                        muts=(mut,) if mut else ())

    def unit(self, sd, p, x, ix, run=None, irun=None):
        """DPTPreActResidualLayer: conv3x3(relu(conv3x3(relu(x)))) + x (+ run through the identity block)."""
        w = lambda k: sd[p + k]  # noqa: E731
        a, ia = self._relu(x, ix, "relu (out of place)")
        c1, ic1 = self.add("conv_gemm", "unit conv3x3", lambda M: conv3(a, w("convolution1.weight"), w("convolution1.bias"), M),
                           {"srcs": [ia]})
        c1r, ic1r = self._relu(c1, ic1, "relu (in place)")
        W2, b2 = w("convolution2.weight"), w("convolution2.bias")
        if run is None:
            return self.add("conv_gemm", "unit conv3x3 + residual",
                            lambda M: conv3_res(c1r, W2, b2, x, M), {"srcs": [ic1r], "res": ix})

        def fused(M):
            if M.mut == "fusion_no_running":
                return conv_fused(c1r, W2, b2, x, None, M)
            if M.mut == "unit1_on_running":
                E = Mode(bound=False)
                h = conv3(V(run.v.clamp_min(0)), w("convolution1.weight"), w("convolution1.bias"), E)
                return conv_fused(V(h.v.clamp_min(0)), W2, b2, run, x, E)
            return conv_fused(c1r, W2, b2, x, run, M)
        return self.add("conv_gemm", "unit conv3x3 + residual + running map", fused, {"srcs": [ic1r, irun], "res": ix},
                        muts=("fusion_no_running", "unit1_on_running"))

    def fuse_head(self, sd, feats):
        """_DepthPlan._fuse_head over the neck maps [(V, index)] (shallow to deep) -> the fp32 NCHW depth map."""
        run = irun = None
        for j, (fe, ife) in enumerate(reversed(feats)):
            p = f"neck.fusion_stage.layers.{j}."
            if run is None:
                x, ix = fe, ife
            else:
                if fe.v.shape[1:3] != run.v.shape[1:3]:
                    size = tuple(run.v.shape[1:3])
                    fe, ife = self.add("bilinear_f16", "bilinear to the running map", lambda M, fe=fe, size=size:
                                       bilinear(fe, size, False, M), {"x": ife}, muts=("bilinear_align",))
                x, ix = self.unit(sd, p + "residual_layer1.", fe, ife, run, irun)
            x, ix = self.unit(sd, p + "residual_layer2.", x, ix)
            size = (2 * x.v.shape[1], 2 * x.v.shape[2])
            up, iup = self.add("bilinear_f16", "bilinear x2", lambda M, x=x, size=size: bilinear(x, size, True, M), {"x": ix},
                               muts=("bilinear_align",))
            run, irun = self.add("gemm_rows", "fusion projection", lambda M, up=up, p=p:
                                 gemm(up, sd[p + "projection.weight"], sd[p + "projection.bias"], M), {"x": iup})
        a, ia = self.add("conv_gemm", "head conv3x3", lambda M: conv3(run, sd["head.head.0.weight"], sd["head.head.0.bias"], M),
                         {"srcs": [irun]})
        size = (2 * a.v.shape[1], 2 * a.v.shape[2])
        u, iu = self.add("bilinear_f16", "bilinear x2", lambda M: bilinear(a, size, True, M), {"x": ia},
                         muts=("bilinear_align",))
        h, ih = self.add("conv_gemm", "head conv3x3", lambda M: conv3(u, sd["head.head.2.weight"], sd["head.head.2.bias"], M),
                         {"srcs": [iu]})
        hr, ihr = self._relu(h, ih, "head relu", mut="head_relu_dropped")
        o, io = self.add("conv_gemm", "head 1x1 (fp32 NCHW)", lambda M: head_out(hr, sd, M), {"srcs": [ihr]})
        return self.add("relu_f32", "relu fp32", lambda M: _exact(o.v.clamp_min(0), M), {"x": io})

    # ---------------------------------------------------------------- BiT backbone and token GEMM
    def gn(self, x, ix, gamma, beta):
        """_HybridPlan._gn_act without a shortcut: the statistics launch, then GN + ReLU."""
        self.add({"gn_stats", "gn_finalize"}, "gn statistics", lambda M: Stats(x, M), {"x": ix})
        return self.add("gn_act_f16", "gn_act (GN + ReLU)", lambda M: gn_act(x, gamma, beta, M), {"x": ix})

    def bottleneck(self, sd, lp, x, ix, stride2_):
        w = lambda k: sd[lp + k]  # noqa: E731
        ws = lambda k, M: standardized(w(k), M)  # noqa: E731
        r = ir = rn = None
        if (lp + "downsample.conv.weight") in sd:
            xs, ixs = x, ix
            if stride2_:
                xs, ixs = self.add("subsample2", "subsample", lambda M: _exact(x.v[:, ::2, ::2], M), {"x": ix})
            r, ir = self.add("conv_gemm", "bit 1x1", lambda M: gemm(xs, ws("downsample.conv.weight", M), None, M),
                             {"srcs": [ixs]}, muts=("ws_off",))
            self.add({"gn_stats", "gn_finalize"}, "gn statistics", lambda M: Stats(r, M), {"x": ir})
            rn = (w("downsample.norm.weight"), w("downsample.norm.bias"))
        c1, ic1 = self.add("conv_gemm", "bit 1x1", lambda M: gemm(x, ws("conv1.weight", M), None, M), {"srcs": [ix]},
                           muts=("ws_off",))
        a, ia = self.gn(c1, ic1, w("norm1.weight"), w("norm1.bias"))
        full, ifull = self.add("conv_gemm", "bit conv3x3", lambda M: conv3(a, ws("conv2.weight", M), None, M),
                               {"srcs": [ia]}, muts=("ws_off",))
        c2, ic2 = full, ifull
        if stride2_:
            ref2 = lambda M: _nhwc(F.conv2d(F.pad(_nchw(a.v), (0, 1, 0, 1)), ws("conv2.weight", M), stride=2))  # noqa: E731
            chk = ("bit conv3x3 stride 2 (conv2d, TF-SAME)",
                   lambda M: stride2(conv3(a, ws("conv2.weight", M), None, M) if (M.bound or M.em) else full, ref2(M), 1, M,
                                     "bit_sub00"), ("bit_sub00",))
            c2, ic2 = self.add("subsample2", "subsample", lambda M: _exact(full.v[:, 1::2, 1::2], M), {"x": ifull},
                               also=[chk])
        a2, ia2 = self.gn(c2, ic2, w("norm2.weight"), w("norm2.bias"))
        c3, ic3 = self.add("conv_gemm", "bit 1x1", lambda M: gemm(a2, ws("conv3.weight", M), None, M), {"srcs": [ia2]},
                           muts=("ws_off",))
        self.add({"gn_stats", "gn_finalize"}, "gn statistics", lambda M: Stats(c3, M), {"x": ic3})
        reads = {"x": ic3, "r": ir if r is not None else ix}
        kind = "gn_act (GN + GN(shortcut) + ReLU)" if rn is not None else "gn_act (GN + shortcut + ReLU)"
        sc = r if r is not None else x
        return self.add("gn_act_f16", kind, lambda M: gn_act(c3, w("norm3.weight"), w("norm3.bias"), M, r=sc, rn=rn), reads,
                        muts=("down_no_gn",) if rn is not None else ())

    def bit(self, sd, cfg, pix, kst=192):
        """_HybridPlan's BiT backbone over fp32 pixels [B, 3, h, w] -> [(stage map, index)] x 3; kst: the im2col rows' width
        (147 columns, zeros after)."""
        bp = "dpt.embeddings.backbone.bit."
        B, _, h, w = pix.shape

        def cols(M):
            pt, pb = (3, 2) if M.mut == "im2col_pads_32" else (2, 3)
            u = F.unfold(F.pad(pix.double(), (pt, pb, pt, pb)), 7, stride=2).transpose(1, 2).reshape(B, h // 2, w // 2, 147)
            return _exact(F.pad(u if _pure(M) else u.float().half().double(), (0, kst - 147)), M)
        rows, irows = self.add("im2col_f16", "im2col 7x7 stride 2", cols, muts=("im2col_pads_32",))
        s0, is0 = self.add("conv_gemm", "bit stem (K 147)", lambda M: gemm(V(rows.v[..., :147]), standardized(
            sd[bp + "embedder.convolution.weight"], M), None, M), {"srcs": [irows]}, muts=("ws_off",))
        a0, ia0 = self.gn(s0, is0, sd[bp + "embedder.norm.weight"], sd[bp + "embedder.norm.bias"])
        pooled, ip = self.add("maxpool_f16", "maxpool 3x3 stride 2", lambda M: _exact(_nhwc(F.max_pool2d(
            F.pad(_nchw(a0.v), (0, 1, 0, 1), value=0.0), 3, 2)), M), {"x": ia0})
        maps, x, ix = [], pooled, ip
        for s, depth in enumerate(cfg["backbone_config"]["depths"]):
            for l in range(depth):
                x, ix = self.bottleneck(sd, f"{bp}encoder.stages.{s}.layers.{l}.", x, ix, s > 0 and l == 0)
            maps.append((x, ix))
        return maps

    def tokens(self, sd, last, ilast, kp, grid):
        """The token GEMM: rows [CLS (a 1 in column C3) | the last stage map] over the [projection | CLS] weight, the resized
        position embedding (+ the projection bias on the patch rows, held in fp16) as residual.  -> (V [B, T, H], index)."""
        B, gh, gw, C3 = last.v.shape
        T = gh * gw + 1
        rows = torch.zeros(B, T, kp, dtype=torch.float64, device=last.v.device)
        rows[:, 0, C3] = 1
        rows[:, 1:, :C3] = last.v.reshape(B, gh * gw, C3)
        Wp = sd["dpt.embeddings.projection.weight"].double().reshape(-1, C3)
        H = Wp.shape[0]
        Wt = torch.cat([Wp, sd["dpt.embeddings.cls_token"].double().reshape(H, 1)], 1)
        pos = sd["dpt.embeddings.position_embeddings"].double()[0]
        g0 = int(round((pos.shape[0] - 1) ** 0.5))
        grid_pos = F.interpolate(pos[1:].reshape(1, g0, g0, H).permute(0, 3, 1, 2), size=(gh, gw), mode="bilinear")
        res = torch.cat([pos[:1], grid_pos.permute(0, 2, 3, 1).reshape(gh * gw, H)])
        bias = sd["dpt.embeddings.projection.bias"].double()
        res[1:] += bias
        pamax = pos.abs().amax()

        def f(M):
            rr = res.roll(1, 0) if M.mut == "pos_shift" else res
            rv = rr.expand(B, T, H)
            if M.em:
                rv = rv.float().half().double()
            o = gemm(V(rows[..., :C3 + 1]), Wt, None, M, res=V(rv))
            if not M.bound:
                return o
            # the host's fp32 position resize and bias add, then the fp16 residual
            return V(o.v, o.e + U16 * rv.abs() + TINY + 8 * U * (pamax + bias.abs()))
        return self.add("gemm_rows", "token gemm", f, {"x": rows.half()}, muts=("pos_shift",))

    # ---------------------------------------------------------------- hint stem
    def hint(self, sd, hint):
        """UNet.hint_features over fp32 hint [N, 3, 8h, 8w] -> (fp32 NCHW [N, 4, h, w], index).  stem_im2col's rows: 64
        columns, k = tap * 3 + c, zeros from 27."""
        from oracle.controlnet_oracle import HINT_CHANNELS
        N, _, Hh, Wh = hint.shape

        def cols(M):
            u = F.unfold(F.pad(hint.double(), (1, 1, 1, 1)), 3).reshape(N, 3, 9, Hh * Wh).transpose(1, 2)
            u = u.reshape(N, 27, Hh, Wh).permute(0, 2, 3, 1)
            return _exact(F.pad(u if _pure(M) else u.float().half().double(), (0, 64 - 27)), M)
        x, ix = self.add("stem_im2col", "stem_im2col", cols)
        last_i = len(HINT_CHANNELS) - 1
        for i, (ci, co, stride) in enumerate(HINT_CHANNELS):
            W = sd[f"add_embedding.input_hint_block.{2 * i}.weight"]
            b = sd[f"add_embedding.input_hint_block.{2 * i}.bias"]
            if i == 0:
                Wr = W.double().permute(0, 2, 3, 1).reshape(co, 27)
                x, ix = self.add("conv_gemm", "hint conv (stem rows)", lambda M, x=x: gemm(V(x.v[..., :27]), Wr, b.double(), M),
                                 {"srcs": [ix]})
            elif i == last_i:
                o, io = self.add("conv_gemm", "hint conv (fp32 NCHW)", lambda M, x=x, W=W, b=b: conv3(x, W, b, M, out16=False),
                                 {"srcs": [ix]})
                return o, io
            else:
                x, ix = self.add("conv_gemm", "hint conv3x3", lambda M, x=x, W=W, b=b: conv3(x, W, b, M), {"srcs": [ix]})
            if stride == 2:
                full, ifull = x, ix
                x, ix = self.add("subsample2", "subsample", lambda M, full=full: _exact(full.v[:, ::2, ::2], M), {"x": ifull})
            mut = "hint_no_silu" if i == 3 else None
            x, ix = self.add("silu_f16_", "silu", lambda M, x=x, mut=mut: silu(x, M, mut), {"x": ix},
                             muts=(mut,) if mut else ())


def conv3_res(a, W, b, x, M):
    """conv3x3(a) + b + the residual x (the fusion unit2's last conv)."""
    return conv_fused(a, W, b, x, None, M)


def head_out(x, sd, M):
    """head.head.4: 1x1 to one channel, fp32 NCHW out (out_mode 1)."""
    return conv([(_map(x, _nchw), sd["head.head.4.weight"], "1x1")], [sd["head.head.4.bias"]], M, out16=False)


def silu(x, M, mut=None):
    """silu_f16_ in place: SiLU of fp16 x, one rounding (_silu_allow before it)."""
    if M.mut is not None and M.mut == mut:
        return V(x.v)
    v = _silu64(x.v)
    if M.em:
        return V(v.half().double())
    if not M.bound:
        return V(v)
    return V(v, _silu_allow(x.v) + U16 * v.abs() + TINY)


# ------------------------------------------------------------------------------------------------------------------------------
# whole models (the plans' order)
# ------------------------------------------------------------------------------------------------------------------------------
def dpt(wk, sd, cfg, hidden, grid):
    """_DepthPlan after the layers: hidden = the hidden states after backbone_out_indices (V [B, T, H])."""
    c = dict(cfg)
    feats = [wk.reassemble(sd, c, i, hs, grid) for i, hs in enumerate(hidden)]
    return wk.fuse_head(sd, feats)


def hybrid(wk, sd, cfg, pix, kp, vit):
    """_HybridPlan outside the layers: vit(tokens V) -> the two hidden states the neck reads (the layers are not restated
    here; the GPU test passes the plan's own, the CPU test a float64 stack)."""
    B, _, h, w = pix.shape
    grid = (h // 16, w // 16)
    maps = wk.bit(sd, cfg, pix)
    emb, iemb = wk.tokens(sd, maps[2][0], maps[2][1], kp, grid)
    h1, h2 = vit(emb)
    feats = [wk.add("conv_gemm", "neck conv3x3", lambda M, m=m: conv3(m, sd[f"neck.convs.{i}.weight"], None, M),
                    {"srcs": [im]}) for i, (m, im) in enumerate(maps[:2])]
    feats += [wk.reassemble(sd, cfg, 2, h1, grid), wk.reassemble(sd, cfg, 3, h2, grid)]
    return wk.fuse_head(sd, feats), maps

