"""GPU: k2_conv_gemm beyond the 3x3 body convolutions -- the flat-row GEMMs of every transformer tower (both diffusion priors,
the CLIP ViT-bigG text and image towers, XLM-RoBERTa-large), the UNet's and the MoVQ's attention projections, the MoVQ
ResBlock with its nin_shortcut as a second K segment, the fp32 NCHW output heads (out_mode 1), the per-row epilogue fallback
(Cout % 64 != 0, split-K with Cout % 32 != 0) and the k2_stem_im2col stems -- at the geometry the models build
(tests/gemm_ref.py derives it; tests/test_cpu_gemm_geometry.py pins the list).

Every case runs in two modes, each over every launch configuration the autotuner could bake in (launch_plan.tune): the
library's own choice, N tiles 128 / 192 / 256 x epilogue warp sets 1 / 2, and split-K 2, 3, 4 at each N tile wherever the
library accepts the split (k2_conv_plan says so without a launch).
  exact   integer operands (tests/gemm_ref.py): the output must equal the rounding of the exact sum bit for bit, which pins
          every index, tile, split, K chunk, bias column, residual row and epilogue path;
  random  Gaussian fp16 data against float64 with tests/test_gpu_conv_float64.py's bound: the output's rounding plus fp32
          accumulation over K terms, + 2 for bias and residual, + the number of splits for the split-K finalize pass.
          Configurations with the same split factor must agree bit for bit (N tile and epilogue sets never change a result),
          and every split must repeat itself bit for bit.
Each case prints its worst share of the bound (run with -s)."""
import pytest
import torch

from tests.gemm_ref import Gemm, all_gemms, check_exact, exact_expected, exact_scale, ints, scale_odd_rows
from tests.test_gpu_conv_float64 import EPS16, _check, _conv64

pytestmark = pytest.mark.gpu

CASES = all_gemms()


def _configs(c):
    """Launch configurations (k2_conv_gemm_cfg's cfg, None = automatic) the tuner could pick for this launch."""
    from kandinsky2 import ops
    NB, H, W = c.geom
    taps = 9 if any(t == 9 for _, t in c.srcs) else 1
    plan = lambda: ops.conv_plan(NB, H, W, taps, c.ktot, c.cout, out_mode=c.out_mode, want_gn_partial=False)  # noqa: E731
    auto = plan()
    bns = [bn for bn in (128, 192, 256) if bn - 64 < c.cout] if c.cout > 64 else [auto["n_tile"]]
    splits = [1]
    for sp in (2, 3, 4):
        ops.set_tuning(1, sp)
        try:
            if plan()["splits"] == sp:
                splits.append(sp)
        finally:
            ops.set_tuning(1, 0)
    cfgs = [None]
    for sp in splits:
        for bn in bns:
            for es in ((1, 2) if bn in (128, 256) else (1,)):
                cfgs.append((bn, 1, sp, es))
    return cfgs


def _operands(c, mode, seed):
    """(sources for the launch, packed weight, bias, residual, reference function) of case c."""
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(seed)
    NB, H, W = c.geom
    dev = "cuda"
    exact = mode == "exact"
    s = exact_scale(c.k_terms)

    def act(*shape):
        return ints(g, shape, device=dev) if exact else torch.randn(*shape, device=dev, generator=g).half()

    def weight(*shape):
        if exact:
            return scale_odd_rows(ints(g, shape, device=dev), s)
        return (torch.randn(*shape, device=dev, generator=g) / c.k_terms ** 0.5).half()

    bias = ints(g, (c.cout,), lim=64, device=dev, dtype=torch.float32) if exact else torch.randn(c.cout, device=dev, generator=g)
    res = None
    if c.residual:
        res = ints(g, (NB, H, W, c.cout), lim=64, device=dev) if exact else torch.randn(NB, H, W, c.cout, device=dev,
                                                                                       generator=g).half()
    if c.stem:
        cx, c2, c3, mul23 = c.stem
        f32 = lambda ch: (ints(g, (NB, ch, H, W), device=dev, dtype=torch.float32) if exact  # noqa: E731
                          else torch.randn(NB, ch, H, W, device=dev, generator=g))
        x, x2, x3 = f32(cx), f32(c2) if c2 else None, f32(c3) if c3 else None
        kpad = c.srcs[0][0]
        patches = ops.stem_im2col(x, x2, x3, mul23=bool(mul23), kpad=kpad)
        check_exact(patches, _im2col(x, x2, x3, mul23, kpad), f"{c.name}: stem_im2col")
        w = weight(c.cout, sum(c.stem[:3]), 3, 3)
        wp = ops.pad_rows(ops.pack_stem_weight(w), c.w_rows)
        srcs = [(patches, 1)]

        def ref(absolute):
            a, b = patches.double(), wp[:c.cout].double()
            if absolute:
                a, b = a.abs(), b.abs()
            return (a.reshape(-1, kpad) @ b.T).reshape(NB, H, W, c.cout)
        return srcs, wp, bias, res, ref
    xs = [act(NB, H, W, C) for C, _ in c.srcs]
    ws = [weight(c.cout, C, 3, 3) if t == 9 else weight(c.cout, C) for C, t in c.srcs]
    wp = torch.cat([ops.pack_conv_weight(w) for w in ws], 1).contiguous()
    wp = ops.pad_rows(wp, c.w_rows)
    srcs = list(zip(xs, [t for _, t in c.srcs]))

    def ref(absolute):
        out = 0
        for (x, t), w in zip(srcs, ws):
            xa, wa = (x.abs(), w.abs()) if absolute else (x, w)
            if t == 9:
                out = out + _conv64(xa, wa, 1)
            else:
                out = out + (xa.double().reshape(-1, xa.shape[-1]) @ wa.double().T).reshape(NB, H, W, c.cout)
        return out
    return srcs, wp, bias, res, ref


def _im2col(x, x2, x3, mul23, kpad):
    """torch construction of k2_stem_im2col: fp16 [NB, H, W, kpad], k = tap * Cin + c over cat(x, x2 (* x3[:, :1]), x3)."""
    parts = [x]
    if x2 is not None:
        parts.append(x2 * x3[:, :1] if mul23 else x2)
    if x3 is not None:
        parts.append(x3)
    xc = torch.cat(parts, 1)
    NB, cin, H, W = xc.shape
    xp = torch.nn.functional.pad(xc, (1, 1, 1, 1))
    taps = [xp[:, :, ky:ky + H, kx:kx + W] for ky in range(3) for kx in range(3)]
    cols = torch.stack(taps, 1).permute(0, 3, 4, 1, 2).reshape(NB, H, W, 9 * cin)
    out = torch.zeros(NB, H, W, kpad, device=x.device, dtype=torch.float16)
    out[..., :9 * cin] = cols.half()
    return out


def _run(c, srcs, wp, bias, res, cfg):
    from kandinsky2 import ops
    info = [0] * 7
    if c.rows:
        x = srcs[0][0].reshape(c.m, -1)
        y = ops.gemm_rows(x, wp, c.cout, bias=bias, residual=None if res is None else res.reshape(c.m, c.cout), cfg=cfg,
                          info=info)
        y = y.view(c.geom + (c.cout,))
    else:
        y = ops.conv_gemm(srcs, wp, c.cout, bias=bias, residual=res, out_mode=c.out_mode, cfg=cfg, info=info)
    return y, info


def _to_out(c, t):
    """NHWC float64 -> the launch's output layout (NCHW for out_mode 1)."""
    return t.permute(0, 3, 1, 2) if c.out_mode == 1 else t


@pytest.mark.parametrize("mode", ["exact", "random"])
@pytest.mark.parametrize("c", CASES, ids=[c.name for c in CASES])
def test_gemm_vs_float64(c: Gemm, mode):
    srcs, wp, bias, res, ref = _operands(c, mode, seed=len(c.name) * 7919 + c.m + c.cout)
    acc = ref(False) + bias.double()
    if res is not None:
        acc = acc + res.double()
    acc = _to_out(c, acc)
    out_dtype = torch.float16 if c.out_mode == 0 else torch.float32
    runs = {}   # effective split factor -> first output
    worst, seen = 0.0, []
    if mode == "exact":
        # the exact sum is an integer; rounding removes whatever a float64 convolution algorithm may leave behind
        want = exact_expected(acc.round(), out_dtype)
        if c.out_mode == 0:
            assert (acc.abs() > 2048).any(), "no exact sum above 2048: fp16-precision accumulation would go unnoticed"
    else:
        absum = ref(True) + bias.double().abs()
        if res is not None:
            absum = absum + res.double().abs()
        absum = _to_out(c, absum)
    for cfg in _configs(c):
        y, info = _run(c, srcs, wp, bias, res, cfg)
        torch.cuda.synchronize()
        sp = info[2]
        seen.append((cfg, info[0], sp))
        what = f"{c.name} {mode} cfg={cfg} (N tile {info[0]}, splits {sp})"
        if cfg is not None:
            assert (info[0], info[2]) == (cfg[0], cfg[2]), (what, info)
        if mode == "exact":
            check_exact(y, want, what)
            continue
        k_terms = c.k_terms + 2 + (sp if sp > 1 else 0)
        worst = max(worst, _check(y, acc, absum, k_terms, eps_out=EPS16 if c.out_mode == 0 else 0.0))
        if sp in runs:
            check_exact(y, runs[sp], f"{what}: differs from another configuration with the same split factor")
        else:
            runs[sp] = y.clone()
        if sp > 1:
            y2, _ = _run(c, srcs, wp, bias, res, cfg)
            torch.cuda.synchronize()
            check_exact(y2, y, f"{what}: a second run differs")
    splits = sorted({s for _, _, s in seen})
    if mode == "exact":
        print(f"{c.name}: bit-exact in {len(seen)} configurations (splits {splits})")
    else:
        print(f"{c.name}: {len(seen)} configurations (splits {splits}), worst {worst:.3f} of the bound")
