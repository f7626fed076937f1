"""GPU: GroupNorm statistics, the fused normalise (+FiLM) (+SiLU) (+resample) (+concat) apply, SpatialNorm and SiLU against
float64 evaluations of the same fp16 tensors, at the UNet's and the MoVQ decoder's real geometry.

The reference statistics are exact two-pass float64 mean / variance of the fp16 values the kernel reads, one image at a time.
Every bound is in fp16 ulps of the float64 output (`_ulp16`) plus absolute terms for what the kernels' fp32 arithmetic can
legitimately move, each derived where it is computed:
  - the apply evaluates t = fma(x, A, B) with A = gamma rstd (1 + s), B = (beta - mean A')(1 + s) + shift: a handful of fp32
    roundings of the terms |x A|, |mean A|, |beta (1 + s)|, |shift|, which cancel where x ~ mean (2^-20 of their sum);
  - statistics that come from fp32 partial sums carry that format's error (`_stats_allowance`);
  - SiLU's own error is <= 2^-20 + 2^-23 |t| relative (k2_common.cuh silu_f), and its slope is at most 1.1.
Each test prints its worst error in ulps and its largest share of the bound (run with -s)."""
import math

import pytest
import torch
import torch.nn.functional as F

from tests.test_gpu_prior_kernels import _ulp16

pytestmark = pytest.mark.gpu

U = 2.0 ** -24          # fp32 unit roundoff
SILU_SLOPE = 1.1        # max |d silu / dt| = 1.0998
CHAIN_PARTIAL = 21      # longest fp32 chain behind one conv partial: 16 rows per half warp, + the other half, + 4 warps
# stated figures for the conv partials' mean (in std) and rstd error at mean / std 10 and 100, with about 2x margin over
# the worst measured on an H100 (2^-16.9 and 2^-10.1, the 8-image ragged boxes): the raw fp32 (sum, sumsq) format is below
# one fp16 ulp of rstd at 10 and not at 100
PARTIAL_REL = {10.0: 2.0 ** -15, 100.0: 2.0 ** -9}


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


def _silu64(t):
    return t * torch.sigmoid(t)


def _silu_allow(t):
    return (2.0 ** -20 + 2.0 ** -23 * t.abs()) * _silu64(t).abs()


# ------------------------------------------------------------------------------------------------------------------------------
# geometry: derived from the model code, not chosen here
# ------------------------------------------------------------------------------------------------------------------------------
def _unet_norms():
    """{(H, C0, C1, resample)} of the ResBlock GroupNorms of bench.py's UNet at 768 x 768 (latent 96 x 96): C1 > 0 where the
    up path's input is the concat [h | skip]; resample 1 / 2 for the down / up ResBlocks (in-norm with h_upd / x_upd)."""
    import bench
    from kandinsky2.model.unet import _topology
    cfg = bench.UNET_CFG
    mc, mult, nrb = cfg["model_channels"], tuple(cfg["channel_mult"]), cfg["num_res_blocks"]
    inp, mid, out = _topology(cfg["in_channels"], mc, mult, nrb, tuple(cfg["attention_resolutions"]))
    H, shapes, chans = 96, set(), []
    for blk in inp:
        for item in blk:
            if item[0] == "res":
                _, cin, cout, ud = item
                shapes.add((H, cin, 0, 1 if ud == "down" else 0))
                if ud == "down":
                    H //= 2
                shapes.add((H, cout, 0, 0))
        chans.append([it for it in blk if it[0] in ("conv", "res")][-1][2])
    for item in mid:
        if item[0] == "res":
            shapes.add((H, item[1], 0, 0))
    for blk in out:
        for item in blk:
            if item[0] == "res":
                _, cin, cout, ud = item
                if ud is None:
                    skip = chans.pop()
                    shapes.add((H, cin - skip, skip, 0))
                else:
                    shapes.add((H, cin, 0, 2))
                    H *= 2
                shapes.add((H, cout, 0, 0))
    return sorted(shapes)


def _movq_norms(latent=96):
    """[(H, C)] of the MoVQ decoder's SpatialNorms (CONFIG_2_2's ddconfig) for a latent x latent input."""
    from kandinsky2 import configs
    from kandinsky2.vqgan.autoencoder import _topology
    dd = configs.CONFIG_2_2["image_enc_params"]["params"]["ddconfig"]
    block_in, levels = _topology(dd)
    H, out = latent, {(latent, block_in)}
    for lv in levels:
        for cin, cout in lv["blocks"]:
            out.add((H, cin))
            out.add((H, cout))
        if lv["up"]:
            H *= 2
    return sorted(out)


def test_derived_geometry_is_the_issue_geometry():
    """The shapes below are what the model code builds: cfg-2 levels 96 / 48 / 24 / 12 at 384 / 768 / 1152 / 1536 channels, the
    up path's straddling concats, and MoVQ's 512 @ 96, 256 @ 192 / 384, 128 @ 768."""
    un = _unet_norms()
    assert {(h, c0 + c1) for h, c0, c1, _ in un} >= {(96, 384), (48, 768), (24, 1152), (12, 1536)}
    cats = {(h, c0, c1) for h, c0, c1, _ in un if c1}
    for h, c0, c1 in ((12, 1536, 1152), (24, 1152, 768), (48, 768, 384)):
        assert (h, c0, c1) in cats, cats
    assert {r for *_, r in un} == {0, 1, 2}
    mv = _movq_norms()
    assert {(96, 512), (192, 256), (384, 256), (768, 128)} <= set(mv), mv


# ------------------------------------------------------------------------------------------------------------------------------
# inputs
# ------------------------------------------------------------------------------------------------------------------------------
RATIOS = (10.0, 100.0, 300.0, 1000.0)


def _channel_stats(kind, NB, C, cpg, eps, seed, ratio=None):
    """Per (image, channel) (mean, std) of the kind, following _ln_rows of test_gpu_prior_kernels; cpg channels per group.
    `ratio` puts every group of an `offset` input at that mean / std (alternating signs between groups)."""
    g = _gen(seed)
    mean = torch.zeros(NB, C, device="cuda", dtype=torch.float64)
    std = torch.ones(NB, C, device="cuda", dtype=torch.float64)
    sign = torch.where(torch.arange(NB, device="cuda") % 2 == 0, 1.0, -1.0).double()[:, None]
    gi = torch.arange(C, device="cuda") // cpg
    if kind == "offset":          # group mean / std of 10, 100, 300 and 1000, both signs
        mean = sign * torch.tensor(RATIOS, device="cuda", dtype=torch.float64)[gi % 4][None, :]
        if ratio is not None:
            mean = sign * ratio * torch.where(gi % 2 == 0, 1.0, -1.0).double()[None, :]
    elif kind == "constant":      # zero variance: every output of a group is act(beta (1 + s) + shift)
        mean = torch.tensor([0.0, 0.3, -7.5, 1000.0], device="cuda", dtype=torch.float64)[gi % 4][None, :].expand(NB, C)
        std = torch.zeros(NB, C, device="cuda", dtype=torch.float64)
    elif kind == "tiny_var":      # variance 0.09 eps: eps decides rstd
        std = std * 0.3 * math.sqrt(eps)
    elif kind == "massive":       # one channel of each image at +-3e4 in otherwise O(1) data
        mean = mean.clone()
        mean[torch.arange(NB, device="cuda"), (torch.arange(NB, device="cuda") * 7 + 3) % C] = sign[:, 0] * 3e4
    elif kind == "mixed_means":   # the group's variance is mostly between its channels
        mean = 8.0 * torch.randn(NB, C, device="cuda", generator=g, dtype=torch.float64)
    return mean, std


def _direct_input(kind, NB, H, W, C, groups, eps, seed):
    mean, std = _channel_stats(kind, NB, C, C // groups, eps, seed)
    z = torch.randn(NB, H, W, C, device="cuda", generator=_gen(seed + 1))
    return (z.double() * std[:, None, None, :] + mean[:, None, None, :]).half()


def _conv_input(kind, NB, H, W, C, cpg, eps, seed, cin=64, taps=9, cfg=None, ratio=None):
    """The tensor through the producing conv: the bias sets each channel's mean, the weight scale its std (a zero weight with a
    bias gives a constant).  Returns (y, partials, row groups per image, info)."""
    from kandinsky2 import ops
    mean, std = _channel_stats(kind, 1, C, cpg, eps, seed, ratio)
    mean, std = mean[0], std[0]
    g = _gen(seed + 2)
    Hi, Wi = (H // 2, W // 2) if taps == 4 else (H, W)
    x = torch.randn(NB, Hi, Wi, cin, device="cuda", generator=g).half()
    w = torch.randn(C, cin, 3, 3, device="cuda", generator=g) / (3 * cin ** 0.5) * std[:, None, None, None].float()
    wp = ops.pack_conv_weight_up2(w) if taps == 4 else ops.pack_conv_weight(w)
    part = torch.full((ops.gn_part_floats(NB, H, W, C),), float("nan"), device="cuda")
    info = [0] * 7
    y = ops.conv_gemm([(x, taps)], wp, C, bias=mean.float(), gn_part=part, info=info, cfg=cfg)
    assert info[5] in (1, 2) and info[6] % NB == 0, info
    return y, part, info[6] // NB, info


# ------------------------------------------------------------------------------------------------------------------------------
# float64 reference and bounds
# ------------------------------------------------------------------------------------------------------------------------------
def _ref_stats(xn, groups):
    """Exact two-pass statistics of one image [H, W, C] (float64): (mean [G], var [G], mean |x - p| [G], mean (x - p)^2 [G],
    mean |x| [G], mean x^2 [G]) with p = the channel's value at the first pixel (gn_stats' pivot)."""
    HW, C = xn.shape[0] * xn.shape[1], xn.shape[2]
    x = xn.reshape(HW, groups, C // groups)
    mean = x.mean((0, 2))
    var = ((x - mean[None, :, None]) ** 2).mean((0, 2))
    d = x - x[:1]
    return mean, var, d.abs().mean((0, 2)), (d * d).mean((0, 2)), x.abs().mean((0, 2)), (x * x).mean((0, 2))


def _stats_allowance(source, rs, eps, chain):
    """(mean error, relative rstd error) per group that the statistics' own arithmetic may leave, from fp32 sums whose longest
    rounding chain is `chain` terms: a sum of terms t_i is off by <= chain U sum |t_i|.
      gn_stats: sums of d = x - pivot (exact) and d^2; mean off by chain U mean|d|, variance by 3 chain U mean d^2.
      conv partials: raw sums of x and x^2 (the format the epilogue writes); the same with x for d.
    Both then fold in float64 and round mean and rstd to fp32 (U, U).
      "partials_measured": the conv partials held to the stated figure `chain` (PARTIAL_REL) of std on the mean and of rstd."""
    mean, var, ad, d2, ax, x2 = rs
    if source == "partials_measured":
        return chain * var.sqrt() + 2 * U * mean.abs(), torch.full_like(var, chain + 2 * U)
    a1, a2 = (ad, d2) if source == "stats" else (ax, x2)
    e_mean = chain * U * a1 + U * mean.abs()
    e_rel = 3 * chain * U * (a2 + 2 * mean.abs() * a1) / (2 * (var + eps)) + 2 * U
    return e_mean, e_rel


def _check_stats(st, x_imgs, groups, eps, source, chain, what):
    """st: [NB, G, 2] (mean, rstd) from the kernel vs float64; returns the worst share of the bound."""
    worst = 0.0
    for n, xn in enumerate(x_imgs):
        rs = _ref_stats(xn, groups)
        mean, var = rs[0], rs[1]
        rstd = 1.0 / torch.sqrt(var + eps)
        e_mean, e_rel = _stats_allowance(source, rs, eps, chain)
        dm = (st[n, :, 0].double() - mean).abs()
        dr = (st[n, :, 1].double() - rstd).abs() / rstd
        assert (dm <= e_mean).all(), (what, "mean", n, dm.max().item(), mean[dm.argmax()].item(), e_mean[dm.argmax()].item())
        assert (dr <= e_rel).all(), (what, "rstd", n, dr.max().item(), var[dr.argmax()].item(), e_rel[dr.argmax()].item())
        worst = max(worst, (dm / e_mean).max().item(), (dr / e_rel).max().item())
    return worst


def _image(srcs, n):
    return torch.cat([s[n].double() for s in srcs], -1)


def _check_apply(y, srcs, groups, eps, gamma, beta, film, act, resample, source, chain, what, xres=None, mod=None):
    """y (fp16 NHWC) of gn_apply / gn_apply_fold / sn_apply against float64 with exact statistics.  mod = (my, mb) fp64
    [NB, H, W, C] SpatialNorm modulation and its magnitude (|my|, |mb| term sums) instead of FiLM.  Returns (worst ulps,
    worst share of the bound)."""
    NB = y.shape[0]
    C = sum(s.shape[-1] for s in srcs)
    cpg = C // groups
    gd, bd = gamma.double(), beta.double()
    ulps = share = 0.0
    for n in range(NB):
        x = _image(srcs, n)
        rs = _ref_stats(x, groups)
        mean, var = rs[0], rs[1]
        rstd = 1.0 / torch.sqrt(var + eps)
        e_mean, e_rel = _stats_allowance(source, rs, eps, chain)
        mu, rho = mean.repeat_interleave(cpg), rstd.repeat_interleave(cpg)
        em, er = e_mean.repeat_interleave(cpg), e_rel.repeat_interleave(cpg)
        xc = x - mu
        if mod is None:
            sc = 1 + film[n, :C].double() if film is not None else torch.ones_like(gd)
            sh = film[n, C:2 * C].double() if film is not None else torch.zeros_like(gd)
            A = gd * rho * sc
            t = xc * A + bd * sc + sh
            terms = (x * A).abs() + (mu * A).abs() + (bd * sc).abs() + sh.abs()
            scale = A.abs()
        else:
            my, mb, my_abs, mb_abs = (m[n] for m in mod)
            A = gd * rho
            t = (xc * A + bd) * my + mb
            terms = ((x * A).abs() + (mu * A).abs() + bd.abs()) * my_abs + mb_abs
            scale = A.abs() * my.abs()
        # fp32 evaluation of the affine: at most ten roundings (mean and rstd to fp32, gamma rstd, its products, beta - mean A,
        # the modulation's or FiLM's fmas, the final fma), each of at most U times the terms; then the statistics' allowance
        allow = 2.0 ** -20 * terms + scale * em + (xc * A).abs() * (my.abs() if mod is not None else 1) * er
        if act:
            o, allow = _silu64(t), SILU_SLOPE * allow + _silu_allow(t)
        else:
            o = t
        if resample == 1:
            # the kernel rounds each activation to fp16 before the 2 x 2 average (as the reference's fp16 graph does)
            pool = lambda v: F.avg_pool2d(v.permute(2, 0, 1)[None], 2)[0].permute(1, 2, 0)  # noqa: E731
            ref, allow = pool(o), pool(allow + 0.5 * _ulp16(o))
        elif resample == 2:
            up = lambda v: v.repeat_interleave(2, 0).repeat_interleave(2, 1)  # noqa: E731
            ref, allow = up(o), up(allow)
        else:
            ref = o
        got = y[n].double()
        err = (got - ref).abs()
        bound = _ulp16(ref) + allow
        bad = ~(err <= bound)
        assert not bad.any(), (what, n, int(bad.sum()), err[bad][:4].tolist(), ref[bad][:4].tolist(), bound[bad][:4].tolist())
        ulps = max(ulps, (err / _ulp16(ref)).max().item())
        share = max(share, (err / bound).max().item())
        if xres is not None:
            if resample == 1:
                rx = F.avg_pool2d(x.permute(2, 0, 1)[None], 2)[0].permute(1, 2, 0)
                assert ((xres[n].double() - rx).abs() <= _ulp16(rx)).all(), (what, "xres")
            else:
                rx = x if resample == 0 else x.repeat_interleave(2, 0).repeat_interleave(2, 1)
                assert torch.equal(xres[n].double(), rx), (what, "xres")
    return ulps, share


def _affine(C, seed, film_nb=None):
    g = _gen(seed)
    gamma = 1 + 0.5 * torch.randn(C, device="cuda", generator=g)
    beta = 0.5 * torch.randn(C, device="cuda", generator=g)
    film = 0.3 * torch.randn(film_nb, 2 * C, device="cuda", generator=g) if film_nb else None
    return gamma, beta, film


def _report(what, ulps, share, stat_share=None):
    s = f", statistics at {stat_share:.2f} of their bound" if stat_share is not None else ""
    print(f"{what}: worst {ulps:.2f} ulp, {share:.2f} of the bound{s}")


# ------------------------------------------------------------------------------------------------------------------------------
# 1. gn_stats -> gn_apply at every UNet ResBlock norm shape and the MoVQ shapes
# ------------------------------------------------------------------------------------------------------------------------------
_KINDS = ("randn", "offset", "constant", "tiny_var", "massive", "mixed_means")


def _unet_cases():
    cases = []
    for i, (H, C0, C1, rs) in enumerate(_unet_norms()):
        NB = 8
        extra = _KINDS[2 + i % 4]
        for kind in ("randn", "offset", extra):
            cases.append((NB, H, C0, C1, rs, kind))
    cases.append((4, 128, 384, 0, 0, "randn"))      # cfg-3: NB = 4 at 128 x 128
    cases.append((4, 128, 384, 0, 0, "offset"))
    return cases


def _stats_chain(NB, HW, C):
    """Longest fp32 chain of gn_stats: the pixels one lane sums in its chunk, then the 16 lanes."""
    from kandinsky2 import _native as nat
    chunks = (nat.load().k2_gn_scratch_floats(NB, HW, C) - 1024) // (NB * C * 2)
    chunk = -(-HW // chunks)
    return -(-chunk // 16) + 16


@pytest.mark.parametrize("NB,H,C0,C1,resample,kind", _unet_cases())
def test_gn_stats_apply_unet_vs_float64(NB, H, C0, C1, resample, kind):
    """k2_gn_stats -> k2_gn_apply with FiLM + SiLU (and act = 0 on the randn inputs), the up path's concat read as two sources,
    resample with xres where the ResBlock resamples."""
    from kandinsky2 import ops
    W, C, eps = H, C0 + C1, 1e-5
    x = _direct_input(kind, NB, H, W, C, 32, eps, seed=H * 7 + C + len(kind))
    x0, x1 = x[..., :C0].contiguous(), (x[..., C0:].contiguous() if C1 else None)
    srcs = [x0] + ([x1] if C1 else [])
    gamma, beta, film = _affine(C, seed=C + H, film_nb=NB)
    st = ops.gn_stats(x0, x1, groups=32, eps=eps)
    chain = _stats_chain(NB, H * W, C)
    imgs = [_image(srcs, n) for n in range(NB)]
    stat_share = _check_stats(st, imgs, 32, eps, "stats", chain, kind)
    del imgs
    y, xr = ops.gn_apply(x0, x1, st, gamma, beta, film=film, act=1, resample=resample, want_xres=True)
    ulps, share = _check_apply(y, srcs, 32, eps, gamma, beta, film, 1, resample, "stats", chain, kind, xres=xr)
    if kind == "constant":
        # zero variance makes rstd = 1 / sqrt(eps) = 316, so B = (beta - mean gamma rstd)(1 + s) + shift cancels in fp32 by
        # about 2^-24 |mean| 316 |gamma (1 + s)|: the output is fp16(silu(beta (1 + s) + shift)) to within one ulp only
        # where that is small (the groups at 0 and 0.3); the error at -7.5 and 1000 is measured and printed
        sc, sh = 1 + film[:, :C].double(), film[:, C:].double()
        want = _silu64(beta.double()[None] * sc + sh)
        got = (y[:, 0, 0, :] if resample != 2 else y[:, 0, 0, :]).double()
        cval = x[:, 0, 0, :].double()
        err = (got - want).abs() / _ulp16(want)
        small = cval.abs() <= 0.3
        assert (err[small] <= 1.0 + 1e-9).all(), ("constant", err[small].max().item())
        print(f"constant groups: worst {err[small].max().item():.2f} ulp at |mean| <= 0.3, "
              f"{err[~small].max().item():.1f} ulp at -7.5 / 1000")
    if kind == "randn" and resample == 0:
        y0 = ops.gn_apply(x0, x1, st, gamma, beta, act=0)
        u0, s0 = _check_apply(y0, srcs, 32, eps, gamma, beta, None, 0, 0, "stats", chain, "act0")
        ulps, share = max(ulps, u0), max(share, s0)
    _report(f"gn_stats->gn_apply NB={NB} {H}x{H} C={C0}+{C1} resample={resample} {kind}", ulps, share, stat_share)


def _movq_cases():
    cases = []
    for i, (H, C) in enumerate(_movq_norms()):
        kinds = ("randn", "offset") if H >= 384 else ("randn", "offset", _KINDS[2 + i % 4])
        cases += [(H, C, k) for k in kinds]
    return cases


@pytest.mark.parametrize("H,C,kind", _movq_cases())
def test_gn_stats_movq_vs_float64(H, C, kind):
    """k2_gn_stats with MoVQ's eps 1e-6 at the decoder's shapes for a 96 x 96 latent, B = 4 (up to 4 x 768^2 x 128)."""
    from kandinsky2 import ops
    NB, eps = 4, 1e-6
    x = _direct_input(kind, NB, H, H, C, 32, eps, seed=H + C + len(kind))
    st = ops.gn_stats(x, None, groups=32, eps=eps)
    worst = 0.0
    chain = _stats_chain(NB, H * H, C)
    for n in range(NB):   # one image at a time: a 768^2 x 128 image is 600 MB in float64
        worst = max(worst, _check_stats(st[n:n + 1], [x[n].double()], 32, eps, "stats", chain, kind))
    print(f"gn_stats MoVQ NB={NB} {H}x{H} C={C} {kind}: statistics at {worst:.2f} of their bound")


# ------------------------------------------------------------------------------------------------------------------------------
# 2-5. conv-produced partials -> gn_finalize -> gn_apply, and -> gn_apply_fold
# ------------------------------------------------------------------------------------------------------------------------------
_CONV_CASES = [
    # (NB, H, C0, C1, taps, cfg, kinds)                           path (input channels 64, 1152 where split-K is forced)
    (8, 96, 384, 0, 9, None, _KINDS),                              # single-image boxes, level 1
    (8, 24, 1152, 768, 9, None, ("randn", "offset", "mixed_means")),   # straddling concat, 60 channels per group
    (8, 48, 768, 384, 9, None, ("randn", "mixed_means")),          # straddling concat, 36 channels per group
    (8, 12, 1536, 0, 9, None, ("randn", "offset", "tiny_var", "mixed_means")),  # 8-image 4 x 4 boxes
    (8, 12, 1536, 0, 9, None, ("constant", "massive")),
    (15, 4, 1536, 0, 9, None, ("randn", "offset", "mixed_means")),  # 8-image boxes, ragged: the second tile holds 7 images
    (8, 12, 1536, 1152, 9, None, ("randn", "mixed_means")),        # 8-image boxes, straddling concat, 84 per group
    (8, 24, 1152, 0, 9, (0, 0, 2, 0), ("randn", "offset", "tiny_var")),  # forced split-K: the second pass's 16-row partials
    (4, 48, 768, 0, 4, None, ("randn", "offset", "massive")),      # taps = 4: 3x3 over the nearest-2x upsampling
]


@pytest.mark.parametrize("NB,H,C0,C1,taps,cfg,kinds", _CONV_CASES)
def test_conv_partials_finalize_and_fold_vs_float64(NB, H, C0, C1, taps, cfg, kinds):
    from kandinsky2 import ops
    W, C, eps = H, C0 + C1, 1e-5
    for kind in kinds:
        outs, parts, rgs, modes = [], [], [], []
        for i, Cs in enumerate((C0, C1) if C1 else (C0,)):
            y, part, rg, info = _conv_input(kind, NB, H, W, Cs, C // 32, eps, seed=H + Cs + i + len(kind), taps=taps,
                                            cfg=cfg, cin=64 if cfg is None else 1152)
            outs.append(y)
            parts.append(part)
            rgs.append(rg)
            modes.append(tuple(info[2:6]))
        if cfg is not None:
            assert all(m[0] == 2 and m[3] == 2 for m in modes), modes      # split-K and its second pass's partials
        if H in (4, 12) and taps == 9 and cfg is None:
            assert all(m[2] == 8 and m[3] == 1 for m in modes), modes      # 8-image 4 x 4 boxes, epilogue partials
        x0, x1 = outs[0], (outs[1] if C1 else None)
        p0, p1 = parts[0], (parts[1] if C1 else None)
        st = torch.empty(NB, 32, 2, device="cuda")
        ops.gn_finalize(p0, C0, p1, C1, NB, rgs[0], H * W, st, eps=eps, rg1=rgs[1] if C1 else None)
        imgs = [_image(outs, n) for n in range(NB)]
        stat_share = _check_stats(st, imgs, 32, eps, "partials", CHAIN_PARTIAL, f"finalize {kind}")
        del imgs
        gamma, beta, film = _affine(C, seed=C + H + 1, film_nb=NB)
        ulps = share = 0.0
        for resample in ((0, 1) if H % 2 == 0 and H >= 24 else (0,)):
            y = ops.gn_apply(x0, x1, st, gamma, beta, film=film, act=1, resample=resample)
            u, s = _check_apply(y, outs, 32, eps, gamma, beta, film, 1, resample, "partials", CHAIN_PARTIAL, f"finalize {kind}")
            ulps, share = max(ulps, u), max(share, s)
            yf = ops.gn_apply_fold(x0, x1, p0, rgs[0], p1, rgs[1] if C1 else 0, gamma, beta, film=film, act=1,
                                   resample=resample, eps=eps)
            u, s = _check_apply(yf, outs, 32, eps, gamma, beta, film, 1, resample, "partials", CHAIN_PARTIAL, f"fold {kind}")
            ulps, share = max(ulps, u), max(share, s)
        _report(f"conv partials NB={NB} {H}x{W} C={C0}+{C1} taps={taps} cfg={cfg} {kind} (finalize + fold)", ulps, share,
                stat_share)


_RATIO_PATHS = {   # (NB, H, C, taps, cfg, input channels)
    "boxes1": (8, 96, 384, 9, None, 64),              # single-image boxes, one partial per M tile of 128 rows
    "boxes8": (8, 12, 1536, 9, None, 64),             # 8-image 4 x 4 boxes, one partial per (image, 16 pixels)
    "boxes8_ragged": (15, 4, 1536, 9, None, 64),      # the same with a last tile of 7 images
    "splitk": (8, 24, 1152, 9, (0, 0, 2, 0), 1152),   # the split-K second pass's 16-row partials
    "up2": (4, 48, 768, 4, None, 64),                 # taps = 4: four phases per box
}


@pytest.mark.parametrize("ratio", [10.0, 100.0, 300.0, 1000.0])
@pytest.mark.parametrize("path", list(_RATIO_PATHS))
def test_conv_partials_per_ratio_vs_float64(path, ratio):
    """Every group at one mean / std, through the real producer of each partial format, then gn_finalize + gn_apply and
    gn_apply_fold.  At mean / std 10 and 100 mean and rstd are held to the stated PARTIAL_REL figures, which the outputs
    inherit; at 300 and 1000 to the partial format's worst-case bound.  The measured rstd error is printed for each."""
    from kandinsky2 import ops
    NB, H, C, taps, cfg, cin = _RATIO_PATHS[path]
    eps = 1e-5
    source = "partials_measured" if ratio in PARTIAL_REL else "partials"
    chain = PARTIAL_REL.get(ratio, CHAIN_PARTIAL)
    y, part, rg, info = _conv_input("offset", NB, H, H, C, C // 32, eps, seed=C + int(ratio), cin=cin, taps=taps, cfg=cfg,
                                    ratio=ratio)
    if cfg is not None:
        assert info[2] == 2 and info[5] == 2, info
    elif taps == 9 and H in (4, 12):
        assert info[4] == 8 and info[5] == 1, info
    st = torch.empty(NB, 32, 2, device="cuda")
    ops.gn_finalize(part, C, None, 0, NB, rg, H * H, st, eps=eps)
    rel = 0.0
    for n in range(NB):
        rs = _ref_stats(y[n].double(), 32)
        rel = max(rel, ((st[n, :, 1].double() * torch.sqrt(rs[1] + eps)) - 1).abs().max().item())
    stat_share = _check_stats(st, [y[n].double() for n in range(NB)], 32, eps, source, chain, f"{path} {ratio}")
    gamma, beta, film = _affine(C, seed=C + 3, film_nb=NB)
    out = ops.gn_apply(y, None, st, gamma, beta, film=film, act=1)
    ulps, share = _check_apply(out, [y], 32, eps, gamma, beta, film, 1, 0, source, chain, f"{path} {ratio}")
    outf = ops.gn_apply_fold(y, None, part, rg, None, 0, gamma, beta, film=film, act=1, eps=eps)
    u, s = _check_apply(outf, [y], 32, eps, gamma, beta, film, 1, 0, source, chain, f"fold {path} {ratio}")
    _report(f"conv partials {path} mean/std {ratio:g}: rstd off by {rel:.2e} relative (2^{math.log2(max(rel, 1e-300)):.1f});"
            f" finalize + fold", max(ulps, u), max(share, s), stat_share)


# ------------------------------------------------------------------------------------------------------------------------------
# 6. sn_apply: statistics from gn_finalize and from gn_stats, zq at ratios 1, 2, 4, 8 and 3 (the non-shift path)
# ------------------------------------------------------------------------------------------------------------------------------
def _sn_inputs(NB, C, zh, zw, seed):
    g = _gen(seed)
    zq = torch.randn(NB, zh, zw, 4, device="cuda", generator=g)
    gamma = 1 + 0.1 * torch.randn(C, device="cuda", generator=g)
    beta = 0.1 * torch.randn(C, device="cuda", generator=g)
    wy, by = torch.randn(C, 4, device="cuda", generator=g) / 2, torch.randn(C, device="cuda", generator=g) / 4 + 1
    wb, bb = torch.randn(C, 4, device="cuda", generator=g) / 2, torch.randn(C, device="cuda", generator=g) / 4
    return zq, gamma, beta, torch.cat([wy, by[:, None], wb, bb[:, None]], 1).contiguous()


def _sn_mod(zq, sn_w, H, W):
    """float64 (my, mb, |my| term sum, |mb| term sum) [NB, H, W, C] of the nearest-resized latent."""
    zu = F.interpolate(zq.double().permute(0, 3, 1, 2), size=(H, W), mode="nearest").permute(0, 2, 3, 1)
    sw = sn_w.double()
    my = zu @ sw[:, :4].T + sw[:, 4]
    mb = zu @ sw[:, 5:9].T + sw[:, 9]
    return my, mb, zu.abs() @ sw[:, :4].abs().T + sw[:, 4].abs(), zu.abs() @ sw[:, 5:9].abs().T + sw[:, 9].abs()


@pytest.mark.parametrize("H,C,ratio,kind,src", [
    (96, 512, 1, "randn", "stats"), (96, 512, 1, "offset", "finalize"), (96, 512, 3, "tiny_var", "stats"),
    (192, 256, 2, "randn", "finalize"), (192, 256, 2, "mixed_means", "stats"), (192, 256, 3, "offset", "stats"),
    (384, 256, 4, "randn", "stats"), (384, 256, 4, "constant", "finalize"),
    (768, 128, 8, "randn", "finalize"), (768, 128, 8, "offset", "stats"),
])
def test_sn_apply_vs_float64(H, C, ratio, kind, src):
    """MoVQ SpatialNorm + swish at the decoder's shapes (B = 4, eps 1e-6): y = silu(GN(x) (wy.z + by) + (wb.z + bb)) with z
    the latent pixel under (y, x)."""
    from kandinsky2 import ops
    NB, W, eps = 4, H, 1e-6
    if src == "finalize":
        x, part, rg, _ = _conv_input(kind, NB, H, W, C, C // 32, eps, seed=H + C + ratio)
        st = torch.empty(NB, 32, 2, device="cuda")
        ops.gn_finalize(part, C, None, 0, NB, rg, H * W, st, eps=eps)
        source, chain = "partials", CHAIN_PARTIAL
    else:
        x = _direct_input(kind, NB, H, W, C, 32, eps, seed=H + C + ratio)
        st = ops.gn_stats(x, None, eps=eps)
        source, chain = "stats", _stats_chain(NB, H * W, C)
    zq, gamma, beta, sn_w = _sn_inputs(NB, C, -(-H // ratio), -(-W // ratio), seed=C + ratio)
    y = ops.sn_apply(x, st, gamma, beta, zq, sn_w, act=1)
    ulps = share = 0.0
    for n in range(NB):
        stat_share = _check_stats(st[n:n + 1], [x[n].double()], 32, eps, source, chain, kind)
        mod = _sn_mod(zq[n:n + 1], sn_w, H, W)
        u, s = _check_apply(y[n:n + 1], [x[n:n + 1]], 32, eps, gamma, beta, None, 1, 0, source, chain, kind, mod=mod)
        ulps, share = max(ulps, u), max(share, s)
    _report(f"sn_apply {H}x{W} C={C} zq 1/{ratio} {kind} stats from {src}", ulps, share, stat_share)


# ------------------------------------------------------------------------------------------------------------------------------
# SiLU wherever it is applied
# ------------------------------------------------------------------------------------------------------------------------------
def _all_f16():
    return torch.arange(-32768, 32768, dtype=torch.int32, device="cuda").to(torch.int16).view(torch.float16).clone()


def _check_silu_f16(y, x, what):
    """Finite inputs: within one ulp of float64 silu (correctly rounded up to fp32 error near a rounding tie).  +inf -> +inf,
    -inf and NaN -> NaN, as torch's fp32 SiLU gives."""
    fin = torch.isfinite(x)
    t32 = F.silu(x[~fin].float())
    assert torch.equal(torch.isnan(y[~fin]), torch.isnan(t32)), what
    assert torch.equal(y[~fin].float()[~torch.isnan(t32)], t32[~torch.isnan(t32)]), what
    xd = x[fin].double()
    ref = _silu64(xd)
    got = y[fin].double()
    ulps = (got - ref).abs() / _ulp16(ref)
    worst = ulps.argmax()
    exact = (got == ref.half().double()).double().mean().item()
    print(f"silu {what}: worst {ulps[worst].item():.3f} ulp at x = {xd[worst].item()!r}; {exact:.4%} correctly rounded")
    assert ulps.max().item() <= 1.0, (what, xd[ulps > 1][:6].tolist(), got[ulps > 1][:6].tolist(), ref[ulps > 1][:6].tolist())


def test_silu_f16_every_fp16_value():
    from kandinsky2 import ops
    x = _all_f16()
    _check_silu_f16(ops.silu_f16_(x.clone()), x, "silu_f16_")


def test_silu_through_gn_apply_every_fp16_value():
    """gn_apply with a hand-built statistics buffer (mean 0, rstd 1), gamma 1, beta 0: t = fma(x, 1, 0) = x, y = silu(x)."""
    from kandinsky2 import ops
    x = _all_f16().view(1, 16, 32, 128)
    st = torch.tensor([0.0, 1.0], device="cuda").repeat(1, 32, 1).contiguous()
    one, zero = torch.ones(128, device="cuda"), torch.zeros(128, device="cuda")
    for resample in (0, 2):
        y = ops.gn_apply(x, None, st, one, zero, act=1, resample=resample)
        if resample == 2:
            y = y[:, ::2, ::2]
        _check_silu_f16(y.reshape(-1), x.reshape(-1), f"gn_apply resample={resample}")


def test_silu_through_sn_apply_every_fp16_value():
    """sn_apply with mean 0, rstd 1, gamma 1, beta 0 and modulation coefficients wy = 0, by = 1, wb = 0, bb = 0: a = 1,
    b = 0 whatever the latent, so y = silu(x)."""
    from kandinsky2 import ops
    x = _all_f16().view(1, 16, 32, 128)
    st = torch.tensor([0.0, 1.0], device="cuda").repeat(1, 32, 1).contiguous()
    one, zero = torch.ones(128, device="cuda"), torch.zeros(128, device="cuda")
    sn_w = torch.zeros(128, 10, device="cuda")
    sn_w[:, 4] = 1.0
    zq = torch.randn(1, 4, 8, 4, device="cuda", generator=_gen(3))
    y = ops.sn_apply(x, st, one, zero, zq, sn_w, act=1)
    _check_silu_f16(y.reshape(-1), x.reshape(-1), "sn_apply")


def test_silu_fp32_through_linear():
    """ops.linear(x, I, silu_out=True) and ops.linear(x, I, silu_in=True): an identity weight makes the product exact, so the
    fp32 outputs are silu_f itself.  Bound, relative to the float64 value: ex2.approx (2^-22), the rounding of -x log2 e
    (2^-24 |x| after the exponential, plus 2^-25 |x| for the fp32 constant), rcp.approx (2^-23), 1 + e and the product
    (2 x 2^-24): within 2^-20 + 2^-23 |x|.  Inputs: every fp32 exponent of [-30, 30] with random mantissas, and the fp16 grid."""
    from kandinsky2 import ops
    g = _gen(11)
    N = 64
    mant = 1 + torch.rand(4096, device="cuda", generator=g)
    ex = torch.randint(-24, 5, (4096,), device="cuda", generator=g).float()
    sgn = torch.where(torch.rand(4096, device="cuda", generator=g) < 0.5, -1.0, 1.0)
    x = torch.cat([sgn * mant * torch.exp2(ex), torch.linspace(-30, 30, 8192, device="cuda"),
                   _all_f16().float()[torch.isfinite(_all_f16().float())]])
    x = x[x.abs() <= 30]
    x = torch.cat([x, torch.zeros(-x.numel() % N, device="cuda")]).view(-1, N).contiguous()
    eye = torch.eye(N, device="cuda")
    ref = _silu64(x.double())
    bound = (2.0 ** -20 + 2.0 ** -23 * x.double().abs()) * ref.abs() + 2.0 ** -149
    worst = 0.0
    for kw in (dict(silu_out=True), dict(silu_in=True)):
        y = ops.linear(x, eye, **kw)
        err = (y.double() - ref).abs()
        bad = err > bound
        assert not bad.any(), (kw, x[bad][:4].tolist(), err[bad][:4].tolist(), ref[bad][:4].tolist())
        worst = max(worst, (err / bound).max().item())
    rel = ((ops.linear(x, eye, silu_out=True).double() - ref).abs() / ref.abs().clamp(min=1e-30)).max().item()
    print(f"silu fp32 through linear: worst relative error {rel:.3g} (2^{math.log2(max(rel, 1e-300)):.1f}), "
          f"{worst:.2f} of the bound")
