"""k2_conv_gemm's 3x3 and up2 (3x3 over a nearest-2x upsampling) convolutions against a float64 convolution of the same fp16
data and fp16 weights, computed one image per call, with bounds that allow only the kernel's own roundings: the fp16 rounding
of the stored output (2^-11 relative) plus fp32 accumulation over K terms (K * 2^-23, the unit roundoff of a truncating fp32
add, times the sum of absolute products).  Covered: the output boxes of the step's levels, ragged images, partial channel
chunks, row-strided sources with NaN in the gap columns, all four up2 phases, the up-path ResBlock's three K segments, split-K
at 2 to 7 splits, bias and residual, the fused GroupNorm partial sums, and run-to-run bit identity."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

EPS16 = 2.0 ** -11  # fp16 rounding to nearest, relative
EPS32 = 2.0 ** -23  # fp32 add, rounding or truncating, relative
TINY = 2.0 ** -25   # half the fp16 subnormal step


def _rand(g, *shape, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).half()


def _conv64(x_nhwc, w, pad):
    """float64 conv2d, one image per call: NHWC in, NHWC out."""
    wd = w.double()
    out = [F.conv2d(x_nhwc[n:n + 1].double().permute(0, 3, 1, 2), wd, padding=pad) for n in range(x_nhwc.shape[0])]
    return torch.cat(out).permute(0, 2, 3, 1)


def _up2_conv64(x_nhwc, wp, cin, cout):
    """float64 reference of a taps == 4 source from the packed phase weights: output pixel (2y + a, 2x + b) sums source
    pixels (y + ty + a - 1, x + tx + b - 1) times block ((a, b), (ty, tx)) of the packed matrix."""
    c64 = (cin + 63) // 64 * 64
    NB, H, W, _ = x_nhwc.shape
    out = torch.zeros(NB, 2 * H, 2 * W, cout, dtype=torch.float64, device=x_nhwc.device)
    wabs = torch.zeros_like(out)
    for a in (0, 1):
        for b in (0, 1):
            k = torch.zeros(cout, cin, 2, 2, dtype=torch.float64, device=x_nhwc.device)
            for ty in (0, 1):
                for tx in (0, 1):
                    blk = ((a * 2 + b) * 4 + ty * 2 + tx) * c64
                    k[:, :, ty, tx] = wp[:cout, blk:blk + cin].double()
            for n in range(NB):
                xn = F.pad(x_nhwc[n:n + 1].double().permute(0, 3, 1, 2), (1, 1, 1, 1))
                y = F.conv2d(xn, k)[:, :, a:a + H, b:b + W]
                ya = F.conv2d(xn.abs(), k.abs())[:, :, a:a + H, b:b + W]
                out[n, a::2, b::2] = y[0].permute(1, 2, 0)
                wabs[n, a::2, b::2] = ya[0].permute(1, 2, 0)
    return out, wabs


def _check(y, ref, absum, k_terms, eps_out=EPS16):
    """|y - ref| <= rounding of the output (eps_out relative: fp16 by default, 0 for fp32 outputs) + fp32 accumulation error
    over k_terms products (+ subnormal step).  Returns the worst share of the bound."""
    bound = eps_out * ref.abs() + 1.01 * k_terms * EPS32 * absum + TINY
    err = (y.double() - ref).abs()
    worst = (err / bound).max().item()
    assert worst <= 1.0, f"error exceeds the fp32-accumulation bound by {worst:.3f}x (max abs err {err.max().item():.3e})"
    return worst


def _case(g, NB, H, W, C, Cout, *, taps=9, strided=False, residual=False, skips=None, split=0, gn=False):
    """Runs one conv through k2_conv_gemm twice and checks it against float64; returns (info, y, part)."""
    from kandinsky2 import ops
    if strided:
        buf = _rand(g, NB, H, W, C + 24)
        buf[..., C:] = float("nan")  # gap columns of a row-strided view: never read
        x = buf[..., :C]
    else:
        x = _rand(g, NB, H, W, C)
    Ho, Wo = (2 * H, 2 * W) if taps == 4 else (H, W)
    w = torch.randn(Cout, C, 3, 3, device="cuda", generator=g) / (3 * C ** 0.5)
    wp = ops.pack_conv_weight_up2(w) if taps == 4 else ops.pack_conv_weight(w)
    srcs = [(x, taps)]
    k_terms = (4 if taps == 4 else 9) * C
    skip_in = None
    if skips:
        ca, cb = skips
        sbuf = _rand(g, NB, H, W, ca + cb + 8)
        xa, xb = sbuf[..., :ca], sbuf[..., ca:ca + cb]
        w1 = torch.randn(Cout, ca + cb, 1, 1, device="cuda", generator=g) / (ca + cb) ** 0.5
        wp = torch.cat([wp, ops.pack_conv_weight(w1, split=(ca, cb))], 1).contiguous()
        srcs += [(xa, 1), (xb, 1)]
        skip_in = (torch.cat([xa, xb], -1), w1)
        k_terms += ca + cb
    b = torch.randn(Cout, device="cuda", generator=g)
    res = _rand(g, NB, Ho, Wo, Cout) if residual else None
    outs = []
    for _ in range(2):
        info = [0] * 7
        part = torch.zeros(ops.gn_part_floats(NB, Ho, Wo, Cout), device="cuda") if gn else None
        y = ops.conv_gemm(srcs, wp, Cout, bias=b, residual=res, gn_part=part, info=info, cfg=(0, 0, split, 0))
        torch.cuda.synchronize()
        outs.append((y.clone(), None if part is None else part.clone(), info))
    (y, part, info), (y2, part2, _) = outs
    assert torch.equal(y.view(torch.int16), y2.view(torch.int16)), "two runs differ"
    if gn:
        assert torch.equal(part.view(torch.int32), part2.view(torch.int32)), "two runs' GroupNorm partials differ"
    if taps == 4:
        ref, absum = _up2_conv64(x, wp, C, Cout)
    else:
        wh = w.half()
        ref = _conv64(x, wh, 1)
        absum = _conv64(x.abs(), wh.abs(), 1)
    if skip_in is not None:
        xs, w1 = skip_in
        ref = ref + _conv64(xs, w1.half(), 0)
        absum = absum + _conv64(xs.abs(), w1.half().abs(), 0)
    ref = ref + b.double()
    absum = absum + b.double().abs()
    if residual:
        ref = ref + res.double()
        absum = absum + res.double().abs()
        k_terms += 2
    _check(y, ref, absum, k_terms)
    return info, y, part


@pytest.mark.parametrize("NB,H,W,C,Cout,box", [
    (2, 96, 96, 64, 128, (1, 8, 16)),     # 96^2 / 48^2 levels: 8 x 16 boxes
    (2, 24, 24, 128, 192, (1, 5, 24)),    # 24^2 level: 5 x 24 boxes
    (8, 12, 12, 128, 256, (8, 4, 4)),     # 12^2 level: 8 images x 4 x 4 per box
])
def test_step_boxes(NB, H, W, C, Cout, box):
    g = torch.Generator(device="cuda").manual_seed(10)
    info, _, _ = _case(g, NB, H, W, C, Cout, residual=True)
    tn = box[0]
    assert info[4] == tn
    assert info[3] == (NB // tn) * -(-H // box[1]) * -(-W // box[2]), info


@pytest.mark.parametrize("NB,H,W,C,Cout", [
    (3, 7, 9, 64, 64),       # ragged: the box does not divide H or W
    (2, 20, 28, 96, 128),    # C not a multiple of 64
    (2, 17, 23, 40, 192),    # C < 64
])
def test_ragged_and_partial_chunks(NB, H, W, C, Cout):
    g = torch.Generator(device="cuda").manual_seed(11)
    _case(g, NB, H, W, C, Cout)


@pytest.mark.parametrize("C", [64, 72])
def test_row_strided_source_with_nan_gaps(C):
    g = torch.Generator(device="cuda").manual_seed(12)
    _case(g, 2, 20, 28, C, 128, strided=True, residual=True)


@pytest.mark.parametrize("NB,H,W,C,Cout", [(2, 12, 12, 96, 128), (2, 24, 24, 128, 192), (8, 6, 6, 64, 128)])
def test_up2_all_phases(NB, H, W, C, Cout):
    g = torch.Generator(device="cuda").manual_seed(13)
    _case(g, NB, H, W, C, Cout, taps=4)


def test_up_path_three_segments():
    """3x3 of h plus the 1x1 skip over the un-materialised concat [xa | xb] (the up-path ResBlock), with residual."""
    g = torch.Generator(device="cuda").manual_seed(14)
    _case(g, 2, 24, 24, 192, 192, skips=(128, 72), residual=True)


@pytest.mark.parametrize("split", [2, 3, 4, 5, 6, 7])
def test_split_k(split):
    """43 channel chunks x 9 taps: every split from 2 to 7 is legal, none empty."""
    g = torch.Generator(device="cuda").manual_seed(15)
    info, _, _ = _case(g, 8, 12, 12, 43 * 64, 128, residual=True, split=split)
    assert info[2] == split, info


@pytest.mark.parametrize("NB,H,W,C,Cout", [(2, 24, 24, 128, 192), (8, 12, 12, 128, 256), (2, 40, 40, 96, 128)])
def test_fused_groupnorm_partials(NB, H, W, C, Cout):
    """The epilogue's (sum, sumsq) partials, one per M tile (single-image boxes) or per (image, spatial tile) (8-image 4 x 4
    boxes), summed per image, against float64 sums of the stored fp16 outputs."""
    g = torch.Generator(device="cuda").manual_seed(16)
    info, y, part = _case(g, NB, H, W, C, Cout, residual=True, gn=True)
    assert info[5] == 1, info  # fused in the epilogue
    rg = info[6]
    assert rg % NB == 0
    p = part[:rg * Cout * 2].view(NB, rg // NB, Cout, 2).double().sum(1)
    yd = y.double().reshape(NB, H * W, Cout)
    s1, s2 = yd.sum(1), (yd * yd).sum(1)
    n = H * W
    assert ((p[..., 0] - s1).abs() <= 1.01 * n * EPS32 * yd.abs().sum(1) + 1e-6).all()
    assert ((p[..., 1] - s2).abs() <= 1.01 * n * EPS32 * s2 + 1e-6).all()
