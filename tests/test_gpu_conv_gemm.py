"""GPU parity of k2_conv_gemm (wgmma implicit-GEMM conv) against torch fp32 conv2d on the same fp16 data."""
import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu


def _ref_conv(x_nhwc, w, b, pad):
    y = F.conv2d(x_nhwc.float().permute(0, 3, 1, 2), w.half().float(), b, padding=pad)
    return y.permute(0, 2, 3, 1)


@pytest.fixture(autouse=True)
def _no_tf32():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False


@pytest.mark.parametrize("NB,H,W,Cin,Cout", [
    (2, 16, 16, 64, 128),     # one (16x8) box geometry, BN=128
    (1, 96, 96, 128, 256),    # metric geometry, BN=256, multi-tile persistent loop
    (3, 24, 24, 192, 192),    # TW=24 TH=5 partial boxes, BN=192
    (4, 12, 12, 128, 384),    # 12x6 boxes
    (5, 4, 4, 64, 64),        # TN>1: several images per tile, BN=64
    (2, 8, 12, 64, 320),      # non-square, Cout not a multiple of the N tile
])
def test_conv3x3(NB, H, W, Cin, Cout):
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(NB, H, W, Cin, device="cuda", generator=g).half()
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) / (3 * Cin ** 0.5)
    b = torch.randn(Cout, device="cuda", generator=g)
    y = ops.conv_gemm([(x, 9)], ops.pack_conv_weight(w), Cout, bias=b)
    torch.cuda.synchronize()
    ref = _ref_conv(x, w, b, 1)
    err = (y.float() - ref).abs().max().item()
    assert err < 2e-2 * max(1.0, ref.abs().max().item()) / 4, f"max abs err {err}"
    # fp16 output rounding only: relative error of the bulk must be ~1e-3
    rel = ((y.float() - ref).norm() / ref.norm()).item()
    assert rel < 1e-3, rel


def test_gemm_rows_bias_residual():
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(1)
    M, K, N = 1000, 256, 384
    x = torch.randn(M, K, device="cuda", generator=g).half()
    w = torch.randn(N, K, device="cuda", generator=g) / K ** 0.5
    b = torch.randn(N, device="cuda", generator=g)
    r = torch.randn(M, N, device="cuda", generator=g).half()
    y = ops.gemm_rows(x, ops.pack_conv_weight(w), N, bias=b, residual=r)
    torch.cuda.synchronize()
    ref = x.float() @ w.half().float().t() + b + r.float()
    rel = ((y.float() - ref).norm() / ref.norm()).item()
    assert rel < 1e-3, rel


def test_conv_plus_skip_segments():
    """3x3 conv of h plus 1x1 skip of the (virtual) concat [xa | xb] accumulated in one kernel, + residual-free."""
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(2)
    NB, H, W, Ch, Ca, Cb, Cout = 2, 16, 16, 128, 64, 128, 256
    h = torch.randn(NB, H, W, Ch, device="cuda", generator=g).half()
    buf = torch.randn(NB, H, W, Ca + Cb + 64, device="cuda", generator=g).half()
    xa, xb = buf[..., :Ca], buf[..., Ca:Ca + Cb]            # channel-slice views (row stride > C)
    w3 = torch.randn(Cout, Ch, 3, 3, device="cuda", generator=g) / (3 * Ch ** 0.5)
    w1 = torch.randn(Cout, Ca + Cb, 1, 1, device="cuda", generator=g) / (Ca + Cb) ** 0.5
    b = torch.randn(Cout, device="cuda", generator=g)
    wp = torch.cat([ops.pack_conv_weight(w3), ops.pack_conv_weight(w1, split=(Ca, Cb))], 1).contiguous()
    y = ops.conv_gemm([(h, 9), (xa, 1), (xb, 1)], wp, Cout, bias=b)
    torch.cuda.synchronize()
    ref = _ref_conv(h, w3, b, 1) + _ref_conv(torch.cat([xa, xb], -1), w1, None, 0)
    rel = ((y.float() - ref).norm() / ref.norm()).item()
    assert rel < 1e-3, rel


def test_head_fp32_nchw():
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(3)
    NB, H, W, Cin, Cout = 2, 32, 32, 128, 8
    x = torch.randn(NB, H, W, Cin, device="cuda", generator=g).half()
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) / (3 * Cin ** 0.5)
    b = torch.randn(Cout, device="cuda", generator=g)
    wp = ops.pad_rows(ops.pack_conv_weight(w), 16)
    y = ops.conv_gemm([(x, 9)], wp, Cout, bias=b, out_mode=1)
    torch.cuda.synchronize()
    ref = F.conv2d(x.float().permute(0, 3, 1, 2), w.half().float(), b, padding=1)
    assert y.shape == ref.shape and y.dtype == torch.float32
    assert (y - ref).abs().max().item() < 2e-3


@pytest.mark.parametrize("split", [0, 1, 3, 5])
def test_splitk_small_m(split):
    """Bottom-of-the-U geometry (M = 8*12*12 rows, K = 9*1536): split-K partials + deterministic finalize, with bias,
    residual and a second (1x1 skip) K segment; split 0 = automatic choice, 1 = off, n = forced."""
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(4)
    NB, H, W, Cin, Cs, Cout = 8, 12, 12, 1536, 192, 768
    h = torch.randn(NB, H, W, Cin, device="cuda", generator=g).half()
    xs = torch.randn(NB, H, W, Cs, device="cuda", generator=g).half()
    res = torch.randn(NB, H, W, Cout, device="cuda", generator=g).half()
    w3 = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) / (3 * Cin ** 0.5)
    w1 = torch.randn(Cout, Cs, 1, 1, device="cuda", generator=g) / Cs ** 0.5
    b = torch.randn(Cout, device="cuda", generator=g)
    wp = torch.cat([ops.pack_conv_weight(w3), ops.pack_conv_weight(w1)], 1).contiguous()
    ops.set_tuning(1, split)
    try:
        ops.reset_launch_count()
        y = ops.conv_gemm([(h, 9), (xs, 1)], wp, Cout, bias=b, residual=res)
        y2 = ops.conv_gemm([(h, 9), (xs, 1)], wp, Cout, bias=b, residual=res)
        launches = ops.launch_count()
    finally:
        ops.set_tuning(1, 0)
    torch.cuda.synchronize()
    assert torch.equal(y, y2), "split-K reduction must be deterministic"
    if split > 1:
        assert launches == 4  # (conv + finalize) x 2
    ref = _ref_conv(h, w3, b, 1) + _ref_conv(xs, w1, None, 0) + res.float()
    rel = ((y.float() - ref).norm() / ref.norm()).item()
    assert rel < 1e-3, rel


@pytest.mark.parametrize("epi_sets", [1, 2])
@pytest.mark.parametrize("NB,H,W,Cin,Cout,C1", [(2, 24, 24, 128, 256, 0), (3, 16, 12, 64, 384, 128), (1, 96, 96, 64, 192, 0)])
def test_conv_fused_groupnorm_partials(epi_sets, NB, H, W, Cin, Cout, C1):
    """The conv epilogue's per-tile (sum, sumsq) partials + k2_gn_finalize == a statistics pass over the stored output
    (also over the concat with a second producer's output), with one or two epilogue warp sets (tuning key 10)."""
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(8)
    ops.set_tuning(10, epi_sets)
    try:
        outs, parts, rgs = [], [], []
        for cout in [Cout] + ([C1] if C1 else []):
            x = torch.randn(NB, H, W, Cin, device="cuda", generator=g).half()
            w = torch.randn(cout, Cin, 3, 3, device="cuda", generator=g) / (3 * Cin ** 0.5)
            b = torch.randn(cout, device="cuda", generator=g)
            res = torch.randn(NB, H, W, cout, device="cuda", generator=g).half()
            part = torch.zeros(ops.gn_part_floats(NB, H, W, cout), device="cuda")
            info = [0] * 7
            y = ops.conv_gemm([(x, 9)], ops.pack_conv_weight(w), cout, bias=b, residual=res, gn_part=part, info=info)
            assert info[5] in (1, 2) and (info[5] == 2) == (info[2] > 1), info   # epilogue partials, or split-K second pass
            rgs.append(info[6] // NB)
            outs.append(y)
            parts.append(part)
    finally:
        ops.set_tuning(10, 1)
    st = torch.empty(NB, 32, 2, device="cuda")
    ops.gn_finalize(parts[0], Cout, parts[1] if C1 else None, C1, NB, rgs[0], H * W, st, rg1=rgs[1] if C1 else None)
    ref = ops.gn_stats(outs[0], outs[1] if C1 else None)
    torch.cuda.synchronize()
    assert torch.allclose(st[..., 0], ref[..., 0], atol=2e-5), (st[..., 0] - ref[..., 0]).abs().max()
    assert torch.allclose(st[..., 1], ref[..., 1], rtol=2e-5)


def test_splitk_fused_groupnorm_partials():
    """split-K second pass emits the partial statistics (16-row groups) of its rounded output."""
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(9)
    NB, H, W, Cin, Cout = 8, 12, 12, 1536, 1536
    x = torch.randn(NB, H, W, Cin, device="cuda", generator=g).half()
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) / (3 * Cin ** 0.5)
    b = torch.randn(Cout, device="cuda", generator=g)
    part = torch.zeros(ops.gn_part_floats(NB, H, W, Cout), device="cuda")
    info = [0] * 7
    ops.set_tuning(1, 2)  # force a 2-way K split (the heuristic keeps this shape unsplit)
    try:
        y = ops.conv_gemm([(x, 9)], ops.pack_conv_weight(w), Cout, bias=b, gn_part=part, info=info)
    finally:
        ops.set_tuning(1, 0)
    assert info[2] == 2 and info[5] == 2 and info[6] == NB * H * W // 16, info
    st = torch.empty(NB, 32, 2, device="cuda")
    ops.gn_finalize(part, Cout, None, 0, NB, info[6] // NB, H * W, st)
    ref = ops.gn_stats(y, None)
    torch.cuda.synchronize()
    assert torch.allclose(st[..., 0], ref[..., 0], atol=2e-5) and torch.allclose(st[..., 1], ref[..., 1], rtol=2e-5)


@pytest.mark.parametrize("NB", [8, 5])
def test_multi_image_tile_fused_groupnorm_partials(NB):
    """12x12 latents use (4 x 4 pixels x 8 images) tiles: the epilogue emits one partial per (image, spatial tile) from each
    half warp; also with a ragged last image group (NB = 5)."""
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(10)
    H, W, Cin, Cout = 12, 12, 256, 512
    x = torch.randn(NB, H, W, Cin, device="cuda", generator=g).half()
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) / (3 * Cin ** 0.5)
    b = torch.randn(Cout, device="cuda", generator=g)
    res = torch.randn(NB, H, W, Cout, device="cuda", generator=g).half()
    part = torch.zeros(ops.gn_part_floats(NB, H, W, Cout), device="cuda")
    info = [0] * 7
    ops.set_tuning(1, 1)
    try:
        y = ops.conv_gemm([(x, 9)], ops.pack_conv_weight(w), Cout, bias=b, residual=res, gn_part=part, info=info)
    finally:
        ops.set_tuning(1, 0)
    ref_y = F.conv2d(x.float().permute(0, 3, 1, 2), w.half().float(), b, padding=1).permute(0, 2, 3, 1) + res.float()
    assert ((y.float() - ref_y).norm() / ref_y.norm()).item() < 1e-3
    if NB == 8:
        assert info[4] == 8 and info[5] == 1, info  # (4 x 4 x 8) tiles, statistics fused
    if info[5] == 1:
        assert info[6] % NB == 0, info
        st = torch.empty(NB, 32, 2, device="cuda")
        ops.gn_finalize(part, Cout, None, 0, NB, info[6] // NB, H * W, st)
        ref = ops.gn_stats(y, None)
        torch.cuda.synchronize()
        assert torch.allclose(st[..., 0], ref[..., 0], atol=2e-5) and torch.allclose(st[..., 1], ref[..., 1], rtol=2e-5)


@pytest.mark.parametrize("NB,H,W,Cin,Cout,taps,res,split", [
    (8, 48, 48, 768, 768, 9, True, 0), (8, 96, 96, 384, 384, 9, False, 0), (1, 1, 18432, 768, 2304, 1, False, 0),
    (8, 24, 24, 1152, 1152, 9, True, 0), (8, 12, 12, 1536, 1536, 9, True, 0), (8, 12, 12, 1536, 1536, 9, False, 2),
    (2, 24, 24, 128, 192, 9, True, 0)])
def test_two_epilogue_sets_bit_identical(NB, H, W, Cin, Cout, taps, res, split):
    """Two epilogue warp sets (both consumer warpgroups drain the accumulator, k2_conv_gemm_cfg cfg[3] = 2) against one:
    outputs and GroupNorm partials must be bit-identical (same arithmetic, different warps)."""
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(12)
    x = torch.randn(NB, H, W, Cin, device="cuda", generator=g).half()
    w = torch.randn(Cout, Cin, 3 if taps == 9 else 1, 3 if taps == 9 else 1, device="cuda", generator=g) / (Cin * taps) ** 0.5
    b = torch.randn(Cout, device="cuda", generator=g)
    r = torch.randn(NB, H, W, Cout, device="cuda", generator=g).half() if res else None
    wp = ops.pack_conv_weight(w)
    outs = []
    for sets in (1, 2):
        part = torch.zeros(ops.gn_part_floats(NB, H, W, Cout), device="cuda")
        info = [0] * 7
        y = ops.conv_gemm([(x, taps)], wp, Cout, bias=b, residual=r, gn_part=part, info=info, cfg=(0, 0, split, sets))
        torch.cuda.synchronize()
        outs.append((y.clone(), part.clone(), list(info)))
    assert outs[0][2] == outs[1][2]
    assert torch.equal(outs[0][0], outs[1][0])
    assert torch.equal(outs[0][1], outs[1][1])


@pytest.mark.parametrize("bn", [128, 192, 256])
def test_n_tile_choice_is_bit_identical(bn):
    """k2_conv_gemm_cfg: the N tile never changes a result bit (the launch plans' autotuner relies on it)."""
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(13)
    x = torch.randn(4, 24, 24, 320, device="cuda", generator=g).half()
    w = torch.randn(384, 320, 3, 3, device="cuda", generator=g) / 54
    b = torch.randn(384, device="cuda", generator=g)
    wp = ops.pack_conv_weight(w)
    outs = []
    # baseline: the library's own N tile, unsplit (the cycle model splits K for this shape on 132 SMs, and a K split does
    # change the fp32 summation order)
    for cfg in ((0, 0, 1, 0), (bn, 0, 1, 1), (bn, 0, 1, 2)):
        part = torch.zeros(ops.gn_part_floats(4, 24, 24, 384), device="cuda")
        y = ops.conv_gemm([(x, 9)], wp, 384, bias=b, gn_part=part, cfg=cfg)
        torch.cuda.synchronize()
        outs.append((y.clone(), part.clone()))
    for y, part in outs[1:]:
        assert torch.equal(y, outs[0][0]) and torch.equal(part, outs[0][1])


@pytest.mark.parametrize("NB,H,W,Cin,Cout", [
    (2, 24, 24, 128, 192),     # odd number of boxes per phase
    (8, 12, 12, 1536, 1536),   # UNet level 3 -> 2: (8 image x 4 x 4) boxes, partials per (image, spatial tile)
    (8, 48, 48, 768, 768),     # UNet level 1 -> 0
    (1, 6, 10, 64, 64),        # N tile 64, ragged box
    (2, 16, 16, 96, 128),      # Cin not a multiple of 64
    (1, 96, 96, 256, 256),     # MoVQ Upsample geometry
])
def test_conv3x3_over_nearest_upsample(NB, H, W, Cin, Cout):
    """taps = 4: conv3x3(nearest_2x(x)) evaluated as four 2x2 phase convolutions over x (unet.py:67-77, movq_modules.py:93-97);
    the 4x larger tensor never exists.  Reference: torch fp32 on the same fp16 data with the ORIGINAL 3x3 weights rounded to
    fp16 -- the pre-summed phase weights are rounded once more, hence the slightly wider tolerance than test_conv3x3.  Also
    checks the fused GroupNorm partials (4 phases per box) through k2_gn_apply_fold against a direct statistics pass."""
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(5)
    x = torch.randn(NB, H, W, Cin, device="cuda", generator=g).half()
    w = torch.randn(Cout, Cin, 3, 3, device="cuda", generator=g) / (3 * Cin ** 0.5)
    b = torch.randn(Cout, device="cuda", generator=g)
    part = torch.zeros(ops.gn_part_floats(NB, 2 * H, 2 * W, Cout), device="cuda")
    info = [0] * 7
    y = ops.conv_gemm([(x, 4)], ops.pack_conv_weight_up2(w), Cout, bias=b, gn_part=part, info=info)
    torch.cuda.synchronize()
    assert tuple(y.shape) == (NB, 2 * H, 2 * W, Cout)
    up = F.interpolate(x.float().permute(0, 3, 1, 2), scale_factor=2, mode="nearest")
    # one image per cuDNN call: at batch 8, 768 -> 768 channels, 96 x 96, cuDNN's batched fp32 convolution has returned wrong
    # values in the high output channels of one image, while per-image calls agree with a float64 evaluation
    ref = torch.cat([F.conv2d(up[i:i + 1], w.half().float(), b, padding=1) for i in range(NB)]).permute(0, 2, 3, 1)
    rel = ((y.float() - ref).norm() / ref.norm()).item()
    err = (y.float() - ref).abs().max().item()
    assert rel < 1.5e-3 and err < 1e-2 * max(1.0, ref.abs().max().item()), (rel, err)
    if Cout % 64 == 0 and info[5]:
        gamma = torch.randn(Cout, device="cuda", generator=g)
        beta = torch.randn(Cout, device="cuda", generator=g)
        got = ops.gn_apply_fold(y, None, part, info[6] // NB, None, 0, gamma, beta, act=1)
        want = ops.gn_apply(y, None, ops.gn_stats(y), gamma, beta, act=1)
        torch.cuda.synchronize()
        assert (got.float() - want.float()).abs().max().item() <= 2e-3 * max(1.0, want.float().abs().max().item())
