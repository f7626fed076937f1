"""k2_conv_gemm issues one m64nNk16 wgmma per K step for the whole N tile (N = 128 / 192 / 256).  The launch plans' autotuner
and bench.py --dump-outputs rely on the N tile never changing a result bit, so every wide configuration must reproduce the
N tile 64 kernel (one m64n64k16 per K step) exactly: the stored output and the fused GroupNorm partial statistics."""
import pytest
import torch

pytestmark = pytest.mark.gpu

# (N tile, epilogue warp sets); two sets exist for the N tiles 128 and 256 only
WIDE = [(128, 1), (128, 2), (192, 1), (256, 1), (256, 2)]


def _rand(g, *shape, scale=1.0):
    return (torch.randn(*shape, device="cuda", generator=g) * scale).half()


def _case(name, g):
    """-> (run(cfg) -> (out, partials or None), splits)"""
    from kandinsky2 import ops
    if name == "level1_three_segments":
        # up-path ResBlock at UNet level 1: 3x3 of the normed h plus the 1x1 skip over the un-materialised concat [x | skip]
        NB, H, W, Ch, Ca, Cb, Cout = 8, 48, 48, 768, 768, 384, 768
        h = _rand(g, NB, H, W, Ch)
        buf = _rand(g, NB, H, W, Ca + Cb)
        xa, xb = buf[..., :Ca], buf[..., Ca:]
        w3 = torch.randn(Cout, Ch, 3, 3, device="cuda", generator=g) / (3 * Ch ** 0.5)
        w1 = torch.randn(Cout, Ca + Cb, 1, 1, device="cuda", generator=g) / (Ca + Cb) ** 0.5
        wp = torch.cat([ops.pack_conv_weight(w3), ops.pack_conv_weight(w1, split=(Ca, Cb))], 1).contiguous()
        b = torch.randn(Cout, device="cuda", generator=g)
        srcs, kw, geom, splits = [(h, 9), (xa, 1), (xb, 1)], dict(bias=b), (NB, H, W), 1
    elif name == "identity_skip_residual":
        NB, H, W, C = 8, 24, 24, 1152
        x = _rand(g, NB, H, W, C)
        wp = ops.pack_conv_weight(torch.randn(C, C, 3, 3, device="cuda", generator=g) / (3 * C ** 0.5))
        kw = dict(bias=torch.randn(C, device="cuda", generator=g), residual=_rand(g, NB, H, W, C))
        srcs, Cout, geom, splits = [(x, 9)], C, (NB, H, W), 1
    elif name == "up2_four_taps":
        NB, H, W, C = 8, 24, 24, 1152
        x = _rand(g, NB, H, W, C)
        wp = ops.pack_conv_weight_up2(torch.randn(C, C, 3, 3, device="cuda", generator=g) / (3 * C ** 0.5))
        kw = dict(bias=torch.randn(C, device="cuda", generator=g))
        srcs, Cout, geom, splits = [(x, 4)], C, (NB, 2 * H, 2 * W), 1
    elif name == "split_k2":
        NB, H, W, C = 8, 12, 12, 1536
        x = _rand(g, NB, H, W, C)
        wp = ops.pack_conv_weight(torch.randn(C, C, 3, 3, device="cuda", generator=g) / (3 * C ** 0.5))
        kw = dict(bias=torch.randn(C, device="cuda", generator=g), residual=_rand(g, NB, H, W, C))
        srcs, Cout, geom, splits = [(x, 9)], C, (NB, H, W), 2
    elif name == "per_image_weights":
        # MoVQ attention scores: image n multiplies its query rows by its own key rows (ragged N: 576 = 2 x 256 + 64)
        NB, T, C = 2, 576, 512
        q = _rand(g, NB, 1, T, C)
        k = _rand(g, NB, T, C, scale=C ** -0.5)
        out = torch.empty(NB, 1, T, T, dtype=torch.float16, device="cuda")

        def run(cfg):
            info = [0] * 7
            y = ops.conv_gemm([(q, 1)], k[0], T, out=out, info=info, cfg=cfg, w_batch_stride=T * C)
            assert info[0] == cfg[0] and info[2] == 1, info
            return y.clone(), None
        return run, 1
    elif name == "gemm_rows_qkv":
        M, K, N = 18432, 768, 2304
        x = _rand(g, M, K)
        wp = ops.pack_conv_weight(torch.randn(N, K, device="cuda", generator=g) / K ** 0.5)
        b = torch.randn(N, device="cuda", generator=g)

        def run(cfg):
            info = [0] * 7
            y = ops.gemm_rows(x, wp, N, bias=b, cfg=cfg, info=info)
            assert info[0] == cfg[0] and info[2] == 1, info
            return y.clone(), None
        return run, 1
    else:
        raise AssertionError(name)

    def run(cfg):
        part = torch.zeros(ops.gn_part_floats(*geom, Cout), device="cuda")
        info = [0] * 7
        y = ops.conv_gemm(srcs, wp, Cout, gn_part=part, info=info, cfg=cfg, **kw)
        assert info[0] == cfg[0] and info[2] == cfg[2], info
        assert info[5] == (1 if cfg[2] == 1 else 2), info  # the partials come from the epilogue / the split-K second pass
        return y.clone(), part.clone()
    return run, splits


@pytest.mark.parametrize("name", ["level1_three_segments", "identity_skip_residual", "up2_four_taps", "split_k2",
                                  "per_image_weights", "gemm_rows_qkv"])
def test_wide_n_tile_matches_n64(name):
    g = torch.Generator(device="cuda").manual_seed(21)
    run, splits = _case(name, g)
    ref_y, ref_part = run((64, 0, splits, 1))
    torch.cuda.synchronize()
    assert ref_y.abs().float().max().item() > 0
    for bn, es in WIDE:
        y, part = run((bn, 0, splits, es))
        torch.cuda.synchronize()
        assert torch.equal(y, ref_y), f"N tile {bn}, {es} epilogue set(s): output differs from N tile 64"
        if ref_part is not None:
            assert torch.equal(part, ref_part), f"N tile {bn}, {es} epilogue set(s): GroupNorm partials differ"
