"""GPU: the UNet's and the MoVQ's attention kernels against float64 in fp16 ulps, at the geometry the model builds.

  k2_attention_d64    the UNet's head-width-64 attention (wgmma, TMA-fed), at every attention level of bench.py's UNet for
                      cfg-2 (96 x 96, batch 8), cfg-2' (64 x 96, batch 8) and cfg-3 (128 x 128, batch 4 per GPU), with the
                      encoder-token counts the 2.1 and 2.2 plans are built with;
  k2_attention_d512   the MoVQ AttnBlock (one head of width 512, output channels split over two CTAs), at the token counts of
                      CONFIG_2_2's decoder and encoder at latents 64^2, 96^2, 64 x 96 and 128^2, at lengths the ABI accepts and
                      the model never builds, with scores up to +-60, NaN next to the data, value halves drawn differently,
                      and for bit identity across batch sizes and graph replay;
  k2_softmax_rows     the unfused MoVQ attention's softmax (C != 512), with its own allowance.
The attention bound is tests/attention_ref.py's: one fp16 ulp of the float64 value plus the first-order error of the kernels'
fp32 arithmetic.  Every reference is evaluated one image at a time.  Each test prints its worst error in ulps and its largest
share of the bound (run with -s)."""
import inspect

import pytest
import torch

from tests.attention_ref import U, check, check_d64, ref_attention
from tests.test_gpu_prior_kernels import _ulp16

pytestmark = pytest.mark.gpu


def _gen(seed):
    return torch.Generator(device="cuda").manual_seed(seed)


# ------------------------------------------------------------------------------------------------------------------------------
# geometry: derived from the model code, not chosen here
# ------------------------------------------------------------------------------------------------------------------------------
def _unet_attention_levels():
    """{(downsampling factor, heads)} of bench.py's UNet attention blocks (num_head_channels 64)."""
    import bench
    from kandinsky2.model.unet import _topology
    cfg = bench.UNET_CFG
    mult = tuple(cfg["channel_mult"])
    inp, mid, out = _topology(cfg["in_channels"], cfg["model_channels"], mult, cfg["num_res_blocks"],
                              tuple(cfg["attention_resolutions"]))
    ds, levels = 1, set()
    for blk in inp:
        for item in blk:
            if item[0] == "attn":
                levels.add((ds, item[1] // 64))
            if item[0] == "res" and item[3] == "down":
                ds *= 2
    levels |= {(ds, item[1] // 64) for item in mid if item[0] == "attn"}
    for blk in out:
        for item in blk:
            if item[0] == "attn":
                levels.add((ds, item[1] // 64))
            if item[0] == "res" and item[3] == "up":
                ds //= 2
    return sorted(levels)


def _encoder_tokens():
    """{version: encoder tokens} of the UNet plans: 2.2 = num_image_embs of bench.py's UNet; 2.1 = CONFIG_2_1's
    num_image_embs image tokens + the text encoder's sequence (the pipelines' embedder length)."""
    import bench
    from kandinsky2 import configs
    from kandinsky2.pipelines import SyntheticEmbedder
    text_len = inspect.signature(SyntheticEmbedder).parameters["text_len"].default
    return {"2.1": configs.CONFIG_2_1["model_config"]["num_image_embs"] + text_len, "2.2": bench.UNET_CFG["num_image_embs"]}


UNET_CFGS = {"cfg-2": (8, 96, 96), "cfg-2'": (8, 64, 96), "cfg-3": (4, 128, 128)}   # (UNet batch, latent h, latent w)


def _movq_attention(dd, h, w):
    """{(T, C)} of the MoVQ decoder's and encoder's AttnBlocks for an h x w latent (image 2^(levels - 1) times larger)."""
    from kandinsky2.vqgan.autoencoder import _enc_topology, _topology
    block_in, levels = _topology(dd)
    out, H, W = {(h * w, block_in)}, h, w          # decoder mid block
    for lv in levels:
        if lv["attn"]:
            out.add((H * W, lv["ch"]))
        if lv["up"]:
            H, W = 2 * H, 2 * W
    elv = _enc_topology(dd)
    s = 2 ** (len(elv) - 1)
    H, W = h * s, w * s
    for lv in elv:
        if lv["attn"]:
            out.add((H * W, lv["ch"]))
        if lv["down"]:
            H, W = H // 2, W // 2
    out.add((H * W, elv[-1]["ch"]))                 # encoder mid block
    return out


MOVQ_LATENTS = {(64, 64): 2, (96, 96): 4, (64, 96): 2, (128, 128): 2}   # latent -> batch


def _movq_d512_geometry():
    from kandinsky2 import configs
    dd = configs.CONFIG_2_2["image_enc_params"]["params"]["ddconfig"]
    cases = []
    for (h, w), B in MOVQ_LATENTS.items():
        tc = _movq_attention(dd, h, w)
        assert {C for _, C in tc} == {512}, tc
        cases += [(B, T) for T, _ in sorted(tc)]
    return cases


def test_derived_geometry_is_the_model_geometry():
    assert _unet_attention_levels() == [(2, 12), (4, 18), (8, 24)]
    assert _encoder_tokens() == {"2.1": 87, "2.2": 32}
    assert _movq_d512_geometry() == [(2, 4096), (4, 9216), (2, 6144), (2, 16384)]
    assert _softmax_geometry() == [(64, 64), (1024, 256), (9216, 512)]


# ------------------------------------------------------------------------------------------------------------------------------
# k2_attention_d64 at the UNet's geometry
# ------------------------------------------------------------------------------------------------------------------------------
def _d64_inputs(B, heads, T, Tc, seed, std=1.0):
    g = _gen(seed)
    qkv = (torch.randn(B, T, heads * 192, device="cuda", generator=g) * std)
    qkv.view(B, T, heads, 3, 64)[:, :, :, 2] /= std            # values of unit scale
    enc = torch.randn(B, Tc, heads * 128, device="cuda", generator=g)
    enc.view(B, Tc, heads, 2, 64)[:, :, :, 0] *= std
    return qkv.half(), enc.half()


def _d64_cases():
    cases = []
    for name, (N, h, w) in UNET_CFGS.items():
        for ds, heads in _unet_attention_levels():
            for ver, Tc in _encoder_tokens().items():
                cases.append((name, ver, N, heads, (h // ds) * (w // ds), Tc))
    return cases


@pytest.mark.parametrize("cfg,version,B,heads,T,Tc", _d64_cases())
def test_attention_d64_unet_geometry(cfg, version, B, heads, T, Tc):
    from kandinsky2 import ops
    qkv, enc = _d64_inputs(B, heads, T, Tc, seed=T + Tc + heads)
    out = ops.attention_d64(qkv, heads, enc)
    assert torch.isfinite(out).all()
    ulps, share = check_d64(out, qkv, enc, heads, (cfg, version))
    print(f"attention_d64 {cfg} {version} B={B} heads={heads} T={T} Tc={Tc}: worst {ulps:.2f} ulp, {share:.3f} of the bound")


@pytest.mark.parametrize("T,Tc", [(2304, 87), (576, 32), (300, 87)])
def test_attention_d64_large_scores_late_maximum(T, Tc):
    """q and k at std 3.6: scaled scores up to about +-60.  Query rows 0-2 get a dominant key at the last, second-to-last and
    first key of the last spatial block (their maximum arrives in the last key block), row 3 at the last key of the block
    before, rows 4-5 at the last two encoder keys."""
    from kandinsky2 import ops
    heads = 2
    qkv, enc = _d64_inputs(2, heads, T, Tc, seed=T + Tc, std=3.6)
    q = qkv.view(2, T, heads, 3, 64)
    e = enc.view(2, Tc, heads, 2, 64)
    for r, key in enumerate([T - 1, T - 2, (T - 1) // 128 * 128, (T - 1) // 128 * 128 - 1]):
        q[:, r, :, 0] = (q[:, key, :, 1].float() * 0.4).half()
    for r, key in ((4, Tc - 1), (5, Tc - 2)):
        q[:, r, :, 0] = (e[:, key, :, 0].float() * 0.4).half()
    out = ops.attention_d64(qkv, heads, enc)
    assert torch.isfinite(out).all()
    s = torch.einsum("thc,shc->hts", q[0, :, :, 0].double(), q[0, :, :, 1].double()) * 0.125
    assert s.abs().max() > 40
    ulps, share = check_d64(out, qkv, enc, heads, "large")
    print(f"attention_d64 large scores T={T} Tc={Tc}: worst {ulps:.2f} ulp, {share:.3f} of the bound")


# ------------------------------------------------------------------------------------------------------------------------------
# k2_attention_d512
# ------------------------------------------------------------------------------------------------------------------------------
def _d512_inputs(B, T, seed, std=1.0, guard_rows=0):
    """fp16 qkv [B, T, 1536].  V's channels 0-255 ~ N(1, 1), 256-511 ~ N(-1, 4): a split-CTA mix-up of the halves shows.
    Query rows 0-3 of each image get a dominant key at the first / last key of a 16-key block and at T - 1 (the maximum
    arrives in the last key block).  guard_rows: the tensor is the start of an allocation whose following rows are NaN."""
    g = _gen(seed)
    qkv = torch.randn(B, T, 1536, device="cuda", generator=g)
    qkv[..., :1024] *= std
    qkv[..., 1024:1280] += 1.0
    qkv[..., 1280:] = 2.0 * qkv[..., 1280:] - 1.0
    for r, key in enumerate([T - 1, 0, min(15, T - 1), (T // 2) // 16 * 16]):
        if r < T:
            kk = qkv[:, key, 512:1024]
            qkv[:, r, :512] = kk * (24.0 / (kk.pow(2).sum(-1, keepdim=True) * 512 ** -0.5))
    qkv = qkv.half()
    if guard_rows:
        buf = torch.full((B * T + guard_rows, 1536), float("nan"), device="cuda", dtype=torch.float16)
        buf[:B * T] = qkv.view(B * T, 1536)
        qkv = buf[:B * T].view(B, T, 1536)
    return qkv


def check_d512(out, qkv, what, images=None):
    scale = 512 ** -0.5
    ulps = share = 0.0
    for b in (range(qkv.shape[0]) if images is None else images):
        q, k, v = qkv[b, :, None].split(512, -1)
        u, s = check(out[b, :, None], *ref_attention(q, k, v, scale), (what, b))
        ulps, share = max(ulps, u), max(share, s)
    return ulps, share


@pytest.mark.parametrize("B,T", _movq_d512_geometry())
def test_attention_d512_movq_geometry(B, T):
    from kandinsky2 import ops
    qkv = _d512_inputs(B, T, seed=T + B)
    out = ops.attention_d512(qkv, 512 ** -0.5)
    assert torch.isfinite(out).all()
    ulps, share = check_d512(out, qkv, T)
    print(f"attention_d512 B={B} T={T}: worst {ulps:.2f} ulp, {share:.3f} of the bound")


@pytest.mark.parametrize("T", [1, 15, 17, 100, 200, 64, 5184])
def test_attention_d512_abi_lengths(T):
    """Partial 16-key blocks (1, 15, 17, 100, 200) and a half-filled last 128-row query tile (64, 5184), at std 1 and at
    std 3.2 (scores up to about +-60); the rows after the last image are NaN."""
    from kandinsky2 import ops
    ulps = share = 0.0
    for std in (1.0, 3.2):
        qkv = _d512_inputs(2, T, seed=T + int(std), std=std, guard_rows=160)
        out = ops.attention_d512(qkv, 512 ** -0.5)
        assert torch.isfinite(out).all()
        if std > 1 and T >= 64:
            q, k = qkv[0, :, :512].double(), qkv[0, :, 512:1024].double()
            assert (q @ k.T * 512 ** -0.5).abs().max() > 40
        u, s = check_d512(out, qkv, (T, std))
        ulps, share = max(ulps, u), max(share, s)
    print(f"attention_d512 T={T}: worst {ulps:.2f} ulp, {share:.3f} of the bound")


def test_attention_d512_large_scores_full_size():
    from kandinsky2 import ops
    qkv = _d512_inputs(1, 9216, seed=5, std=3.2)
    out = ops.attention_d512(qkv, 512 ** -0.5)
    assert torch.isfinite(out).all()
    ulps, share = check_d512(out, qkv, "large")
    print(f"attention_d512 T=9216 scores up to +-60: worst {ulps:.2f} ulp, {share:.3f} of the bound")


def test_attention_d512_next_image_nan():
    """Image 1 is all NaN: image 0's key and value loads must stop at its own last row."""
    from kandinsky2 import ops
    qkv = _d512_inputs(2, 9216, seed=6)
    qkv[1] = float("nan")
    out = ops.attention_d512(qkv, 512 ** -0.5)
    assert torch.isfinite(out[0]).all()
    ulps, share = check_d512(out, qkv, "nan", images=[0])
    print(f"attention_d512 T=9216 next image NaN: worst {ulps:.2f} ulp, {share:.3f} of the bound")


def test_attention_d512_bit_identity():
    """At T = 9216: a batch of 2 equals each image run alone; graph replay equals the eager launch; the batch-2 launch is
    unchanged after a launch at batch size 1 and one at 4.  Each comparison runs at most three times."""
    from kandinsky2 import ops
    T, scale = 9216, 512 ** -0.5
    qkv = _d512_inputs(4, T, seed=7)
    two = qkv[:2]
    eager = ops.attention_d512(two, scale)
    for b in range(2):
        assert torch.equal(ops.attention_d512(qkv[b:b + 1], scale)[0], eager[b]), b
    out = torch.empty_like(eager)
    s = torch.cuda.Stream()
    s.wait_stream(torch.cuda.current_stream())
    with torch.cuda.stream(s):
        ops.attention_d512(two, scale, out=out)
    torch.cuda.current_stream().wait_stream(s)
    graph = torch.cuda.CUDAGraph()
    with torch.cuda.graph(graph):
        ops.attention_d512(two, scale, out=out)
    for _ in range(3):
        out.zero_()
        graph.replay()
        torch.cuda.synchronize()
        assert torch.equal(out, eager)
    for other in (1, 4):
        ops.attention_d512(qkv[:other], scale)
        out.zero_()
        graph.replay()
        again = ops.attention_d512(two, scale)
        torch.cuda.synchronize()
        assert torch.equal(out, eager) and torch.equal(again, eager), other
    print("attention_d512 T=9216: batch of 2 = images alone, replay = eager, unchanged after batch 1 and 4")


# ------------------------------------------------------------------------------------------------------------------------------
# k2_softmax_rows: the unfused MoVQ attention (C != 512)
# ------------------------------------------------------------------------------------------------------------------------------
def _softmax_geometry():
    """[(n, C)]: the token counts and widths of the MoVQ configs that run the unfused path -- the golden tiny decoder (its
    fixture's ddconfig and latent) and the mid decoder of tests/test_gpu_movq_sampler.py (ch 64, mult (1, 2, 4),
    resolution 128, 32 x 32 latent) -- and T = 9216 at C = 512."""
    import os
    from oracle import movq_oracle as mo
    fx = torch.load(os.path.join(os.path.dirname(__file__), "golden", "movq_tiny.pt"), weights_only=False)
    h, w = fx["z"].shape[2:]
    tiny = _movq_attention(fx["dd"], h, w)
    mid = _movq_attention(dict(mo.DDCONFIG_2_1, ch=64, ch_mult=(1, 2, 4), resolution=128), 32, 32)
    return sorted(tiny | mid) + [(9216, 512)]


@pytest.mark.parametrize("n,C", _softmax_geometry())
def test_softmax_rows_vs_float64(n, C):
    """softmax(scale x) of fp16 scores x = q.k (unscaled, as the batched GEMM writes them), scale = C^-0.5, against float64
    of the same fp16 x.  The kernel computes m = max x, mo = m c (c = scale log2 e in fp32), p = exp2f(fmaf(x, c, -mo)),
    the row sum (a chain of n / 256 + 13 fp32 additions), 1 / sum and the product.  Per element, relative to the output p:
      eta_s = 2^-22 (|s| + |max s|) + 2^-21   the fma's rounding and exp2f (2 ulp), as in tests/attention_ref.py,
      sum_j p_j eta_j                           the row sum's weights,
      (n / 256 + 16) 2^-24                      the row sum's chain, 1 / sum and the product,
    plus one fp16 ulp of p.  The bound starts from the fp16 scores: their own rounding is not in it.  At C = 512 that
    rounding is 2^-11 |x| relative, i.e. up to 2^-11 |s| in a scaled score s; at |s| = 20 a weight moves by 1 %, about 2^11
    times the kernel's own allowance.  The unfused path is therefore only as accurate as fp16 scores allow, and C = 512
    runs the fused kernel, whose scores stay fp32."""
    from kandinsky2 import ops
    rows = 256
    g = _gen(n + C)
    ulps = share = 0.0
    for spread in (1.0, 8.0):                 # scaled scores ~ N(0, spread^2): up to about +-40 at 8
        x = (torch.randn(rows, n, device="cuda", generator=g) * (spread * C ** 0.5)).half()
        x[0, -1] = x[0].max() + 30 * C ** 0.5     # a row whose maximum is its last element
        y = ops.softmax_rows(x, C ** -0.5)
        s = x.double() * C ** -0.5
        p = torch.softmax(s, -1)
        eta = 2.0 ** -22 * (s.abs() + s.amax(-1, keepdim=True).abs()) + 2.0 ** -21
        allow = p * (eta + (p * eta).sum(-1, keepdim=True) + (n / 256 + 16) * U)
        err = (y.double() - p).abs()
        bound = _ulp16(p) + allow
        bad = ~(err <= bound)
        assert not bad.any(), (n, C, spread, int(bad.sum()), y.double()[bad][:4].tolist(), p[bad][:4].tolist())
        ulps = max(ulps, (err / _ulp16(p)).max().item())
        share = max(share, (err / bound).max().item())
    print(f"softmax_rows n={n} C={C}: worst {ulps:.2f} ulp, {share:.3f} of the bound")
