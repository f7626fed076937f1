"""CPU: the per-block float64 bounds of tests/plan_blocks_ref.py are neither too tight nor vacuous, on CONFIG_TINY /
DDCONFIG_TINY, all in float64.

Each block's inputs are the fp32 oracle's own activations at that block (recorded by wrapping the oracle's block functions),
rounded to fp16 as a plan holds them.  An emulated plan -- fp16 weights (the up2 phase sums rounded once), fp16 rounding at
every storage point, float64 elsewhere -- must stay inside the bound; every wiring error of plan_blocks_ref.MUTATIONS must
leave it by a factor of at least 4 on some element."""
import pytest
import torch
import torch.nn.functional as F

from tests import plan_blocks_ref as R

MIN_REJECT = 4.0


def _h(x):
    """An activation as the plan stores it: fp16, read back exactly."""
    v = x.half().double()
    return R.V(v, torch.zeros_like(v))


def _check(kind, name, ref, emulated, muts):
    worst, med = R.share(emulated, ref)
    print(f"{kind} {name}: emulated plan at {worst:.3f} of the bound (median {med:.3f})")
    assert worst <= 1.0, (kind, name, worst)
    for mut, got in muts.items():
        w, _ = R.share(got, ref)
        print(f"  mutation {mut}: {w:.1f} x the bound")
        assert w >= MIN_REJECT, (kind, name, mut, w)
    return set(muts)


def _check_block(kind, name, run, muts):
    """run(M, snap) -> {stage: V}.  The emulated plan's stages are the snapshots each exact stage starts from, as the plan's
    are on the GPU; each mutation is evaluated from the same snapshots."""
    em = run(R.Mode(em=True), None)
    snap = {k: R.V(v.v, torch.zeros_like(v.v)) for k, v in em.items() if k != "out"}
    ref = run(R.EXACT, snap)
    worst, med, per = R.check_stages({k: v.v for k, v in em.items()}, ref)
    print(f"{kind} {name}: emulated plan at {worst:.3f} of the bound (median {med:.3f}) " +
          " ".join(f"{k} {s:.2f}" for k, s in per.items()))
    assert worst <= 1.0, (kind, name, per)
    for mut, M in muts.items():
        got = run(M, snap)
        w, _, per = R.check_stages({k: v.v for k, v in got.items()}, ref)
        print(f"  mutation {mut}: {w:.1f} x the bound")
        assert w >= MIN_REJECT, (kind, name, mut, per)
    return set(muts)


def _unet_inputs(cfg, seed=5):
    from oracle import synth
    from oracle import unet_oracle as uo
    sd = synth.synth_state_dict(uo.unet_param_spec(cfg), seed=seed)
    g = torch.Generator().manual_seed(seed)
    B, H, W = 2, 16, 16
    kw = dict(image_emb=torch.randn(B, cfg["image_encoder_in_dim"], generator=g),
              full_emb=torch.randn(B, 7, cfg["text_encoder_in_dim1"], generator=g),
              pooled_emb=torch.randn(B, cfg["text_encoder_in_dim2"], generator=g))
    x = torch.randn(B, 4, H, W, generator=g)
    t = torch.tensor([981.0, 40.0])
    return sd, x, t, kw


def test_unet_tiny_blocks(monkeypatch):
    from oracle import unet_oracle as uo
    cfg = uo.CONFIG_TINY
    sd, x, t, kw = _unet_inputs(cfg)
    rec = []
    orig_res, orig_attn = uo._res, uo._attn
    monkeypatch.setattr(uo, "_res", lambda x, emb, sd_, p, ud: rec.append(("res", p, x, emb, ud)) or orig_res(x, emb, sd_, p, ud))
    monkeypatch.setattr(uo, "_attn", lambda x, xf, sd_, p, hc: rec.append(("attn", p, x, xf, None)) or orig_attn(x, xf, sd_, p, hc))
    with torch.no_grad():
        uo.unet_forward(sd, cfg, x, t, **kw)
    monkeypatch.undo()
    table = {p: c0 for p, _, c0 in R.unet_block_table(cfg)}
    lay = R.film_layout(cfg)
    assert [r[1] for r in rec] == list(table)
    seen = set()
    for kind, p, xin, side, ud in rec:
        c0 = table[p]
        a = _h(xin[:, :c0])
        b = _h(xin[:, c0:]) if c0 < xin.shape[1] else None
        if kind == "res":
            film_of = lambda q: F.linear(F.silu(side.double()), sd[q + "emb_layers.1.weight"].double(),  # noqa: E731
                                         sd[q + "emb_layers.1.bias"].double())
            film, film_nb = film_of(p), film_of(R.film_neighbour(lay, p))

            def run(M, snap, film=film, film_nb=film_nb):
                return R.unet_res(sd, p, a, b, film_nb if M.mut == "film_neighbour" else film, ud, M, snap)
            names = ["film_neighbour", "film_scale"] + (["gn_first_source"] if b is not None else [])
            names += (["res_unresampled"] if ud is not None else []) + (["up2_plain"] if ud == "up" else [])
        else:
            enc = (F.conv1d(side, sd[p + "encoder_kv.weight"], sd[p + "encoder_kv.bias"]).permute(0, 2, 1)).half()
            run = lambda M, snap: R.unet_attn(sd, p, a, enc, M, snap)  # noqa: E731
            names = ["no_enc"]
        seen |= _check_block(kind, p, run, {m: R.Mode(mut=m) for m in names})
    assert seen == {"film_neighbour", "film_scale", "gn_first_source", "res_unresampled", "up2_plain", "no_enc"}


def test_unet_tiny_film_chain():
    """The forked conditioning branch (time embedding, time_embed MLP + xf_proj, the one FiLM GEMM over every ResBlock) as an
    emulated plan: fp32 storage of e0 / e1 / emb / film, fp16 FiLM weights."""
    from oracle import unet_oracle as uo
    cfg = uo.CONFIG_TINY
    sd, _, t, _ = _unet_inputs(cfg)
    lay = R.film_layout(cfg)
    xf_proj = torch.randn(2, 4 * cfg["model_channels"], generator=torch.Generator().manual_seed(12))
    run = lambda M, snap: R.film_chain(sd, lay, t, xf_proj, M, snap)  # noqa: E731
    names = ["film_packed_neighbour", "emb_no_xf_proj", "film_no_silu_in"]
    _check_block("film", "chain", run, {m: R.Mode(mut=m) for m in names})
    # the emulated chain equals the oracle's own emb_layers(silu(emb)) to fp16-weight accuracy: the restatement's wiring
    emb = uo.timestep_embedding(t, cfg["model_channels"]).double()
    emb = F.linear(F.silu(F.linear(emb, sd["time_embed.0.weight"].double(), sd["time_embed.0.bias"].double())),
                   sd["time_embed.2.weight"].double(), sd["time_embed.2.bias"].double()) + xf_proj.double()
    want = torch.cat([F.linear(F.silu(emb), sd[p + "emb_layers.1.weight"].double(), sd[p + "emb_layers.1.bias"].double())
                      for p in lay], 1)
    assert torch.allclose(run(R.Mode(bound=False), None)["out"].v, want, rtol=1e-5, atol=1e-5)


def test_unet_tiny_stem_and_head():
    from oracle import unet_oracle as uo
    cfg = uo.CONFIG_TINY
    sd, x, _, _ = _unet_inputs(cfg)
    ref = R.unet_stem(sd, x)
    _check("stem", "input_blocks.0.0", ref, R.unet_stem(sd, x, R.Mode(em=True)).v, {})
    h = _h(torch.randn(2, 64, 16, 16, generator=torch.Generator().manual_seed(3), dtype=torch.float64) * 2 + 0.5)
    _check("head", "out", R.unet_head(sd, h), R.unet_head(sd, h, R.Mode(em=True)).v, {})


def _movq_sd(dd, seed=7):
    from oracle import movq_oracle as mo
    from oracle import synth
    return synth.synth_state_dict(mo.movq_param_spec(dd, 4, 64), seed=seed)


def test_movq_tiny_decoder_blocks(monkeypatch):
    from oracle import movq_oracle as mo
    dd = mo.DDCONFIG_TINY
    sd = _movq_sd(dd)
    z = torch.randn(2, 4, 8, 8, generator=torch.Generator().manual_seed(1))
    rec = []
    orig_res, orig_attn = mo._res, mo._attn
    monkeypatch.setattr(mo, "_res", lambda x, zq, sd_, p: rec.append(("res", p, x)) or orig_res(x, zq, sd_, p))
    monkeypatch.setattr(mo, "_attn", lambda x, zq, sd_, p: rec.append(("attn", p, x)) or orig_attn(x, zq, sd_, p))
    with torch.no_grad():
        mo.movq_decode(sd, dd, z)
    monkeypatch.undo()
    seen = set()
    for kind, p, xin in rec:
        a = _h(xin)
        if kind == "res":
            run = lambda M, snap: R.movq_res(sd, p, a, z, M, snap)  # noqa: E731
            names = ["zq_offset"]
        else:
            assert xin.shape[1] != 512
            run = lambda M, snap: R.movq_attn(sd, p, a, z, False, M, snap)  # noqa: E731
            names = ["no_scale", "zq_offset"]
        seen |= _check_block(kind, p, run, {m: R.Mode(mut=m) for m in names})
    assert seen == {"zq_offset", "no_scale"} and any(k == "attn" for k, *_ in rec)
    # the up conv, the stem and the head
    h = _h(torch.randn(2, 64, 8, 8, generator=torch.Generator().manual_seed(2), dtype=torch.float64))
    p = "decoder.up.1."
    _check("upconv", p, R.movq_upconv(sd, p, h), R.movq_upconv(sd, p, h, R.Mode(em=True)).v,
           {"up2_plain": R.movq_upconv(sd, p, h, R.Mode(mut="up2_plain")).v})
    ref_up = F.conv2d(F.interpolate(h.v, scale_factor=2.0, mode="nearest"), sd[p + "upsample.conv.weight"].double(),
                      sd[p + "upsample.conv.bias"].double(), padding=1)
    assert torch.allclose(R.movq_upconv(sd, p, h).v, ref_up, rtol=1e-12, atol=1e-12)
    _check("stem", "decoder.conv_in", R.movq_dec_stem(sd, z), R.movq_dec_stem(sd, z, R.Mode(em=True)).v, {})
    h2 = _h(torch.randn(2, 32, 32, 32, generator=torch.Generator().manual_seed(4), dtype=torch.float64))
    _check("head", "decoder.conv_out", R.movq_dec_head(sd, h2, z), R.movq_dec_head(sd, h2, z, R.Mode(em=True)).v, {})


def test_movq_tiny_encoder_blocks(monkeypatch):
    from oracle import movq_oracle as mo
    dd = mo.DDCONFIG_TINY
    sd = _movq_sd(dd)
    img = torch.rand(2, 3, 32, 32, generator=torch.Generator().manual_seed(6)) * 2 - 1
    rec = []
    orig_res, orig_attn = mo._enc_res, mo._enc_attn
    monkeypatch.setattr(mo, "_enc_res", lambda x, sd_, p: rec.append(("res", p, x)) or orig_res(x, sd_, p))
    monkeypatch.setattr(mo, "_enc_attn", lambda x, sd_, p: rec.append(("attn", p, x)) or orig_attn(x, sd_, p))
    with torch.no_grad():
        mo.movq_encode(sd, dd, img)
    monkeypatch.undo()
    for kind, p, xin in rec:
        a = _h(xin)
        if kind == "res":
            run = lambda M, snap: R.movq_res(sd, p, a, None, M, snap)  # noqa: E731
            names = []
        else:
            run = lambda M, snap: R.movq_attn(sd, p, a, None, False, M, snap)  # noqa: E731
            names = ["no_scale"]
        _check_block("enc " + kind, p, run, {m: R.Mode(mut=m) for m in names})
    h = _h(torch.randn(2, 32, 32, 32, generator=torch.Generator().manual_seed(8), dtype=torch.float64))
    p = "encoder.down.0."
    ref = R.movq_downconv(sd, p, h)
    assert torch.allclose(ref.v, R.downsample_oracle(sd, p, h.v), rtol=1e-12, atol=1e-12)
    _check("downconv", p, ref, R.movq_downconv(sd, p, h, R.Mode(em=True)).v, {})
    _check("stem", "encoder.conv_in", R.movq_enc_stem(sd, img), R.movq_enc_stem(sd, img, R.Mode(em=True)).v, {})
    h2 = _h(torch.randn(2, 64, 16, 16, generator=torch.Generator().manual_seed(9), dtype=torch.float64))
    _check("head", "encoder.conv_out", R.movq_enc_head(sd, h2), R.movq_enc_head(sd, h2, R.Mode(em=True)).v, {})


@pytest.mark.parametrize("C", [64, 512])
def test_fused_attention_bound_covers_emulation(C):
    """The fused route's bound (kernel allowance + input errors) against an emulation that rounds q, k, v to fp16 from an
    exact float64 projection: the carried input error must cover the difference."""
    g = torch.Generator().manual_seed(C)
    T = 64
    q, k, v = (torch.randn(T, 1, C, generator=g, dtype=torch.float64) * 2 for _ in range(3))
    e = lambda t: R.V(t, R.U16 * t.abs() + R.TINY)  # noqa: E731
    ref = R.attend(e(q), e(k), e(v), C ** -0.5, R.EXACT, fused=True)
    got = R.attend(R.V(q.half().double()), R.V(k.half().double()), R.V(v.half().double()), C ** -0.5, R.Mode(em=True)).v
    worst, _ = R.share(got, ref)
    assert worst <= 1.0, worst
