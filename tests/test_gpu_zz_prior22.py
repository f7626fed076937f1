"""GPU: the Kandinsky 2.2 diffusion prior -- the two copy kernels of the graph-replayed step (k2_prior_tokens, k2_f16_to_f32),
the UnCLIP rows on k2_sampler_step, the step graph against PriorTransformer.forward and the oracle loop (tests/prior22_oracle.py),
the full 2.2 size on synthetic weights, and PriorEmbedder22 behind the 2.2 pipelines.

The full-size test is calibrated as tests/test_gpu_zz_prior_full.py is: the product must be at least as close to the fp32
oracle as the oracle in fp16 is, in max-abs AND relative L2, with the GEMM weights as the product stores them (fp16).  About
12 GB of device memory."""
import pytest
import torch

from tests import prior22_oracle as p22

pytestmark = pytest.mark.gpu


def _bits16(t):
    return t.contiguous().view(torch.int16)


def test_prior_tokens_bit_exact_against_the_torch_composition():
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(0)
    M, N, n = 6, 2048 + 6, 9
    # fp32 rows around fp16 rounding ties, large values that round to fp16 infinity, and tiny ones that go subnormal
    x_full = torch.randn(M, N + 10, device="cuda", generator=g) * torch.tensor([1.0, 1e-6, 3e4, 7e4, 1.0, 0.001],
                                                                              device="cuda")[:, None]
    x = x_full[:, 3:3 + N]
    pos_full = (torch.randn(n, N + 4, device="cuda", generator=g) * 2).half()
    pos = pos_full[:, :N]
    seq = torch.full((M, n, N), float("nan"), device="cuda", dtype=torch.float16)
    # one positional row for all M rows, written at the sequence's row stride (the step's token rows 78 / 79)
    ops.prior_tokens(x, pos[4:5].expand(M, N), seq[:, 4])
    ref = x.half() + pos[4]
    assert torch.equal(_bits16(seq[:, 4]), _bits16(ref))
    assert torch.isnan(seq[:, :4]).all() and torch.isnan(seq[:, 5:]).all()      # neighbours untouched
    # per-row positional rows (the text tokens of one sample), and one source row for every output row (prd_emb)
    out = torch.full((n, N), float("nan"), device="cuda", dtype=torch.float16)
    xr = torch.randn(n, N, device="cuda", generator=g)
    ops.prior_tokens(xr, pos, out)
    assert torch.equal(_bits16(out), _bits16(xr.half() + pos))
    one = torch.randn(1, N, device="cuda", generator=g)
    ops.prior_tokens(one.expand(M, N), pos[8:9].expand(M, N), seq[:, 8])
    assert torch.equal(_bits16(seq[:, 8]), _bits16((one.half() + pos[8]).expand(M, N)))


def test_f16_to_f32_exact():
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(1)
    x = (torch.randn(5, 81, 2048, device="cuda", generator=g) * 300).half()
    x[0, -1, :4] = torch.tensor([float("inf"), -float("inf"), 6e-8, -0.0], device="cuda").half()
    last = x[:, -1]                                              # the strided last-token rows
    out = torch.full((5, 2048 + 8), float("nan"), device="cuda")
    ops.f16_to_f32(last, out=out[:, :2048])
    assert torch.equal(out[:, :2048], last.float())
    assert torch.isnan(out[:, 2048:]).all()
    assert torch.equal(ops.f16_to_f32(x[0, :3]), x[0, :3].float())


def test_sampler_step_unclip_rows_against_float64():
    """k2_sampler_step with every UnCLIP row of a 25-step schedule (H = 1, W = 320, clip 10, unconditional rows first), against
    float64 of the same fp32 inputs and coefficients: a few fp32 ulps of the terms.  At t = 0 NaN noise gives the zero-noise
    bits."""
    from kandinsky2 import ops
    from kandinsky2.model.prior import UnCLIPSchedule
    B, D, gd = 3, 1280, 4.0
    g = torch.Generator(device="cuda").manual_seed(2)
    pred = torch.zeros(2 * B, 2 * D, device="cuda")
    pred[:, :D] = torch.randn(2 * B, D, device="cuda", generator=g) * 4     # CFG reaches past the +-10 clamp
    x_in = torch.randn(B, D, device="cuda", generator=g)
    z = torch.randn(B, D, device="cuda", generator=g)
    work = torch.empty(B * D + 4096, device="cuda")
    table = torch.from_numpy(UnCLIPSchedule(25).coef_table()).cuda()
    mo = pred.view(2 * B, 8, 1, D // 4)
    worst = 0.0
    for k in range(25):
        r = table[k]
        x = x_in.clone()
        ops.sampler_step(mo, x.view(B, 4, 1, D // 4), z.view(B, 4, 1, D // 4), r, gd, 0, clip=10.0, threshold_mode=0, work=work)
        rd, u, c = r.double(), pred[:B, :D].double(), pred[B:, :D].double()
        eps = u + gd * (c - u)
        x0 = (rd[0] * x_in.double() - rd[1] * eps).clamp(-10, 10)
        noise = rd[6] * torch.exp(0.5 * (0.5 * rd[5] + 0.5 * rd[4])) * z.double()
        ref = rd[2] * x0 + rd[3] * x_in.double() + noise
        scale = (rd[2] * x0).abs() + (rd[3] * x_in.double()).abs() + noise.abs() + 1e-30
        err = ((x.double() - ref).abs() / (scale * 2.0 ** -24)).max().item()
        worst = max(worst, err)
        assert err <= 6.0, (k, err)
    last = table[24]
    assert last[6].item() == 0.0
    xa, xb = x_in.clone(), x_in.clone()
    ops.sampler_step(mo, xa.view(B, 4, 1, D // 4), torch.zeros_like(z).view(B, 4, 1, D // 4), last, gd, 0, clip=10.0, work=work)
    ops.sampler_step(mo, xb.view(B, 4, 1, D // 4), torch.full_like(z, float("nan")).view(B, 4, 1, D // 4), last, gd, 0, clip=10.0,
                     work=work)
    assert torch.equal(xa, xb)
    print(f"UnCLIP rows on k2_sampler_step: worst {worst:.2f} fp32 ulps of the terms")


# ---------------------------------------------------------------------------------------------------------------------------
# tiny prior from a diffusers-named state dict
# ---------------------------------------------------------------------------------------------------------------------------
def _prior_from_diffusers(cfg, seed, round_gemm=False):
    from kandinsky2.checkpoints import diffusers_prior_to_k2
    from kandinsky2.model.prior import PriorTransformer
    from oracle import synth
    dsd = {k: v.cuda() for k, v in synth.synth_state_dict(p22.diffusers_prior_spec(cfg), seed=seed).items()}
    if round_gemm:   # the weights as the product stores them: the transformer and text_enc_proj GEMM matrices in fp16
        gemm = ("attn1.to_q.weight", "attn1.to_k.weight", "attn1.to_v.weight", "attn1.to_out.0.weight", "ff.net.0.proj.weight",
                "ff.net.2.weight", "encoder_hidden_states_proj.weight")
        for k in dsd:
            if k.endswith(gemm):
                dsd[k] = dsd[k].half().float()
    sd, _, _ = diffusers_prior_to_k2(dsd)
    m = PriorTransformer(**cfg, device="cuda")
    m.load_state_dict(sd, strict=True)
    del sd
    return m.finalize(), dsd


def _cond(cfg, B, prompt_len, seed):
    """CFG rows [uncond x B | cond x B] (diffusers' order): the empty prompt's CLIP mask keeps its start and end tokens."""
    g = torch.Generator(device="cuda").manual_seed(seed)
    D, L, X = cfg["clip_dim"], cfg["text_ctx"], cfg["clip_xf_width"]
    text_emb = torch.randn(2, D, device="cuda", generator=g).repeat_interleave(B, 0)
    text_enc = torch.randn(2, L, X, device="cuda", generator=g).repeat_interleave(B, 0)
    lens = torch.tensor([2] * B + [prompt_len] * B, device="cuda")
    mask = torch.arange(L, device="cuda")[None, :] < lens[:, None]
    return text_emb, text_enc, mask, g


@pytest.fixture(scope="module")
def tiny():
    from kandinsky2 import launch_plan
    old = launch_plan.TUNE_SMALL_M
    launch_plan.TUNE_SMALL_M = 0     # bit-identical GEMM configurations only (as bench.py --dump-outputs)
    cfg = p22.CONFIG_PRIOR22_TINY
    m, dsd = _prior_from_diffusers(cfg, seed=5)
    yield cfg, m, dsd
    launch_plan.TUNE_SMALL_M = old


@pytest.mark.parametrize("B", [1, 3])
def test_graph_step_equals_eager_forward_bit_for_bit(tiny, B):
    from kandinsky2.model.prior import UnCLIPSchedule
    cfg, m, _ = tiny
    D = cfg["clip_dim"]
    te, tenc, mask, g = _cond(cfg, B, 4, seed=B)
    x_T = torch.randn(B, D, device="cuda", generator=g)
    sched = UnCLIPSchedule(5)
    plan = m._step_plan(B)
    plan.bind(te, tenc, mask)
    plan.set_schedule(sched, x_T, torch.randn(5, B, D, device="cuda", generator=g), 4.0)
    x = x_T.clone()
    for k, t in enumerate(sched.timesteps[:3]):
        plan.run(True)
        ref = m(torch.cat([x, x]), torch.full((2 * B,), float(t), device="cuda"), text_emb=te, text_enc=tenc, mask=mask)
        assert torch.equal(plan.model_out[:, :D], ref), k
        assert (plan.model_out[:, D:] == 0).all()
        x = plan.x.clone()


def test_graph_replay_equals_step_at_a_time_and_is_deterministic(tiny):
    from kandinsky2.model.prior import sample_prior22
    cfg, m, _ = tiny
    B, D, N = 2, cfg["clip_dim"], 10
    te, tenc, mask, g = _cond(cfg, B, 5, seed=7)
    x_T = torch.randn(B, D, device="cuda", generator=g)
    noise = torch.randn(N, B, D, device="cuda", generator=g)
    mean, std = 0.1 * torch.randn(D, device="cuda", generator=g), 0.5 + torch.rand(D, device="cuda", generator=g)
    a = sample_prior22(m, te, tenc, mask, N, 4.0, mean, std, x_T, noise, use_graph=True)
    b = sample_prior22(m, te, tenc, mask, N, 4.0, mean, std, x_T, noise, use_graph=False)
    c = sample_prior22(m, te, tenc, mask, N, 4.0, mean, std, x_T, noise, use_graph=True)
    assert torch.isfinite(a).all() and torch.equal(a, b) and torch.equal(a, c)
    d = sample_prior22(m, te, tenc, mask, N, 2.0, mean, std, x_T, noise)       # a new guidance scale: a new graph
    assert not torch.equal(a, d)
    assert torch.equal(a, sample_prior22(m, te, tenc, mask, N, 4.0, mean, std, x_T, noise))


@pytest.mark.parametrize("N,guidance", [(5, 4.0), (25, 4.0), (10, 1.0)])
def test_sampling_matches_the_oracle_unclip_loop(tiny, N, guidance):
    """The graph-replayed loop against the diffusers-form forward (fp32) under the float64 UnCLIP loop, same noise.  Without
    guidance the oracle runs the conditional rows alone and the product runs them twice (its CFG of equal halves is exact)."""
    from kandinsky2.model.prior import sample_prior22
    cfg, m, dsd = tiny
    B, D = 2, cfg["clip_dim"]
    te, tenc, mask, g = _cond(cfg, B, 3, seed=N)
    if guidance <= 1.0:
        te, tenc, mask = (torch.cat([t[B:], t[B:]]) for t in (te, tenc, mask))
    x_T = torch.randn(B, D, device="cuda", generator=g)
    noise = torch.randn(N, B, D, device="cuda", generator=g)
    mean, std = 0.1 * torch.randn(D, device="cuda", generator=g), 0.5 + torch.rand(D, device="cuda", generator=g)
    s = sample_prior22(m, te, tenc, mask, N, guidance, mean, std, x_T, noise)
    rows = slice(None) if guidance > 1.0 else slice(B, None)

    def fn(xx, tt):
        return p22.diffusers_prior_forward(dsd, cfg, xx, tt, te[rows], tenc[rows], mask[rows])
    with torch.no_grad():
        ref = p22.unclip_sample(fn, x_T, noise, N, guidance, mean, std).float()
    rel = ((s - ref).norm() / ref.norm()).item()
    print(f"tiny 2.2 prior, {N} steps, guidance {guidance}: rel-L2 {rel:.3e} against the oracle loop")
    assert rel < 3e-2, rel   # the tiny 2.1 golden's prior sampling bound (tests/test_gpu_zz_prior.py)


# ---------------------------------------------------------------------------------------------------------------------------
# full 2.2 size, synthetic weights
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def full():
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = p22.CONFIG_PRIOR22
    m, dsd = _prior_from_diffusers(cfg, seed=11, round_gemm=True)
    yield cfg, m, dsd
    del m, dsd
    torch.cuda.empty_cache()


def _dev(y, ref):
    return (y - ref).abs().max().item(), ((y - ref).norm() / ref.norm()).item()


@pytest.mark.parametrize("B,prompt_len", [(1, 12), (4, 77)])
def test_full_size_forward_fp16_calibration(full, B, prompt_len, monkeypatch):
    from kandinsky2 import ops
    cfg, m, dsd = full
    te, tenc, mask, g = _cond(cfg, B, prompt_len, seed=B)
    N = 2 * B
    x = torch.randn(N, cfg["clip_dim"], device="cuda", generator=g)
    t = torch.tensor([999.0, 500.0, 120.0, 0.0] * B, device="cuda")[:N]
    peaks, gemm_rows = [], ops.gemm_rows

    def recording_gemm_rows(*a, **kw):
        y = gemm_rows(*a, **kw)
        if kw.get("residual") is not None:
            peaks.append(y.abs().amax())
        return y

    monkeypatch.setattr(ops, "gemm_rows", recording_gemm_rows)
    y = m(x, t, text_emb=te, text_enc=tenc, mask=mask)
    monkeypatch.undo()
    assert len(peaks) == 2 * cfg["xf_layers"]
    peak = torch.stack(peaks).max().item()
    assert torch.isfinite(torch.stack(peaks)).all() and torch.isfinite(y).all(), peak
    with torch.no_grad():
        ref32 = p22.diffusers_prior_forward(dsd, cfg, x, t, te, tenc, mask)
        sd16 = {k: v.half() for k, v in dsd.items()}
        ref16 = p22.diffusers_prior_forward(sd16, cfg, x, t, te, tenc, mask, dtype=torch.float16)
        del sd16
    k_abs, k_rel = _dev(y, ref32)
    r_abs, r_rel = _dev(ref16, ref32)
    print(f"2.2 prior full size B={B}: residual stream peak |h| {peak:.1f}; k2 vs fp32 max-abs {k_abs:.3e} rel-L2 {k_rel:.3e} | "
          f"fp16 oracle vs fp32 max-abs {r_abs:.3e} rel-L2 {r_rel:.3e}")
    assert k_rel <= r_rel and k_abs <= r_abs, (k_abs, k_rel, r_abs, r_rel)
    assert k_rel < 5e-3, k_rel


@pytest.mark.parametrize("B", [1, 4])
def test_full_size_sampling(full, B):
    """25-step guided sampling (guidance 4), one graph replay per step, against the float64 UnCLIP loop over the fp32 oracle."""
    from kandinsky2.model.prior import sample_prior22
    cfg, m, dsd = full
    D = cfg["clip_dim"]
    te, tenc, mask, g = _cond(cfg, B, 12, seed=20 + B)
    x_T = torch.randn(B, D, device="cuda", generator=g)
    noise = torch.randn(25, B, D, device="cuda", generator=g)
    mean, std = 0.1 * torch.randn(D, device="cuda", generator=g), 0.5 + torch.rand(D, device="cuda", generator=g)
    s = sample_prior22(m, te, tenc, mask, 25, 4.0, mean, std, x_T, noise)
    with torch.no_grad():
        ref = p22.unclip_sample(lambda xx, tt: p22.diffusers_prior_forward(dsd, cfg, xx, tt, te, tenc, mask), x_T, noise, 25, 4.0,
                                mean, std).float()
    err, rel = _dev(s, ref)
    print(f"2.2 prior full size B={B}, 25 steps, guidance 4: rel-L2 {rel:.3e} max-abs {err:.3e}")
    assert torch.isfinite(s).all() and rel < 1e-2, rel


# ---------------------------------------------------------------------------------------------------------------------------
# PriorEmbedder22 behind Kandinsky2_2
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def embedder():
    from kandinsky2.model.prior import PriorEmbedder22
    from oracle import synth
    cfg = dict(text_ctx=8, xf_width=128, xf_layers=2, xf_heads=2, xf_final_ln=True, xf_padding=False, clip_dim=1280,
               clip_xf_width=1280)
    dsd = synth.synth_state_dict(p22.diffusers_prior_spec(cfg), seed=13)
    calls = []

    def clip_text(prompts):   # deterministic stand-in for the tokenizer + CLIP-bigG text tower
        calls.append(list(prompts))
        outs = []
        for p in prompts:
            g = torch.Generator().manual_seed(len(p) + 17 * sum(map(ord, p)))
            outs.append((torch.randn(1280, generator=g), torch.randn(8, 1280, generator=g), torch.arange(8) < 2 + len(p) % 6))
        return tuple(torch.stack(t) for t in zip(*outs))

    clip_image = lambda img: torch.full((1, 1280), 0.25)   # noqa: E731
    emb = PriorEmbedder22.from_diffusers(dsd, clip_text, clip_image=clip_image, zero_image_emb=torch.full((1280,), -0.5))
    return emb, calls


def test_embedder_rows_steps_and_guidance(embedder, monkeypatch):
    from kandinsky2.model import prior as prior_mod
    emb, calls = embedder
    replays = []
    run = prior_mod._PriorStepPlan.run
    monkeypatch.setattr(prior_mod._PriorStepPlan, "run", lambda self, g: (replays.append(g), run(self, g))[1])
    calls.clear()
    a = emb.image_emb("a red cat", 2, prior_steps=4, prior_guidance_scale=4, negative_prior_prompt="low quality")
    assert calls == [["low quality", "low quality", "a red cat", "a red cat"]]
    assert a.shape == (2, 1280) and torch.isfinite(a).all() and not torch.equal(a[0], a[1])   # each row its own sample
    n0 = len(replays)
    b = emb.image_emb("a red cat", 2, prior_steps=4, prior_guidance_scale=4, negative_prior_prompt="low quality")
    assert torch.equal(a, b) and len(replays) - n0 == 4
    n0 = len(replays)
    c = emb.image_emb("a red cat", 2, prior_steps=7, prior_guidance_scale=4, negative_prior_prompt="low quality")
    assert len(replays) - n0 == 7 and not torch.equal(a, c)
    assert not torch.equal(a, emb.image_emb("a red cat", 2, prior_steps=4, prior_guidance_scale=6,
                                            negative_prior_prompt="low quality"))
    # guidance <= 1: no CFG, the text tower sees the prompt alone, and the result does not depend on the scale
    calls.clear()
    u1 = emb.image_emb("a red cat", 2, prior_steps=4, prior_guidance_scale=1.0, negative_prior_prompt="low quality")
    u2 = emb.image_emb("a red cat", 2, prior_steps=4, prior_guidance_scale=0.5, negative_prior_prompt="ignored")
    assert calls == [["a red cat", "a red cat"]] * 2
    assert torch.equal(u1, u2) and not torch.equal(u1, a)


def test_kandinsky22_methods_run_the_prior(embedder):
    from kandinsky2 import get_kandinsky2
    from tests.test_gpu_movq_sampler import _tiny_overrides
    emb, calls = embedder
    seen = []

    class Spy(type(emb)):
        def image_emb(self, prompt, batch_size, **kw):
            seen.append((prompt, batch_size, kw))
            return super().image_emb(prompt, batch_size, **kw)

    spy = Spy.__new__(Spy)
    spy.__dict__.update(emb.__dict__)
    pipe = get_kandinsky2("cuda", task_type="text2img", model_version="2.2", cache_dir="/nonexistent", embedder=spy,
                          config_overrides=_tiny_overrides())
    kw = dict(batch_size=2, decoder_steps=2, h=64, w=64)
    a = pipe.generate_text2img("a red cat", prior_steps=3, prior_guidance_scale=4, negative_prior_prompt="ugly", **kw)
    assert seen == [("a red cat", 2, dict(prior_steps=3, prior_guidance_scale=4, negative_prior_prompt="ugly"))]
    b = pipe.generate_text2img("a red cat", prior_steps=3, prior_guidance_scale=4, negative_prior_prompt="ugly", **kw)
    assert all(x.tobytes() == y.tobytes() for x, y in zip(a, b))
    c = pipe.generate_text2img("a red cat", prior_steps=3, prior_guidance_scale=9, negative_prior_prompt="ugly", **kw)
    assert a[0].tobytes() != c[0].tobytes()
    # decoder negative: the prior's embedding of negative_decoder_prompt guided against "", not zero_image_emb
    seen.clear()
    pipe.generate_text2img("a red cat", prior_steps=2, negative_decoder_prompt="blurry", **kw)
    assert seen[1] == ("blurry", 2, dict(prior_steps=2, prior_guidance_scale=4, negative_prior_prompt=""))
    seen.clear()
    from PIL import Image
    mixed = pipe.mix_images(["a cat", Image.new("RGB", (8, 8))], [0.3, 0.7], prior_steps=2, negative_prior_prompt="ugly",
                            **kw)
    assert [s[0] for s in seen] == ["a cat"] and seen[0][2]["negative_prior_prompt"] == "ugly"
    lat = torch.randn(1, 4, 8, 8, generator=torch.Generator().manual_seed(0))
    i2i = pipe.generate_img2img("a hat", lat, strength=0.5, prior_steps=2, negative_prior_prompt="ugly", **kw)
    assert len(a) == len(mixed) == len(i2i) == 2
    mask = torch.ones(64, 64)
    mask[:, 40:] = 0
    inp = get_kandinsky2("cuda", task_type="inpainting", model_version="2.2", cache_dir="/nonexistent", embedder=spy,
                         config_overrides=_tiny_overrides())
    assert len(inp.generate_inpainting("a hat", lat, mask.numpy(), prior_steps=2, **kw)) == 2
    cn = get_kandinsky2("cuda", task_type="controlnet", model_version="2.2", cache_dir="/nonexistent", embedder=spy,
                        config_overrides=_tiny_overrides())
    hint = torch.rand(1, 3, 64, 64, generator=torch.Generator().manual_seed(3))
    assert len(cn.generate_controlnet("a red cat", hint, prior_steps=2, **kw)) == 2
