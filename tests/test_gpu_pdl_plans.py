"""GPU: every launch plan with programmatic dependent launch (PDL, tuning key 4) on, bit for bit against the serialised run.

The benchmark and the pipelines run with PDL on: kernel N of a stream may start while kernel N-1 drains, and each kernel's
griddepcontrol.wait (pdl_wait) is what orders it after its predecessor.  The UNet plan also forks: the time embedding and
the 36 FiLM projections (one linear over a 215 MB weight) run on a side stream next to the stem, and the first ResBlock joins
that branch right before its out-norm, which reads the FiLM rows; the up ResBlocks' skip upsampling forks and joins the same
way.  Whether that join stays a full dependency when the launch after it is a PDL launch -- in eager mode and as a
captured graph -- decides whether the out-norm may read FiLM rows that are not written yet.

Reference: the fully serialised run -- PDL off, launch_plan.FORK off (the branch runs in line), eager.
Candidate: PDL on, FORK on, eager and as one CUDA graph, with the fork DELAYED and its outputs POISONED: the first launch
of every fork waits DELAY_CYCLES on the side stream, and before every run / graph replay the buffers the branch writes (the
FiLM rows, the "xres" scratch) are NaN-filled.  A consumer that runs ahead of the branch then reads NaN on its first run,
deterministically, instead of a stale but equal value from the previous run.  Each case runs once: no repeats.
Self-check: the same harness with the first ResBlock's join left out must give non-finite output, so the harness can fail.

Plans that do not fork (MoVQ, the 2.2 prior step, the CLIP towers, XLM-R) are checked with PDL on and off, eager and as a
graph.  Tuning key 11 (GroupNorm apply grid sizing) must not change a bit.  The last test runs the benchmark's own step --
the full-size 2.2 UNet, 4 images at 96x96 latents, DDPM -- as a PDL graph against the serialised eager step."""
import gc
import os

import pytest
import torch

from tests.test_gpu_plan_poison import _fill_nan_

pytestmark = pytest.mark.gpu
ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
GOLD = os.path.join(ROOT, "tests", "golden")

# torch.cuda._sleep spins this many GPU clock cycles: 5 ms at the H100's 1.98 GHz boost clock, longer at lower clocks.  The
# main-stream work between a fork and its join (stem im2col + conv, one norm + conv at the test geometries) takes tens of
# microseconds, so the branch finishes about 100 times later than a consumer that does not wait for it would read it.
DELAY_CYCLES = 10_000_000


@pytest.fixture(autouse=True)
def _restore():
    """Tuning keys 4 and 11 back to the library defaults, every stream drained and the dropped plans freed (a plan is a
    reference cycle: its launch closures hold it), whatever the test did."""
    from kandinsky2 import launch_plan
    small_m = launch_plan.TUNE_SMALL_M
    launch_plan.TUNE_SMALL_M = 0   # bit-identical GEMM configurations only: fixed row groups, so a fixed fold decision
    try:
        yield
    finally:
        from kandinsky2 import ops
        torch.cuda.synchronize()
        ops.set_tuning(4, 0)
        ops.set_tuning(11, 0)
        launch_plan.TUNE_SMALL_M = small_m
        gc.collect()
        torch.cuda.empty_cache()


def _serial(monkeypatch):
    from kandinsky2 import launch_plan, ops
    monkeypatch.setattr(launch_plan, "FORK", False)
    ops.set_tuning(4, 0)


def _pdl(monkeypatch, delay=True):
    """PDL on, the fork on, and (delay) the first launch of every fork held back DELAY_CYCLES on the side stream."""
    from kandinsky2 import launch_plan, ops
    from kandinsky2.launch_plan import LaunchPlan
    monkeypatch.setattr(launch_plan, "FORK", True)
    ops.set_tuning(4, 1)
    if not delay:
        return
    side = LaunchPlan._side

    def _side(plan, fn, kind="misc", flops=0):
        if not plan._side_open:   # opens a fork: this launch is the first on the side stream
            inner = fn

            def fn():
                torch.cuda._sleep(DELAY_CYCLES)
                inner()
        return side(plan, fn, kind, flops)
    monkeypatch.setattr(LaunchPlan, "_side", _side)


def _poison_branch(plan):
    """NaN into what the forked branch writes: the FiLM rows and the up ResBlocks' upsampled skip."""
    _fill_nan_(plan.film)
    for key, t in plan._scratch.items():
        if key[0] == "xres":
            _fill_nan_(t)


def _same(a, b, what):
    assert torch.isfinite(a.float()).all(), f"{what}: {int((~torch.isfinite(a.float())).sum())} non-finite of {a.numel()}"
    assert torch.equal(a, b), f"{what}: max abs difference {(a.float() - b.float()).abs().max().item():.3e}"


# ---------------------------------------------------------------------------------------------------------------------------
# UNet forward
# ---------------------------------------------------------------------------------------------------------------------------
FOLDED, UNFOLDED = (16, 16), (48, 64)   # level-0 row groups per image: 2 (k2_gn_apply_fold) and 24 (> FOLD_MAX_RG = 18)


def _hint_build(cfg, sd):
    from kandinsky2.model.unet import Text2ImUNet
    m = Text2ImUNet(model_dim=cfg["model_dim"], image_encoder_in_dim=cfg["image_encoder_in_dim"],
                    num_image_embs=cfg["num_image_embs"], pooling_type="from_model", in_channels=cfg["in_channels"],
                    model_channels=cfg["model_channels"], out_channels=cfg["out_channels"],
                    num_res_blocks=cfg["num_res_blocks"], attention_resolutions=tuple(cfg["attention_ds"]),
                    channel_mult=cfg["channel_mult"], use_fp16=True, num_head_channels=64, use_scale_shift_norm=True,
                    resblock_updown=True, cond_version="2.2", hint_channels=4)
    m.load_state_dict(sd, strict=True)
    return m.to("cuda")


def _unet_case(variant, hw):
    """-> (model, inputs on the GPU) of a tiny UNet at latent size hw: the golden fixtures' weights and conditioning."""
    from oracle import controlnet_oracle as co, synth, unet_oracle as uo
    from tests.test_gpu_unet import _build
    g = torch.Generator().manual_seed(5)
    if variant in ("2.1", "inpaint"):
        fx = torch.load(os.path.join(GOLD, "unet_tiny.pt" if variant == "2.1" else "unet_tiny_inpaint.pt"))
        cfg, inp = fx["cfg"], dict(fx["inputs"])
        m = _build(cfg, synth.synth_state_dict(uo.unet_param_spec(cfg), seed=fx["weight_seed"]))
    else:
        cfg = dict(uo.CONFIG_TINY, cond="2.2", in_channels=8 if variant == "hint" else 4)
        inp = dict(x=torch.randn(2, 4, *hw, generator=g), t=torch.tensor([981.0, 40.0]),
                   image_emb=torch.randn(2, cfg["image_encoder_in_dim"], generator=g))
        if variant == "hint":
            inp["hint"] = torch.rand(2, 3, 8 * hw[0], 8 * hw[1], generator=g)
            m = _hint_build(cfg, synth.synth_state_dict(co.param_spec(cfg), seed=7))
        else:
            m = _build(cfg, synth.synth_state_dict(uo.unet_param_spec(cfg), seed=5))
    if tuple(inp["x"].shape[2:]) != hw:
        inp["x"] = torch.randn(2, 4, *hw, generator=g)
        if "inpaint_mask" in inp:
            inp["inpaint_image"] = torch.randn(2, 4, *hw, generator=g)
            inp["inpaint_mask"] = (torch.rand(2, 1, *hw, generator=g) > 0.5).float()
    return m, {k: v.cuda() for k, v in inp.items()}


def _unet_plan(m, inp):
    """The model's plan for inp (built on first use, i.e. traced eagerly once), bound and loaded as forward() does it."""
    keys = ("full_emb", "pooled_emb", "image_emb", "hint")
    cond = m.get_text_emb(**{k: inp.get(k) for k in keys})
    x = inp["x"]
    plan = m._plan(x.shape[0], x.shape[2], x.shape[3], cond["xf_out"].shape[1])
    plan.bind(cond)
    plan.x_in.copy_(x)
    plan.t_in.copy_(inp["t"])
    if m._inpainting:
        plan.img_in.copy_(inp["inpaint_image"])
        plan.mask_in.copy_(inp["inpaint_mask"])
    return plan


def _unet_ref(m, inp, monkeypatch):
    _serial(monkeypatch)
    m._plans = {}
    plan = _unet_plan(m, inp)
    plan.run(False)
    out = plan.out.clone()
    m._plans = {}
    return out


def _unet_pdl(m, inp, graph):
    """One PDL run of a fresh plan (delayed, poisoned fork already patched in) -> (output, kind of the launch after the first
    join).  Graph: captured first (the capture's warm-up and first replay are discarded), then poisoned and replayed."""
    m._plans = {}
    plan = _unet_plan(m, inp)
    if graph:
        plan.run(True)
    _poison_branch(plan)
    plan.run(graph)
    kinds = [k for _, k, _ in plan.steps]
    return plan.out.clone(), kinds[kinds.index("join") + 1]


@pytest.mark.parametrize("hw,after_join", [(FOLDED, "gn_apply"), (UNFOLDED, "gn_finalize")], ids=["folded", "unfolded"])
@pytest.mark.parametrize("variant", ["2.1", "2.2", "inpaint", "hint"])
def test_unet_pdl_delayed_fork(variant, hw, after_join, monkeypatch):
    """folded: the launch after the join is the out-norm itself (k2_gn_apply_fold, which reads the FiLM rows);
    unfolded: it is k2_gn_finalize, and the FiLM-reading k2_gn_apply comes one launch later."""
    m, inp = _unet_case(variant, hw)
    ref = _unet_ref(m, inp, monkeypatch)
    _pdl(monkeypatch)
    for graph in (False, True):
        out, nxt = _unet_pdl(m, inp, graph)
        assert nxt == after_join, f"the launch after the first join is {nxt}, not {after_join}: the coverage moved"
        _same(out, ref, f"{variant} {hw} {'graph' if graph else 'eager'}")
    torch.cuda.synchronize()


@pytest.mark.parametrize("hw", [FOLDED, UNFOLDED], ids=["folded", "unfolded"])
def test_harness_catches_a_missing_join(hw, monkeypatch):
    """The same harness with the first ResBlock's join left out: its out-norm no longer waits for the delayed FiLM rows, reads
    the NaN fill, and the output is non-finite -- a missing dependency is caught on its first run.  Eager only (capture
    refuses a stream that is not joined back)."""
    from kandinsky2.launch_plan import LaunchPlan
    m, inp = _unet_case("2.1", hw)
    _pdl(monkeypatch)
    join = LaunchPlan._join

    def _join(plan):
        if plan._side_open and not getattr(plan, "_skipped_join", False):
            plan._skipped_join = True   # the first join of the plan: the first ResBlock's, before its out-norm
            return
        return join(plan)
    monkeypatch.setattr(LaunchPlan, "_join", _join)
    m._plans = {}
    plan = _unet_plan(m, inp)
    _poison_branch(plan)
    plan.run(False)
    out = plan.out.clone()
    torch.cuda.synchronize()
    m._plans = {}
    assert not torch.isfinite(out).all(), "the harness did not see the missing join"


def test_gn_apply_grid_sizing_key11_bit_identical(monkeypatch):
    """Tuning key 11 sizes the GroupNorm apply grids (0 = the kernels' occupancy); the values 0, 1 and 4 change how the
    pixels are split into blocks, not a bit of the result (PDL graph, delayed fork, against the serialised run)."""
    from kandinsky2 import ops
    m, inp = _unet_case("2.2", UNFOLDED)
    ref = _unet_ref(m, inp, monkeypatch)
    _pdl(monkeypatch)
    for bps in (0, 1, 4):
        ops.set_tuning(11, bps)
        out, _ = _unet_pdl(m, inp, graph=True)
        _same(out, ref, f"key 11 = {bps}")


# ---------------------------------------------------------------------------------------------------------------------------
# FusedStep: step_begin + UNet plan + sampler step + step_end as one graph per step
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def mid22():
    """4-level 2.2 UNet at 128 base channels (test_unet_mid_vs_oracle's); at 32x32 latents and 4 UNet rows the first out-norm
    is folded (8 row groups per image)."""
    from oracle import synth, unet_oracle as uo
    from tests.test_gpu_unet import _build
    cfg = dict(uo.CONFIG_2_2, model_channels=128, num_res_blocks=2, model_dim=256)
    m = _build(cfg, synth.synth_state_dict(uo.unet_param_spec(cfg), seed=3))
    yield m
    del m
    gc.collect()
    torch.cuda.empty_cache()


def _schedule(kind, n):
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule, UniPCSchedule, create_ddpm_v22
    ddpm = create_ddpm_v22(n)
    if kind == "ddpm":
        return ddpm
    if kind == "unipc":
        return UniPCSchedule(ddpm.base_alphas_cumprod, n)
    return DPMSolverSchedule(ddpm.base_alphas_cumprod, n, sde=kind == "dpmpp_2m_sde")


def _fused(m, kind, B, H, W, kw, extra, graph, after_join="gn_apply", threshold_mode=0, cond_first=False, n=3):
    """n scheduled steps with per-step noise from a fixed x_T -> the latent.  Eager: FusedStep._launch_step (every launch
    issued one by one).  Graph: advance(), the step graph captured first and the schedule staged again, then the branch
    buffers NaN-filled before every replay; after_join names the launch that must follow the first join."""
    from kandinsky2.model.gaussian_diffusion import FusedStep
    m._plans = {}
    sched = _schedule(kind, n)
    coef, ts = sched._tables(torch.device("cuda"))
    idx = torch.arange(n - 1, -1, -1, device="cuda")
    g = torch.Generator(device="cuda").manual_seed(17)
    x_T = torch.randn(B, 4, H, W, device="cuda", generator=g)
    noise = torch.randn(n, B, 4, H, W, device="cuda", generator=g)
    step = FusedStep(m, B, H, W, kw, 4.0, cond_first, 2.0, threshold_mode, step_kind=sched.step_kind, **extra)
    step.set_schedule(ts[idx], coef[idx], noise)
    x = x_T.clone()
    if not graph:
        for _ in range(n):
            step._launch_step(x, step.st["noise_seq"])
        return x
    kinds = [k for _, k, _ in step.plan.steps]
    assert kinds[kinds.index("join") + 1] == after_join, f"the launch after the first join is not {after_join}"
    step.advance(x_T.clone())
    step.set_schedule(ts[idx], coef[idx], noise)
    for _ in range(n):
        _poison_branch(step.plan)
        step.advance(x)
    return x


def _fused_check(m, kind, B, H, W, kw, extra, monkeypatch, delay=True, **kws):
    """The serialised eager steps against the PDL step graph (folded first out-norm unless after_join says otherwise)."""
    m.del_cache()
    _serial(monkeypatch)
    ref = _fused(m, kind, B, H, W, kw, extra, graph=False, **kws)
    _pdl(monkeypatch, delay)
    out = _fused(m, kind, B, H, W, kw, extra, graph=True, **kws)
    torch.cuda.synchronize()
    m._plans = {}
    _same(out, ref, f"FusedStep {kind}")


@pytest.mark.parametrize("kind", ["ddpm", "dpmpp_2m", "dpmpp_2m_sde", "unipc"])
def test_fused_step_pdl_graph(kind, mid22, monkeypatch):
    B, H, W = 2, 32, 32
    g = torch.Generator(device="cuda").manual_seed(3)
    kw = dict(image_emb=torch.randn(2 * B, 1280, device="cuda", generator=g))
    _fused_check(mid22, kind, B, H, W, kw, {}, monkeypatch)


def test_fused_step_pdl_graph_inpaint_22_renoise(mid22, monkeypatch):
    """Kandinsky 2.2 inpainting: the known region re-noised to the next timestep (inpaint_noise) inside the step kernel."""
    B, H, W = 2, 32, 32
    g = torch.Generator(device="cuda").manual_seed(4)
    kw = dict(image_emb=torch.randn(2 * B, 1280, device="cuda", generator=g))
    init = torch.randn(B, 4, H, W, device="cuda", generator=g)
    mask = (torch.rand(B, 1, H, W, device="cuda", generator=g) > 0.5).float()
    extra = dict(inpaint_init=init, inpaint_mask=mask, inpaint_noise=torch.randn(B, 4, H, W, device="cuda", generator=g))
    _fused_check(mid22, "ddpm", B, H, W, kw, extra, monkeypatch)


def test_fused_step_pdl_graph_inpaint_21_mask(monkeypatch):
    """Kandinsky 2.1 inpainting: the 9-channel stem over [x, image * mask, mask], the known region replacing x0 in the step,
    with the 2.1 dynamic threshold (k2_sampler_x0 / percentile / post)."""
    m, inp = _unet_case("inpaint", FOLDED)
    B, (H, W) = 1, FOLDED
    kw = {k: v for k, v in inp.items() if k not in ("x", "t")}
    extra = dict(inpaint_init=inp["inpaint_image"][:B], inpaint_mask=inp["inpaint_mask"][:B])
    _fused_check(m, "ddpm", B, H, W, kw, extra, monkeypatch, threshold_mode=1, cond_first=True)


# ---------------------------------------------------------------------------------------------------------------------------
# plans that do not fork: PDL on / off x eager / graph against the serialised eager run
# ---------------------------------------------------------------------------------------------------------------------------
def _plain(run, drop, monkeypatch):
    """run(graph) -> output tensors of a plan built on first use; drop() forgets the plans."""
    from kandinsky2 import ops
    _serial(monkeypatch)
    drop()
    ref = run(False)
    for pdl, graph in ((0, True), (1, False), (1, True)):
        drop()
        ops.set_tuning(4, pdl)
        out = run(graph)
        for a, b in zip(out, ref):
            _same(a, b, f"PDL {pdl}, {'graph' if graph else 'eager'}")
    torch.cuda.synchronize()
    drop()


def _movq_plain(m, fn, x, monkeypatch, **kw):
    def run(graph):
        m.use_cuda_graph = graph
        return (getattr(m, fn)(x, **kw).clone(),)

    _plain(run, lambda: setattr(m, "_plans", {}), monkeypatch)


def test_movq_tiny_pdl(monkeypatch):
    """Golden tiny MoVQ: decode, encode and decode_to_uint8 (C = 64 attention as batched GEMMs around softmax_rows)."""
    from tests.test_gpu_plan_poison import _golden_movq
    fx, m = _golden_movq()
    z = fx["z"].cuda()
    _movq_plain(m, "decode", z, monkeypatch)
    _movq_plain(m, "encode", fx["image"].cuda(), monkeypatch)
    _movq_plain(m, "decode_to_uint8", z, monkeypatch, crop_h=14, crop_w=15)


@pytest.mark.parametrize("name,dd,hw", [
    ("mid", dict(ch=64, ch_mult=(1, 2, 4), resolution=128), 32),                           # C = 256, T = 1024
    ("fused512", dict(ch=128, ch_mult=(1, 4), resolution=64, attn_resolutions=()), 16),   # C = 512: k2_attention_d512
])
def test_movq_decode_pdl(name, dd, hw, monkeypatch):
    from oracle import movq_oracle as mo
    from tests.test_gpu_plan_poison import _movq
    m = _movq(dict(mo.DDCONFIG_2_1, **dd), 128, 9)
    z = torch.randn(2, 4, hw, hw, generator=torch.Generator().manual_seed(1)).cuda()
    _movq_plain(m, "decode", z, monkeypatch)


def test_prior22_step_pdl(monkeypatch):
    """The 2.2 prior's UnCLIP step plan (step_begin, time embedding, 2 layers, out_proj, sampler step, step_end), 3 steps."""
    from kandinsky2.model.prior import sample_prior22
    from tests import prior22_oracle as p22
    from tests.test_gpu_zz_prior22 import _cond, _prior_from_diffusers
    cfg = p22.CONFIG_PRIOR22_TINY
    m, _ = _prior_from_diffusers(cfg, seed=5)
    B, D, N = 2, cfg["clip_dim"], 3
    te, tenc, mask, g = _cond(cfg, B, 4, seed=9)
    x_T = torch.randn(B, D, device="cuda", generator=g)
    noise = torch.randn(N, B, D, device="cuda", generator=g)
    mean, std = torch.zeros(D, device="cuda"), torch.ones(D, device="cuda")

    def run(graph):
        return (sample_prior22(m, te, tenc, mask, N, 4.0, mean, std, x_T, noise, use_graph=graph).clone(),)

    _plain(run, lambda: setattr(m, "_step_plans", {}), monkeypatch)


def test_clip_text_tower_pdl(monkeypatch):
    from tests import clip_text_oracle as cto
    from tests.test_gpu_zz_clip_text import _tiny_cfg, _tokenizer, _tower
    fx = torch.load(cto.FIXTURE)
    tok = _tokenizer(fx)
    ids = tok(["a red cat", "A capybara, 4k photo", "", "a <|endoftext|> b"])["input_ids"]
    tower = _tower(_tiny_cfg(fx), 7, tok)
    _plain(lambda graph: tuple(t.clone() for t in tower.forward(ids, graph)), lambda: setattr(tower, "_plans", {}),
           monkeypatch)


def test_clip_vision_tower_pdl(monkeypatch):
    from tests import clip_vision_oracle as cvo
    from tests.test_gpu_zz_clip_vision import _tower
    pix = torch.randn(4, 3, 56, 56, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    tower = _tower(cvo.CONFIG_TINY, 7)
    _plain(lambda graph: tuple(t.clone() for t in tower.forward(pix, graph)), lambda: setattr(tower, "_plans", {}),
           monkeypatch)


def test_clip_vitl14_towers_pdl(monkeypatch):
    from tests import openai_clip_oracle as oo
    from tests.test_gpu_zz_clip_vitl14 import _towers
    geo = torch.load(oo.FIXTURE)["geo"]
    text, image = _towers(geo, 7)
    tok = oo.sample_tokens(geo, 8, n=4)
    pix = torch.randn(4, 3, 56, 56, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    for tower, x in ((text, tok), (image, pix)):
        _plain(lambda graph: tuple(t.clone() for t in tower.forward(x, graph)), lambda: setattr(tower, "_plans", {}),
               monkeypatch)


def test_xlmr_tower_pdl(monkeypatch):
    from tests import xlmr_oracle as xo
    from tests.test_gpu_zz_text_encoder import _tokenizer, _tower
    fx = torch.load(xo.FIXTURE)
    t0 = fx["towers"][0]
    e = _tokenizer(fx)(["a red cat", "A capybara, 4k photo", "", "a <mask> b <pad> c"])
    tower = _tower(t0["cfg"], t0["out_features"], 7)
    _plain(lambda graph: tuple(t.clone() for t in tower.forward(e["input_ids"], e["attention_mask"], graph)),
           lambda: setattr(tower, "_plans", {}), monkeypatch)


# ---------------------------------------------------------------------------------------------------------------------------
# Full size: the benchmark's step (1.22 B-parameter 2.2 UNet, random weights, 4 images x CFG at 96x96 latents, DDPM)
# ---------------------------------------------------------------------------------------------------------------------------
def test_full_size_bench_step_pdl_graph(monkeypatch):
    """The step graph with PDL on and the fork as the benchmark runs it (no delay) against the serialised eager step, 3
    scheduled DDPM steps.  At 96x96 the first out-norm is not folded (72 row groups per image).  About 8 GB of device
    memory."""
    from kandinsky2 import launch_plan
    from kandinsky2.model.unet import Text2ImUNet
    monkeypatch.setattr(launch_plan, "TUNE_SMALL_M", int(os.environ.get("K2_TUNE_SMALL_M", "8192")))  # the benchmark's tuning
    m = Text2ImUNet(model_dim=768, image_encoder_in_dim=1280, text_encoder_in_dim1=1024, text_encoder_in_dim2=768,
                    num_image_embs=32, pooling_type="from_model", in_channels=4, model_channels=384, out_channels=8,
                    num_res_blocks=3, attention_resolutions=(2, 4, 8), channel_mult=(1, 2, 3, 4), use_fp16=True, num_heads=1,
                    num_head_channels=64, use_scale_shift_norm=True, resblock_updown=True, cond_version="2.2", device="cuda",
                    param_dtype=torch.float16)
    m.init_synthetic_(seed=0)
    m.finalize(release_params=True)
    B, H, W = 4, 96, 96
    kw = dict(image_emb=torch.randn(2 * B, 1280, generator=torch.Generator().manual_seed(1234)).cuda())
    _fused_check(m, "ddpm", B, H, W, kw, {}, monkeypatch, delay=False, after_join="gn_finalize")
