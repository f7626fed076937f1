"""GPU: LoRA adapters merged into the Kandinsky 2.2 prior's packed attention weights -- the captured-graph lifecycle (load /
reload / unload / re-pack without rebuilding a step plan), the adapted prior against the fp32 oracle with the adapter run
unfused (tests/prior_lora_oracle.py) at the tiny and the full 2.2 size, and the notebook's flow through Kandinsky2_2 with a
decoder and a prior adapter.

The full-size test is calibrated as tests/test_gpu_zz_prior22.py's is: the product must be at least as close to the fp32
oracle as the oracle in fp16 is, in max-abs AND relative L2, with the GEMM weights as the product stores them (fp16); against
the oracle with the adapter unfused, the rounding of the merged weights to fp16 is accounted for (see that test)."""
import pytest
import torch

from tests import prior22_oracle as p22
from tests import prior_lora_oracle as plo
from tests.test_gpu_zz_prior22 import _cond, _dev, _prior_from_diffusers

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def tiny():
    from kandinsky2 import launch_plan
    old = launch_plan.TUNE_SMALL_M
    launch_plan.TUNE_SMALL_M = 0     # bit-identical GEMM configurations only, so fresh and reused models compare bit for bit
    torch.backends.cuda.matmul.allow_tf32 = False
    cfg = p22.CONFIG_PRIOR22_TINY
    yield cfg
    launch_plan.TUNE_SMALL_M = old


def _run(m, cfg, B, seed, steps=5):
    """(sample_prior22 output through the step graph, the eager forward on one noisy input) for fixed conditioning."""
    from kandinsky2.model.prior import sample_prior22
    D = cfg["clip_dim"]
    te, tenc, mask, g = _cond(cfg, B, 4, seed=seed)
    x_T = torch.randn(B, D, device="cuda", generator=g)
    noise = torch.randn(steps, B, D, device="cuda", generator=g)
    mean, std = 0.1 * torch.randn(D, device="cuda", generator=g), 0.5 + torch.rand(D, device="cuda", generator=g)
    s = sample_prior22(m, te, tenc, mask, steps, 4.0, mean, std, x_T, noise).clone()
    y = m(torch.cat([x_T, x_T]), torch.full((2 * B,), 500.0, device="cuda"), text_emb=te, text_enc=tenc, mask=mask)
    return s, y


def test_lora_graph_lifecycle(tiny):
    """load / reload / unload on a prior whose step graph is already captured: the same plan objects and graphs replay with
    the packed weights at the same addresses and give exactly what a freshly built prior with the adapter gives; a q/k/v-only
    and a to_out-only adapter each change the output; a reload at scale 0.5 equals a fresh load; scale 0 is the base bit for
    bit; unload gives the pre-load output bit for bit with state_dict() unchanged; finalize() (re-packing) re-applies the
    adapter."""
    cfg = tiny
    B = 2
    lora = plo.synth_prior_lora(cfg, rank=4, seed=3)
    qkv_only = plo.synth_prior_lora(cfg, rank=4, seed=4, projections=("to_q", "to_k", "to_v"))
    out_only = plo.synth_prior_lora(cfg, rank=4, seed=5, projections=("to_out",))

    m, _ = _prior_from_diffusers(cfg, seed=5)
    s0, y0 = _run(m, cfg, B, seed=1)
    s0b, y0b = _run(m, cfg, B, seed=1)
    assert torch.equal(s0, s0b) and torch.equal(y0, y0b)
    plans = dict(m._step_plans)
    graphs = {k: p.graph for k, p in plans.items()}
    assert list(plans) == [B] and all(gr is not None for gr in graphs.values())
    ptrs = [(L["attn.qkv"][0].data_ptr(), L["attn.proj"][0].data_ptr()) for L in m._packed["layers"]]
    packed0 = [(L["attn.qkv"][0].clone(), L["attn.proj"][0].clone()) for L in m._packed["layers"]]
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}

    def same_plans():
        assert m._step_plans.keys() == plans.keys() and all(m._step_plans[k] is plans[k] for k in plans)
        assert all(m._step_plans[k].graph is graphs[k] for k in plans)
        assert [(L["attn.qkv"][0].data_ptr(), L["attn.proj"][0].data_ptr()) for L in m._packed["layers"]] == ptrs

    def fresh(adapter, scale):
        f, _ = _prior_from_diffusers(cfg, seed=5)
        f.load_lora(adapter, scale)
        return _run(f, cfg, B, seed=1)

    def same(a, b):
        return torch.equal(a[0], b[0]) and torch.equal(a[1], b[1])

    m.load_lora(lora)
    assert m.lora_scale == 1.0
    r1 = _run(m, cfg, B, seed=1)
    same_plans()
    assert not torch.equal(r1[0], s0) and not torch.equal(r1[1], y0)
    assert same(r1, fresh(lora, 1.0))

    for adapter in (qkv_only, out_only):
        m.load_lora(adapter)
        r = _run(m, cfg, B, seed=1)
        same_plans()
        assert not torch.equal(r[0], s0) and not torch.equal(r[1], y0)
        assert same(r, fresh(adapter, 1.0))

    m.load_lora(lora, scale=0.5)
    assert m.lora_scale == 0.5
    r3 = _run(m, cfg, B, seed=1)
    same_plans()
    assert same(r3, fresh(lora, 0.5)) and not torch.equal(r3[0], r1[0])

    m.load_lora(lora, scale=0.0)
    same_plans()
    assert all(torch.equal(L["attn.qkv"][0].view(torch.int16), q.view(torch.int16)) and
               torch.equal(L["attn.proj"][0].view(torch.int16), p.view(torch.int16))
               for L, (q, p) in zip(m._packed["layers"], packed0))
    assert same(_run(m, cfg, B, seed=1), (s0, y0))

    m.unload_lora()
    assert m.lora_scale is None and m._lora_base is None
    r4 = _run(m, cfg, B, seed=1)
    same_plans()
    assert same(r4, (s0, y0))
    assert all(torch.equal(v, sd0[k]) for k, v in m.state_dict().items())

    m.load_lora(lora)
    m.finalize()          # re-packs the weights: the adapter is merged again into the new packing
    assert m._step_plans == {} and m.lora_scale == 1.0
    assert same(_run(m, cfg, B, seed=1), r1)
    assert all(torch.equal(v, sd0[k]) for k, v in m.state_dict().items())


@pytest.mark.parametrize("scale", [1.0, 0.5])
def test_tiny_forward_vs_oracle(tiny, scale):
    """The adapted forward against the fp32 diffusers-form oracle with the adapter unfused: the tiny prior's forward bound
    (tests/test_gpu_zz_prior.py), while the adapter moves the oracle's output by far more."""
    cfg = tiny
    m, dsd = _prior_from_diffusers(cfg, seed=7)
    lora = plo.synth_prior_lora(cfg, rank=8, seed=8)
    m.load_lora(lora, scale)
    B = 3
    te, tenc, mask, g = _cond(cfg, B, 3, seed=9)
    x = torch.randn(2 * B, cfg["clip_dim"], device="cuda", generator=g)
    t = torch.tensor([999.0, 700.0, 420.0, 120.0, 42.0, 0.0], device="cuda")
    y = m(x, t, text_emb=te, text_enc=tenc, mask=mask)
    with torch.no_grad():
        ref = plo.lora_prior_forward(dsd, cfg, lora, scale, x, t, te, tenc, mask)
        plain = p22.diffusers_prior_forward(dsd, cfg, x, t, te, tenc, mask)
    err, rel = _dev(y, ref)
    moved = _dev(plain, ref)[1]
    print(f"tiny 2.2 prior + LoRA (scale {scale}) forward: rel-L2 {rel:.3e} max-abs {err:.3e}; the adapter moves it {moved:.3e}")
    assert rel < 1e-2, rel
    assert moved > 10 * rel, (moved, rel)


@pytest.mark.parametrize("B", [1, 3])
def test_tiny_sampling_vs_oracle_unclip_loop(tiny, B):
    """25-step guided sampling (guidance 4) of the adapted prior, one graph replay per step, against the float64 UnCLIP loop
    over the fp32 oracle with the adapter unfused: the tiny prior's sampling bound (tests/test_gpu_zz_prior22.py)."""
    from kandinsky2.model.prior import sample_prior22
    cfg = tiny
    m, dsd = _prior_from_diffusers(cfg, seed=10)
    lora = plo.synth_prior_lora(cfg, rank=4, seed=11)
    m.load_lora(lora)
    N, D = 25, cfg["clip_dim"]
    te, tenc, mask, g = _cond(cfg, B, 4, seed=12 + B)
    x_T = torch.randn(B, D, device="cuda", generator=g)
    noise = torch.randn(N, B, D, device="cuda", generator=g)
    mean, std = 0.1 * torch.randn(D, device="cuda", generator=g), 0.5 + torch.rand(D, device="cuda", generator=g)
    s = sample_prior22(m, te, tenc, mask, N, 4.0, mean, std, x_T, noise)
    with torch.no_grad():
        ref = p22.unclip_sample(lambda xx, tt: plo.lora_prior_forward(dsd, cfg, lora, 1.0, xx, tt, te, tenc, mask), x_T, noise,
                                N, 4.0, mean, std).float()
    err, rel = _dev(s, ref)
    print(f"tiny 2.2 prior + LoRA, B={B}, 25 steps, guidance 4: rel-L2 {rel:.3e} max-abs {err:.3e}")
    assert torch.isfinite(s).all() and rel < 3e-2, rel


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


def _stored(m, dsd):
    """dsd with the attention weights the prior's packed attn.qkv / attn.proj hold now (as fp32, diffusers names)."""
    from kandinsky2.checkpoints import unpack_heads
    out = dict(dsd)
    for i, L in enumerate(m._packed["layers"]):
        p = f"transformer_blocks.{i}.attn1."
        for c, w in zip("qkv", unpack_heads(L["attn.qkv"][0], 3)):
            out[f"{p}to_{c}.weight"] = w.float()
        out[p + "to_out.0.weight"] = L["attn.proj"][0].float()
    return out


@pytest.mark.parametrize("rank", [4, 64])
@pytest.mark.parametrize("B,prompt_len", [(1, 12), (4, 77)])
def test_full_size_forward_fp16_calibration(full, rank, B, prompt_len):
    """Full 2.2 size with a rank-4 / rank-64 adapter whose every delta is about 10 % of its weight (Frobenius norms).

    The merge stores fp16(W + delta W): one rounding of each attention weight that an fp16 model running the adapter unfused
    (base weights exact, LoRAAttnProcessor's branch added to the projections' outputs) does not make.  So the error splits in
    two, and each part is held to the oracle's fp16 mode:
      * computation, the rule of tests/test_gpu_zz_prior22.py on the weights as the product stores them: against the fp32
        oracle on the merged weights, no worse than that oracle in fp16 on them, in max-abs and relative L2;
      * against the fp32 oracle with the adapter unfused: relative L2 no worse than that oracle in fp16 (weights and factors
        in fp16, the processor's arithmetic in fp16), and max-abs no worse than its max-abs plus what the stored weights'
        rounding alone moves the fp32 oracle (measured here, not assumed).
    The shared prior is restored afterwards."""
    cfg, m, dsd = full
    lora = plo.synth_prior_lora(cfg, rank=rank, seed=rank, gain=0.1)
    ratios = []
    for key, down in lora.items():
        if key.endswith("down.weight"):
            pre, proj = key.split(".processor.")[0], key.split(".processor.")[1].split("_lora.")[0]
            w = dsd[f"{pre}.{'to_out.0' if proj == 'to_out' else proj}.weight"]
            ratios.append(((lora[key[:-len("down.weight")] + "up.weight"].cuda() @ down.cuda()).norm() / w.norm()).item())
    assert 0.08 < min(ratios) and max(ratios) < 0.12, (min(ratios), max(ratios))
    te, tenc, mask, g = _cond(cfg, B, prompt_len, seed=B)
    N = 2 * B
    x = torch.randn(N, cfg["clip_dim"], device="cuda", generator=g)
    t = torch.tensor([999.0, 500.0, 120.0, 0.0] * B, device="cuda")[:N]
    try:
        m.load_lora(lora)
        y = m(x, t, text_emb=te, text_enc=tenc, mask=mask)
        stored = _stored(m, dsd)
    finally:
        m.unload_lora()
    with torch.no_grad():
        ref32 = plo.lora_prior_forward(dsd, cfg, lora, 1.0, x, t, te, tenc, mask)
        sd16 = {k: v.half() for k, v in dsd.items()}
        ref16 = plo.lora_prior_forward(sd16, cfg, lora, 1.0, x, t, te, tenc, mask, dtype=torch.float16)
        plain = p22.diffusers_prior_forward(dsd, cfg, x, t, te, tenc, mask)
        st32 = p22.diffusers_prior_forward(stored, cfg, x, t, te, tenc, mask)
        sd16 = {k: v.half() for k, v in stored.items()}
        st16 = p22.diffusers_prior_forward(sd16, cfg, x, t, te, tenc, mask, dtype=torch.float16)
        del sd16, stored
    c_abs, c_rel = _dev(y, st32)
    s_abs, s_rel = _dev(st16, st32)
    k_abs, k_rel = _dev(y, ref32)
    r_abs, r_rel = _dev(ref16, ref32)
    w_abs = _dev(st32, ref32)[0]
    moved = _dev(plain, ref32)[1]
    print(f"2.2 prior full size + rank-{rank} LoRA, B={B}: stored weights: k2 vs fp32 max-abs {c_abs:.3e} rel-L2 {c_rel:.3e} | "
          f"fp16 oracle max-abs {s_abs:.3e} rel-L2 {s_rel:.3e}; unfused: k2 vs fp32 max-abs {k_abs:.3e} rel-L2 {k_rel:.3e} | "
          f"fp16 oracle max-abs {r_abs:.3e} rel-L2 {r_rel:.3e} | weight rounding alone max-abs {w_abs:.3e} | "
          f"the adapter moves the output {moved:.3e}")
    assert torch.isfinite(y).all()
    assert c_rel <= s_rel and c_abs <= s_abs, (c_abs, c_rel, s_abs, s_rel)
    assert k_rel <= r_rel and k_abs <= r_abs + w_abs, (k_abs, k_rel, r_abs, r_rel, w_abs)
    assert moved > 10 * k_rel, (moved, k_rel)
    assert m.lora_scale is None and m._lora_base is None


# ---------------------------------------------------------------------------------------------------------------------------
# the notebook's cell 19 flow: a prior adapter and a decoder adapter through Kandinsky2_2
# ---------------------------------------------------------------------------------------------------------------------------
def test_pipeline_with_prior_and_decoder_adapters():
    """Kandinsky2_2 with a decoder adapter (Text2ImUNet.load_lora) and a PriorEmbedder22 whose prior carries a prior adapter
    (embedder.prior.load_lora): generate_text2img equals the embeddings and the decode composed by hand with the same adapters,
    and differs from the run after the prior adapter is unloaded (decoder adapter still loaded)."""
    import numpy as np
    from kandinsky2 import get_kandinsky2
    from kandinsky2.model.prior import PriorEmbedder22
    from oracle import synth
    from tests import lora_oracle as lo
    from tests.test_gpu_movq_sampler import _tiny_overrides
    cfg = dict(text_ctx=8, xf_width=128, xf_layers=2, xf_heads=2, xf_final_ln=True, xf_padding=False, clip_dim=1280,
               clip_xf_width=1280)
    dsd = synth.synth_state_dict(p22.diffusers_prior_spec(cfg), seed=21)

    def clip_text(prompts):   # deterministic stand-in for the tokenizer + CLIP-bigG text tower
        outs = []
        for p in prompts:
            g = torch.Generator().manual_seed(len(p) + 17 * sum(map(ord, p)))
            outs.append((torch.randn(1280, generator=g), torch.randn(8, 1280, generator=g), torch.arange(8) < 2 + len(p) % 6))
        return tuple(torch.stack(t) for t in zip(*outs))

    emb = PriorEmbedder22.from_diffusers(dsd, clip_text, zero_image_emb=torch.full((1280,), -0.5))
    pipe = get_kandinsky2("cuda", task_type="text2img", model_version="2.2", cache_dir="/nonexistent", embedder=emb,
                          config_overrides=_tiny_overrides())
    m = pipe.model
    dec_cfg = dict(in_channels=m.in_channels, model_channels=m.model_channels, channel_mult=m.channel_mult,
                   num_res_blocks=m.num_res_blocks, attention_ds=m.attention_resolutions, model_dim=m.model_dim)
    kw = dict(prior_steps=4, prior_guidance_scale=4, negative_prior_prompt="ugly")
    base_emb = emb.image_emb("a red cat", 2, **kw)

    m.load_lora(lo.synth_lora(dec_cfg, rank=4, seed=22, gain=1.0))
    emb.prior.load_lora(plo.synth_prior_lora(cfg, rank=4, seed=23))
    run = lambda: np.stack([np.asarray(im) for im in pipe.generate_text2img("a red cat", batch_size=2, decoder_steps=3, h=64,  # noqa: E731
                                                                            w=64, **kw)])
    a = run()
    pos = emb.image_emb("a red cat", 2, **kw)
    assert not torch.equal(pos, base_emb)
    by_hand = pipe._decode_loop(pos, emb.zero_image_emb(2), 2, 3, 4, 64, 64)
    assert np.array_equal(a, np.stack([np.asarray(im) for im in by_hand]))

    emb.prior.unload_lora()
    assert torch.equal(emb.image_emb("a red cat", 2, **kw), base_emb)
    b = run()
    assert not np.array_equal(a, b)
    m.unload_lora()
