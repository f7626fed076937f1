"""GPU: LoRA adapters merged into the packed attention weights -- the k2_lora_merge kernel against float64, the merged UNet
against the fp32 oracle with the adapter folded in the diffusers layout (tests/lora_oracle.py), the captured-graph lifecycle
(load / reload / unload without rebuilding a plan) and the 2.2 pipeline."""
import math

import pytest
import torch

from tests import lora_oracle as lo
from tests.test_gpu_unet import _build, _check, _no_tf32

pytestmark = pytest.mark.gpu


def _fp16_ulp(h):
    """Spacing of fp16 at |h| (float64), subnormals included."""
    a = h.double().abs().clamp_min(2.0 ** -14)
    return torch.exp2(torch.floor(torch.log2(a)) - 10)


def _merge_ref(base, up, down, scale):
    return (base.double() + scale * (up.double() @ down.double())).half()


def _merge_tol(out, ref, base, up, down, scale):
    """One fp16 ulp of the result plus the textbook bound of the fp32 arithmetic before the rounding (rank products summed in
    fp32, times scale, plus base: (rank + 2) u (|scale| sum_j |up_j down_j| + |base|), u = 2^-24).  The second term only
    matters where base and the delta cancel to a value far below their own magnitude (down to fp16 subnormals)."""
    rank = up.shape[1]
    fp32 = (rank + 2) * 2.0 ** -24 * (abs(scale) * (up.double().abs() @ down.double().abs()) + base.double().abs())
    return torch.maximum(_fp16_ulp(out), _fp16_ulp(ref)), fp32


@pytest.mark.parametrize("rank", [1, 4, 12, 64, 384])
def test_lora_merge_kernel(rank):
    """Every element within one fp16 ulp of the fp16 rounding of the float64 result, plus the fp32 rounding bound where base
    and the delta cancel; scale 0 returns base bit-identically; two runs are bit-identical; in place equals out of place."""
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(rank)
    rows, cols = 1536, 768
    base = torch.randn(rows, cols, device="cuda", generator=g).half()
    up = torch.randn(rows, rank, device="cuda", generator=g) / rank ** 0.5
    down = torch.randn(rank, cols, device="cuda", generator=g)
    for scale in (1.0, 0.5, -0.75):
        out = ops.lora_merge(base, up, down, scale)
        ref = _merge_ref(base, up, down, scale)
        err = (out.double() - ref.double()).abs()
        ulp, fp32 = _merge_tol(out, ref, base, up, down, scale)
        assert bool((err <= ulp + fp32).all()), (scale, (err / (ulp + fp32)).max().item())
        far = fp32 < ulp / 4   # no cancellation: one fp16 ulp
        assert bool((err[far] <= ulp[far]).all())
        assert torch.equal(out, ops.lora_merge(base, up, down, scale))
    assert torch.equal(ops.lora_merge(base, up, down, 0.0).view(torch.int16), base.view(torch.int16))
    inplace = base.clone()
    ops.lora_merge(inplace, up, down, -0.75, out=inplace)
    assert torch.equal(inplace, ops.lora_merge(base, up, down, -0.75))


@pytest.mark.parametrize("ldb,ldo", [(112, 128), (105, 103)])
def test_lora_merge_ragged(ldb, ldo):
    """Rows and columns that are not tile multiples, row strides wider than the matrix (16-byte aligned or not): the merged
    columns match float64 within the bound above, the columns beyond `cols` are untouched."""
    from kandinsky2 import ops
    g = torch.Generator(device="cuda").manual_seed(7)
    rows, cols, rank = 77, 101, 5
    base_buf = torch.randn(rows, ldb, device="cuda", generator=g).half()
    base = base_buf[:, :cols]
    up = torch.randn(rows, rank, device="cuda", generator=g)
    down = torch.randn(rank, cols, device="cuda", generator=g)
    out_buf = torch.full((rows, ldo), 7.0, device="cuda", dtype=torch.float16)
    ops.lora_merge(base, up, down, 0.5, out=out_buf[:, :cols])
    ref = _merge_ref(base, up, down, 0.5)
    got = out_buf[:, :cols]
    assert bool(((got.double() - ref.double()).abs() <= sum(_merge_tol(got, ref, base, up, down, 0.5))).all())
    assert bool((out_buf[:, cols:] == 7.0).all())
    assert torch.equal(got, ops.lora_merge(base, up, down, 0.5))


def _mid_cfg(inpaint=False):
    from oracle import unet_oracle as uo
    return dict(uo.CONFIG_2_2, model_channels=128, num_res_blocks=2, model_dim=256, inpainting=inpaint)


def _oracle_with_lora(sd, cfg, lora, scale, *args, **kw):
    """fp32 oracle forward of the k2-layout state dict `sd` with the adapter folded in the DIFFUSERS layout."""
    from kandinsky2.checkpoints import diffusers_unet_to_k2, k2_to_diffusers_unet
    from oracle import unet_oracle as uo
    geom = dict(in_channels=sd["input_blocks.0.0.weight"].shape[1], model_channels=cfg["model_channels"],
                channel_mult=tuple(cfg["channel_mult"]), num_res_blocks=cfg["num_res_blocks"],
                attention_ds=tuple(cfg["attention_ds"]))
    folded = diffusers_unet_to_k2(lo.fold_lora(k2_to_diffusers_unet(sd, **geom), lora, scale), **geom)
    with torch.no_grad():
        return uo.unet_forward(folded, cfg, *args, **kw)


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


@pytest.mark.parametrize("inpaint", [False, True])
def test_lora_mid_vs_oracle(inpaint):
    """Mid-size 2.2 decoder (and its inpainting variant) with a notebook-format adapter merged: within the per-forward bound
    of the oracle with the adapter folded in, while the adapter moves the oracle's output by >= 20x that bound."""
    from oracle import synth
    from oracle import unet_oracle as uo
    _no_tf32()
    cfg = _mid_cfg(inpaint)
    sd = synth.synth_state_dict(uo.unet_param_spec(cfg), seed=3)
    lora = lo.synth_lora(cfg, rank=8, seed=4)
    m = _build(cfg, sd)
    g = torch.Generator().manual_seed(11)
    B, H, W = 2, 32, 48
    x = torch.randn(B, 4, H, W, generator=g).cuda()
    t = torch.tensor([981.0, 40.0]).cuda()
    kw = dict(image_emb=torch.randn(B, cfg["image_encoder_in_dim"], generator=g).cuda())
    if inpaint:
        kw["inpaint_image"] = torch.randn(B, 4, H, W, generator=g).cuda()
        kw["inpaint_mask"] = (torch.rand(B, 1, H, W, generator=g) > 0.5).float().cuda()
    m.load_lora(lora, scale=0.8)
    assert m.lora_scale == 0.8
    y = m(x, t, **kw)
    sdc = {k: v.cuda() for k, v in sd.items()}
    ref = _oracle_with_lora(sdc, cfg, lora, 0.8, x, t, **kw)
    with torch.no_grad():
        plain = uo.unet_forward(sdc, cfg, x, t, **kw)
    assert _rel(plain, ref) >= 20 * 2e-3, _rel(plain, ref)
    err, rel = _check(y, ref)
    print(f"inpaint={inpaint}: merged LoRA vs oracle max abs {err:.3e} rel L2 {rel:.3e}; adapter moves output {_rel(plain, ref):.3e}")


def test_lora_through_load_attn_procs(tmp_path):
    """K2UNet2DConditionModel.load_attn_procs (diffusers' loader name) from a saved file, scale 1: the oracle within the
    bound of the fp16 front, and the same numbers as Text2ImUNet.load_lora."""
    from kandinsky2.checkpoints import k2_to_diffusers_unet
    from kandinsky2.diffusers_compat import K2UNet2DConditionModel
    from oracle import synth
    from oracle import unet_oracle as uo
    _no_tf32()
    cfg = _mid_cfg()
    sd = synth.synth_state_dict(uo.unet_param_spec(cfg), seed=6)
    lora = lo.synth_lora(cfg, rank=4, seed=9, dtype=torch.float16)
    path = tmp_path / "pytorch_model.bin"
    torch.save(lora, path)
    front = K2UNet2DConditionModel.from_state_dict(k2_to_diffusers_unet(sd, model_channels=128, num_res_blocks=2),
                                                   model_channels=128, num_res_blocks=2, model_dim=256)
    front.load_attn_procs(str(path))
    assert front.unet.lora_scale == 1.0
    g = torch.Generator().manual_seed(12)
    x = torch.randn(4, 4, 32, 32, generator=g).cuda().half()
    emb = torch.randn(4, 1280, generator=g).cuda().half()
    out = front(x, 640, added_cond_kwargs={"image_embeds": emb}).sample
    t = torch.full((4,), 640.0).cuda()
    ref = _oracle_with_lora({k: v.cuda() for k, v in sd.items()}, cfg, lora, 1.0, x.float(), t, image_emb=emb.float())
    _check(out.float(), ref, max_frac=1.5e-2, rel_l2=3e-3)
    direct = _build(cfg, sd)
    direct.load_lora(lora)
    y = direct(x, t, image_emb=emb)
    assert _rel(out.float(), y.float()) < 2e-3


def test_lora_full_size():
    """Full-size 2.2 decoder, one cfg-2 geometry (96x96 latents) at batch 2, rank-4 adapter, against the fp32 oracle on the GPU.
    The shared full-size model is restored afterwards (unload_lora)."""
    from tests import test_gpu_unet as tu
    from oracle import unet_oracle as uo
    _no_tf32()
    cfg = uo.CONFIG_2_2
    m = tu._full_model()
    lora = lo.synth_lora(cfg, rank=4, seed=2)
    g = torch.Generator(device="cuda").manual_seed(31)
    x = torch.randn(2, 4, 96, 96, device="cuda", generator=g)
    t = torch.tensor([980.0, 420.0], device="cuda")
    img = torch.randn(2, 1280, device="cuda", generator=g)
    try:
        m.load_lora(lora)
        y = m(x, t, image_emb=img)
        ref = _oracle_with_lora(tu._sd_as_stored(tu._full_sd()), cfg, lora, 1.0, x, t, image_emb=img)
        err, rel = _check(y, ref)
        print(f"full size, rank 4: max abs {err:.3e} rel L2 {rel:.3e}")
        del ref
    finally:
        m.unload_lora()
        torch.cuda.empty_cache()
    assert m.lora_scale is None and m._lora_base is None


def _tiny():
    from oracle import synth
    from oracle import unet_oracle as uo
    cfg = dict(uo.CONFIG_TINY, image_encoder_in_dim=1280, num_image_embs=4, cond="2.2")
    return cfg, synth.synth_state_dict(uo.unet_param_spec(cfg), seed=8)


def test_lora_graph_lifecycle():
    """load / reload / unload on a model whose plan is already captured as a CUDA graph: the same plan objects replay with the
    packed weights at the same addresses and give exactly what a freshly built model with the adapter gives; an adapter of
    only the encoder K/V projections changes the output (the cached conditioning was refreshed); a reload at another scale
    equals a fresh load; unload gives the pre-load output bit-identically; re-packing (.to) re-applies the adapter."""
    cfg, sd = _tiny()
    lora = lo.synth_lora(cfg, rank=4, seed=3)
    kv_only = lo.synth_lora(cfg, rank=4, seed=4, projections=("add_k_proj", "add_v_proj"))
    g = torch.Generator().manual_seed(0)
    x = torch.randn(2, 4, 16, 16, generator=g).cuda()
    t = torch.tensor([700.0, 30.0]).cuda()
    kw = dict(image_emb=torch.randn(2, 1280, generator=g).cuda())

    m = _build(cfg, sd)
    y0 = m(x, t, **kw)
    y0b = m(x, t, **kw)
    assert torch.equal(y0, y0b)
    plans = dict(m._plans)
    graphs = {k: p.graph for k, p in plans.items()}
    assert all(gr is not None for gr in graphs.values())
    ptrs = {(p, n): a[n].data_ptr() for p, a in m._packed["attn"].items() for n in ("wqkv", "wenc", "wproj")}
    sd0 = {k: v.clone() for k, v in m.state_dict().items()}

    def same_plans():
        assert m._plans.keys() == plans.keys() and all(m._plans[k] is plans[k] for k in plans)
        assert all(m._plans[k].graph is graphs[k] for k in plans)
        assert {(p, n): a[n].data_ptr() for p, a in m._packed["attn"].items() for n in ("wqkv", "wenc", "wproj")} == ptrs

    def fresh(adapter, scale):
        f = _build(cfg, sd)
        f.load_lora(adapter, scale)
        return f(x, t, **kw)

    m.load_lora(lora)
    y1 = m(x, t, **kw)
    same_plans()
    assert not torch.equal(y1, y0)
    assert torch.equal(y1, fresh(lora, 1.0))

    m.load_lora(kv_only)
    y2 = m(x, t, **kw)
    same_plans()
    assert not torch.equal(y2, y0)
    assert torch.equal(y2, fresh(kv_only, 1.0))

    m.load_lora(lora, scale=0.5)
    assert m.lora_scale == 0.5
    y3 = m(x, t, **kw)
    same_plans()
    assert torch.equal(y3, fresh(lora, 0.5))
    assert not torch.equal(y3, y1)

    m.unload_lora()
    assert m.lora_scale is None
    y4 = m(x, t, **kw)
    same_plans()
    assert torch.equal(y4, y0)
    assert all(torch.equal(v, sd0[k]) for k, v in m.state_dict().items())

    m.load_lora(lora)
    m.to("cuda")          # re-packs the weights: the adapter is merged again into the new packing
    assert m._plans == {} and m.lora_scale == 1.0
    assert torch.equal(m(x, t, **kw), y1)
    assert all(torch.equal(v, sd0[k]) for k, v in m.state_dict().items())


def test_lora_pipeline_22():
    """get_kandinsky2(model_version="2.2") with pipe.model.load_lora: different images; after unload_lora the uint8 images equal
    the pre-load run's."""
    import numpy as np
    from kandinsky2 import get_kandinsky2
    from tests.test_gpu_movq_sampler import _tiny_overrides
    pipe = get_kandinsky2("cuda", task_type="text2img", model_version="2.2", cache_dir="/nonexistent",
                          config_overrides=_tiny_overrides())
    m = pipe.model
    cfg = dict(in_channels=m.in_channels, model_channels=m.model_channels, channel_mult=m.channel_mult,
               num_res_blocks=m.num_res_blocks, attention_ds=m.attention_resolutions, model_dim=m.model_dim)
    lora = lo.synth_lora(cfg, rank=4, seed=5, gain=1.0)
    run = lambda: np.stack([np.asarray(im) for im in pipe.generate_text2img("a red cat", batch_size=2, decoder_steps=4,
                                                                            h=64, w=64)])
    a = run()
    m.load_lora(lora)
    b = run()
    assert not np.array_equal(a, b)
    m.unload_lora()
    c = run()
    assert np.array_equal(a, c)
    assert math.isfinite(float(b.mean()))
