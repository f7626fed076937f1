"""GPU: per-request LoRA adapters in the continuously refilled batch -- the mapped batched GEMM (k2_conv_gemm_wmap) bit for bit
against the unmapped batched GEMM and against float64, the slab tables against load_lora's merge, the isolation of a request
from its neighbours' adapters, parity with load_lora + generate_text2img, and the one captured graph."""
import pytest
import torch

from tests.sampler_cases import _check, _pipe
from tests.test_gpu_batcher import _embeds, _run, _step
from tests.test_gpu_conv_float64 import _check as _check64

pytestmark = pytest.mark.gpu

NAN = float("nan")
SAMPLERS = ("ddpm_sampler", "dpmpp_2m_sampler", "dpmpp_2m_karras_sampler")


def _poisoned(n, pad=1024, dtype=torch.float16):
    """A NaN buffer with n elements in its middle: (view of the n, the whole buffer)."""
    buf = torch.full((n + 2 * pad,), NAN, device="cuda", dtype=dtype)
    return buf[pad:pad + n], buf, pad


def _outside_nan(buf, pad, n):
    return bool(torch.isnan(buf[:pad].float()).all() and torch.isnan(buf[pad + n:].float()).all())


# attention-layer geometries of the UNet at 768 x 768 (T = 144, 576, 2304 tokens) and a ragged small one
GEOMS = [(12, 12), (24, 24), (48, 48), (5, 7)]
MAPS = {"mixed": [2, 0, 2, 3, 1, 2], "one_slab": [3] * 6, "slab0": [0] * 6}


def _mapped_case(H, W, cout, residual, seed, C=128, NB=6, slabs=5, used=(0, 1, 2, 3)):
    g = torch.Generator(device="cuda").manual_seed(seed)
    x = torch.randn(NB, H, W, C, device="cuda", generator=g).half()
    w = (torch.randn(slabs, cout, C, device="cuda", generator=g) / C ** 0.5).half()
    for k in range(slabs):
        if k not in used:
            w[k] = NAN   # a slab the map never names: any read of it would show
    bias = torch.randn(cout, device="cuda", generator=g)
    res = torch.randn(NB, H, W, cout, device="cuda", generator=g).half() if residual else None
    return x, w, bias, res


def _run_mapped(x, w, bias, res, cout, wmap, cfg):
    from kandinsky2 import ops
    NB, H, W, _ = x.shape
    n = NB * H * W * cout
    out, obuf, pad = _poisoned(n)
    gn_n = ops.gn_part_floats(NB, H, W, cout)
    gn, gbuf, gpad = _poisoned(gn_n, dtype=torch.float32)
    info = [0] * 7
    m = torch.tensor(wmap, device="cuda", dtype=torch.int32)
    ops.conv_gemm([(x, 1)], w[0], cout, bias=bias, residual=res, out=out.view(NB, H, W, cout), gn_part=gn, info=info,
                  cfg=cfg, w_batch_stride=w.stride(0), w_map=m, n_slabs=w.shape[0])
    torch.cuda.synchronize()
    assert _outside_nan(obuf, pad, n) and _outside_nan(gbuf, gpad, gn_n)
    return out.view(NB, H, W, cout), gn, info


@pytest.mark.parametrize("geom", GEOMS, ids=[f"{h}x{w}" for h, w in GEOMS])
@pytest.mark.parametrize("layer", ["qkv", "proj_out"])
def test_mapped_gemm_equals_the_batched_gemm_with_the_slab_in_place(geom, layer):
    """Image n of the mapped GEMM has the bits of the unmapped batched GEMM run with slab map[n] at position n: output, and for
    the proj_out form (bias + residual + GroupNorm partials) the partials too, for every N tile and several maps, with NaN
    around the outputs and in the slabs the map does not name."""
    from kandinsky2 import ops
    H, W = geom
    cout, residual = (384, False) if layer == "qkv" else (128, True)
    x, w, bias, res = _mapped_case(H, W, cout, residual, seed=H * 31 + W + cout)
    tiles = (16, 64, 128, 192, 256) if layer == "qkv" else (64, 128, 192, 256)
    for name, wmap in MAPS.items():
        wref = torch.stack([w[k] for k in wmap]).contiguous()
        for bn in tiles:
            cfg = (bn, 0, 0, 1)
            y, gn, info = _run_mapped(x, w, bias, res, cout, wmap, cfg)
            assert info[0] == bn and info[2] == 1 and info[4] == 1, (name, bn, info)
            if layer == "proj_out" and bn >= 64:
                assert info[5] == 1, (name, bn, info)
            want = torch.empty_like(y)
            gw = torch.zeros_like(gn)
            wi = [0] * 7
            ops.conv_gemm([(x, 1)], wref[0], cout, bias=bias, residual=res, out=want, gn_part=gw, info=wi, cfg=cfg,
                          w_batch_stride=wref.stride(0))
            torch.cuda.synchronize()
            assert wi == info, (name, bn, wi, info)
            assert torch.equal(y, want), (geom, layer, name, bn)
            if info[5]:
                k = info[6] * cout * 2
                assert torch.equal(gn[:k], gw[:k]), (geom, layer, name, bn)
            assert torch.isfinite(y).all()


@pytest.mark.parametrize("geom", GEOMS, ids=[f"{h}x{w}" for h, w in GEOMS])
def test_mapped_gemm_vs_float64(geom):
    """Within the bound of tests/test_gpu_gemm_float64.py: one fp16 rounding of the result plus fp32 accumulation over the K
    products, the bias and the residual."""
    H, W = geom
    cout = 128
    x, w, bias, res = _mapped_case(H, W, cout, True, seed=7 * H + W)
    wmap = MAPS["mixed"]
    y, _, _ = _run_mapped(x, w, bias, res, cout, wmap, None)
    wm = torch.stack([w[k] for k in wmap]).double()
    xd = x.double().reshape(x.shape[0], -1, x.shape[-1])
    ref = torch.bmm(xd, wm.transpose(1, 2)).reshape(res.shape) + bias.double() + res.double()
    absum = (torch.bmm(xd.abs(), wm.abs().transpose(1, 2)).reshape(res.shape) + bias.double().abs() + res.double().abs())
    worst = _check64(y, ref, absum, x.shape[-1] + 2)
    print(f"mapped GEMM {geom}: worst {worst:.3f} of the bound")


def test_ops_refuse_maps_the_kernel_would_misread():
    from kandinsky2 import ops
    from kandinsky2._native import K2Error
    x = torch.zeros(2, 4, 4, 64, device="cuda", dtype=torch.float16)
    w = torch.zeros(2, 64, 64, device="cuda", dtype=torch.float16)
    ok = torch.zeros(2, device="cuda", dtype=torch.int32)
    cases = [(dict(w_map=ok.long()), "int32"), (dict(w_map=torch.zeros(4, device="cuda", dtype=torch.int32)[::2]), "contiguous"),
             (dict(w_map=torch.zeros(3, device="cuda", dtype=torch.int32)), "one slab index per image"),
             (dict(w_map=ok, n_slabs=0), "n_slabs")]
    for kw, msg in cases:
        args = dict(n_slabs=2)
        args.update(kw)
        with pytest.raises(K2Error, match=msg):
            ops.conv_gemm([(x, 1)], w[0], 64, w_batch_stride=w.stride(0), **args)


# ---- the batcher --------------------------------------------------------------------------------------------------------------
def _lora(model, rank, seed):
    """A synthetic adapter of `model`'s attention blocks in the format load_lora takes (tests/lora_oracle.py)."""
    from oracle import unet_oracle as uo
    from tests import lora_oracle as lo
    cfg = dict(uo.CONFIG_2_2, in_channels=model.in_channels, model_channels=model.model_channels,
               channel_mult=tuple(model.channel_mult), num_res_blocks=model.num_res_blocks,
               attention_ds=tuple(model.attention_resolutions), model_dim=model.model_dim, inpainting=False)
    return lo.synth_lora(cfg, rank=rank, seed=seed)


def test_slabs_are_the_weights_load_lora_merges():
    """After add_lora(A, s) every layer's slab holds the bits load_lora(A, s) writes into the packed weights, and the adapter's
    encoder_kv weights those too -- also when the pipeline itself has another adapter loaded (both merge from the unmerged
    weights) -- and slab 0 keeps the weights the batcher was made with."""
    pipe = _pipe("2.2", "text2img")
    m = pipe.model
    A, B = _lora(m, 4, 1), _lora(m, 8, 2)
    m.load_lora(B, 0.5)
    b = pipe.batcher(2, 64, 64, max_steps=4, max_loras=2)
    slab0 = {p: (t[0].clone(), u[0].clone()) for p, (t, u) in b.plan.attn_slabs["layers"].items()}
    b.add_lora("a", A, 0.7)
    k, wenc = b._loras["a"]
    assert k == 1
    m.load_lora(A, 0.7)
    for p, a in m._packed["attn"].items():
        wqkv, wproj = b.plan.attn_slabs["layers"][p]
        assert torch.equal(wqkv[k], a["wqkv"]) and torch.equal(wproj[k], a["wproj"]) and torch.equal(wenc[p], a["wenc"]), p
        assert torch.equal(wqkv[0], slab0[p][0]) and torch.equal(wproj[0], slab0[p][1])
    m.unload_lora()
    for p, a in m._packed["attn"].items():
        assert not torch.equal(b.plan.attn_slabs["layers"][p][0][0], a["wqkv"]), p   # slab 0 is B's merge, not the base


def _isolation(pipe, sampler, size, max_steps, req, other):
    """(latent of req alone in slot 0, latent of req in slot 1 of a batch whose other slots run adapter B / no adapter)."""
    m = pipe.model
    A, B = _lora(m, 4, 11), _lora(m, 16, 12)
    la, lb = {}, {}
    alone = pipe.batcher(3, size, size, sampler=sampler, max_steps=max_steps, max_loras=2)
    alone.add_lora("A", A, 0.8)
    h = alone.submit(**req, lora="A")
    _run(alone, la)
    del alone
    mixed = pipe.batcher(3, size, size, sampler=sampler, max_steps=max_steps, max_loras=2)
    mixed.add_lora("B", B, 1.0)
    mixed.add_lora("A", A, 0.8)
    mixed.submit(**other, lora="B")
    _step(mixed, lb)
    h2 = mixed.submit(**req, lora="A")
    mixed.submit(**dict(other, seed=other["seed"] + 1, decoder_steps=2))
    _step(mixed, lb)
    assert mixed.queue.holder[1] == h2 and mixed.w_map.tolist() == [1, 2, 0, 1, 2, 0]   # B in slab 1, A in slab 2
    _run(mixed, lb)
    assert mixed.w_map.tolist() == [0] * 6
    return la[h], lb[h2]


@pytest.mark.parametrize("sampler", SAMPLERS)
def test_request_with_an_adapter_is_isolated_from_the_other_slots(sampler):
    pipe = _pipe("2.2", "text2img")
    pos, neg = _embeds(pipe, "a red cat")
    p2, n2 = _embeds(pipe, "a blue dog")
    req = dict(image_embeds=pos, negative_image_embeds=neg, decoder_steps=6, decoder_guidance_scale=4.0, seed=11)
    other = dict(image_embeds=p2, negative_image_embeds=n2, decoder_steps=7, decoder_guidance_scale=6.0, seed=5)
    a, b = _isolation(pipe, sampler, 64, 8, req, other)
    assert torch.isfinite(a).all() and torch.equal(a, b)


def test_full_size_isolation_with_adapters():
    """The isolation at the full Kandinsky 2.2 UNet, 768 x 768 (96 x 96 latents), the seeds of the full-size batcher test."""
    from kandinsky2 import get_kandinsky2
    pipe = get_kandinsky2("cuda", task_type="text2img", model_version="2.2", cache_dir="/nonexistent")
    seen = []
    orig = pipe._finish
    pipe._finish = lambda lat, h, w: (seen.append(lat.clone()), orig(lat, h, w))[1]
    pipe.seen = seen
    pos, neg = _embeds(pipe, "a red cat")
    p2, n2 = _embeds(pipe, "a blue dog")
    req = dict(image_embeds=pos, negative_image_embeds=neg, decoder_steps=3, decoder_guidance_scale=4.0, seed=3)
    other = dict(image_embeds=p2, negative_image_embeds=n2, decoder_steps=4, decoder_guidance_scale=6.0, seed=9)
    a, b = _isolation(pipe, "ddpm_sampler", 768, 4, req, other)
    assert a.shape == (1, 4, 96, 96) and torch.isfinite(a).all() and torch.equal(a, b)


@pytest.mark.parametrize("sampler", SAMPLERS)
def test_batch_of_one_matches_load_lora_and_the_plain_batcher(sampler):
    """max_batch = 1: a request with adapter A is within the tiny-UNet loop bound of load_lora(A) + generate_text2img, and a
    request without one within it of the batcher made with max_loras=0 (not bit-exact: the mapped GEMMs never split K)."""
    pipe = _pipe("2.2", "text2img")
    A = _lora(pipe.model, 8, 21)
    kw = dict(decoder_steps=5, decoder_guidance_scale=4)
    lats = {}
    b = pipe.batcher(1, 64, 64, sampler=sampler, max_steps=8, max_loras=1)
    b.add_lora("A", A, 0.9)
    ha = b.submit("a red cat", seed=1234, lora="A", **kw)
    hn = b.submit("a red cat", seed=1234, **kw)
    _run(b, lats)
    plain = pipe.batcher(1, 64, 64, sampler=sampler, max_steps=8)
    hp = plain.submit("a red cat", seed=1234, **kw)
    lats_p = {}
    _run(plain, lats_p)
    _check(lats[hn], lats_p[hp], f"max_loras=1 no adapter vs max_loras=0 {sampler}")
    pipe.model.load_lora(A, 0.9)
    pipe.base_seed = 1234
    pipe.generate_text2img("a red cat", batch_size=1, h=64, w=64, sampler=sampler, **kw)
    pipe.model.unload_lora()
    _check(lats[ha], pipe.seen[-1], f"adapter A vs load_lora(A) + generate_text2img {sampler}")
    assert not torch.equal(lats[ha], lats[hn])


def test_registry_keeps_one_graph_and_its_addresses():
    """add_lora, remove_lora, admission and finishing keep the one captured graph and every buffer it reads; one step() is one
    replay; the mapped layers were tuned under keys of their own."""
    from kandinsky2 import launch_plan
    pipe = _pipe("2.2", "text2img")
    m = pipe.model
    b = pipe.batcher(2, 64, 64, max_steps=8, max_loras=2)
    g0 = b.graph
    bufs = [b.slots.x, b.slots.state, b.w_map, b.plan.x_in, b.plan.out, b.plan.xf_proj] + list(b.plan.enc_kv.values())
    bufs += [t for pair in b.plan.attn_slabs["layers"].values() for t in pair]
    ptrs = [t.data_ptr() for t in bufs]
    calls = []
    orig = g0.replay
    g0.replay = lambda: (calls.append(1), orig())[1]
    b.add_lora("A", _lora(m, 4, 31))
    b.add_lora("B", _lora(m, 4, 32))
    b.submit("prompt 0", decoder_steps=3, seed=0, lora="A")
    b.submit("prompt 1", decoder_steps=2, seed=1, lora="B")
    steps = 0
    while b.pending():
        before = len(calls)
        b.step()
        steps += 1
        assert len(calls) == before + 1
    b.remove_lora("B")
    b.add_lora("C", _lora(m, 4, 33))
    assert b._loras["C"][0] == 2
    b.submit("prompt 2", decoder_steps=2, seed=2, lora="C")
    b.run()
    assert steps == 3 and len(calls) == 5 and b.graph is g0 and [t.data_ptr() for t in bufs] == ptrs
    assert any(k[2] == "conv" and k[-1] is True for k in launch_plan._tune_cache)
