"""GPU: the Kandinsky 2.1 continuously refilled batch (batching.Batcher21) -- the cond-first and per-slot thresholded slot steps
against their batch forms bit for bit, the per-slot percentile against float64, a request's isolation from the other slots,
parity with generate_text2img and mix_images, and the one captured graph."""
import numpy as np
import pytest
import torch

from tests.sampler_cases import _check, _pipe
from tests.test_gpu_batcher import ACTIVE, NAN, STATE, _outside_untouched, _poisoned, _run, _state, _step

pytestmark = pytest.mark.gpu

SAMPLERS = ("p_sampler", "ddim_sampler", "dpmpp_2m_sampler", "dpmpp_2m_karras_sampler")


def _rows(kind):
    """Five coefficient rows of the 2.1 schedules: p_sampler's respaced DDPM rows or DPM-Solver++(2M)'s."""
    from kandinsky2.configs import CONFIG_2_1
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule, create_gaussian_diffusion
    dc = CONFIG_2_1["diffusion_config"]
    if kind == "ddpm":
        tab = create_gaussian_diffusion(**dict(dc, timestep_respacing="5")).coef_table()
    else:
        tab = DPMSolverSchedule(create_gaussian_diffusion(**dc).base_alphas_cumprod, 5).coef_table()
    return torch.from_numpy(tab).cuda()


@pytest.mark.parametrize("kind,threshold_mode", [("ddpm", 1), ("ddpm", 0), ("dpmpp_2m", 0)])
def test_cond_first_slot_step_equals_the_batch_step_per_slot(kind, threshold_mode):
    """cond_first = 1 (conditional row s, unconditional row S + s), active slots at different steps with different guidance,
    idle slots whose latent, side buffer and UNet rows are NaN, all operands inside NaN-poisoned memory: every active slot
    equals k2_sampler_step (threshold_mode as given) / k2_dpm_solver_step at B = 1, cond_first = 1, bit for bit -- its latent,
    its x0 and, with the threshold, the percentile the batch form finds for sample 0, which is also max(np.percentile(|x0|,
    99.5), 1) in float64 to the fp32 rounding of the result.  Idle slots (their sval included) and everything outside the
    views stay as they were."""
    from kandinsky2 import ops
    S, H, W = len(STATE), 6, 9
    n = 4 * H * W
    g = torch.Generator(device="cuda").manual_seed(2)
    coef = _rows(kind)[:S].contiguous()
    guid = torch.tensor([1.0, 4.0, 7.5, 2.0, 5.5], device="cuda")[:S]
    mo = torch.randn(2 * S, 8, H, W, device="cuda", generator=g)
    x0 = 3 * torch.randn(S, 4, H, W, device="cuda", generator=g)   # wide enough that the threshold exceeds 1 and clips
    side = torch.randn(S, 4, H, W, device="cuda", generator=g)      # noise (ddpm) / history (dpm)
    for s in range(S):
        if s not in ACTIVE:
            mo[s] = mo[S + s] = x0[s] = side[s] = NAN
        elif coef[s, 4 if kind == "dpmpp_2m" else 6].item() == 0:
            side[s] = NAN
    bm, mo_v, pm, nm = _poisoned(mo.shape, mo)
    bx, x, px, nx = _poisoned(x0.shape, x0)
    bs, sd, ps, ns = _poisoned(side.shape, side)
    bc, cf, pc, nc = _poisoned(coef.shape, coef)
    bg, gv, pg, ng = _poisoned(guid.shape, guid)
    bufs = [(bm, pm, nm), (bx, px, nx), (bs, ps, ns), (bc, pc, nc), (bg, pg, ng)]
    state = _state(S)
    if kind == "ddpm":
        bw, work, pw, nw = _poisoned((S, 4, H, W))
        bv, sval, pv, nv = _poisoned((S,))
        bufs += [(bw, pw, nw), (bv, pv, nv)]
        ops.slot_sampler_step(mo_v, x, sd, cf, gv, state, work, 2.0, cond_first=1, threshold_mode=threshold_mode,
                              sval=sval)
    else:
        ops.slot_dpm_solver_step(mo_v, x, sd, cf, gv, state, cond_first=1)
    torch.cuda.synchronize()
    clipped = 0
    for s in range(S):
        if s not in ACTIVE:
            assert torch.isnan(x[s]).all() and torch.isnan(sd[s]).all()
            if kind == "ddpm":
                assert torch.isnan(work[s]).all() and torch.isnan(sval[s]).item()
            continue
        one_mo = torch.stack([mo[s], mo[S + s]]).contiguous()   # B = 1, conditional row first
        ref = x0[s:s + 1].clone()
        if kind == "ddpm":
            wref = torch.full((n + 4096,), NAN, device="cuda")
            ops.sampler_step(one_mo, ref, side[s:s + 1].contiguous(), coef[s].contiguous(), guid[s].item(), True, clip=2.0,
                             threshold_mode=threshold_mode, work=wref)
            torch.cuda.synchronize()
            assert torch.equal(work[s].reshape(-1), wref[:n])
            if threshold_mode:
                assert torch.equal(sval[s], wref[n]), (s, sval[s].item(), wref[n].item())
                a = work[s].double().abs().cpu().numpy().reshape(-1)
                want = max(float(np.percentile(a, 99.5)), 1.0)
                assert abs(sval[s].item() - want) <= 2.0 ** -23 * want, (s, sval[s].item(), want)
                clipped += sval[s].item() > 1.0
            else:
                assert torch.isnan(sval).all()
        else:
            hist = side[s:s + 1].clone()
            ops.dpm_solver_step(one_mo, ref, hist, coef[s].contiguous(), guid[s].item(), True)
            torch.cuda.synchronize()
            assert torch.equal(sd[s], hist[0])
        assert torch.equal(x[s], ref[0]), (kind, threshold_mode, s)
        assert torch.isfinite(x[s]).all()
    if threshold_mode:
        assert clipped >= 2   # the threshold did more than the +-2 clamp
    assert torch.equal(state, _state(S))
    for b, p, m in bufs:
        assert _outside_untouched(b, p, m)


def test_cond_first_steps_differ_from_the_22_order():
    """The row order reaches the kernels: on the same operands cond_first 0 and 1 give different latents."""
    from kandinsky2 import ops
    S, H, W = 2, 4, 4
    g = torch.Generator(device="cuda").manual_seed(3)
    mo = torch.randn(2 * S, 8, H, W, device="cuda", generator=g)
    x = torch.randn(S, 4, H, W, device="cuda", generator=g)
    coef = _rows("dpmpp_2m")[:S].contiguous()
    guid = torch.full((S,), 4.0, device="cuda")
    state = torch.tensor([[0, 1], [5, 5]], dtype=torch.int32, device="cuda")
    outs = []
    for cf in (0, 1):
        xx, hist = x.clone(), torch.zeros_like(x)
        ops.slot_dpm_solver_step(mo, xx, hist, coef, guid, state, cond_first=cf)
        outs.append(xx)
    assert not torch.equal(outs[0], outs[1])


# ---- the batcher on the tiny 2.1 pipeline ----------------------------------------------------------------------------------
@pytest.mark.parametrize("sampler", SAMPLERS)
def test_request_is_isolated_from_the_other_slots(sampler):
    """A request's final latent and image are the same bits alone in the batcher (slot 0, every other slot idle) and alongside
    requests admitted at other steps, with other prompts, guidance scales and step counts, while it sits in slot 2."""
    pipe = _pipe("2.1", "text2img")
    req = dict(num_steps=6, guidance_scale=7.0, seed=11)
    lat_a, lat_b = {}, {}
    alone = pipe.batcher(3, 64, 64, sampler=sampler, max_steps=12)
    h = alone.submit("a red cat", **req)
    img_alone = _run(alone, lat_a)[h]
    mixed = pipe.batcher(3, 64, 64, sampler=sampler, max_steps=12)
    mixed.submit("a blue dog", num_steps=8, guidance_scale=4.0, negative_decoder_prompt="blurry", seed=5)
    _step(mixed, lat_b)
    mixed.submit("a green bird", num_steps=4, guidance_scale=2.0, seed=7)
    _step(mixed, lat_b)
    _step(mixed, lat_b)
    h2 = mixed.submit("a red cat", **req)
    out = _step(mixed, lat_b)
    assert mixed.queue.holder[2] == h2
    out.update(_run(mixed, lat_b))
    assert mixed.queue.holder == [None, None, None]
    assert torch.equal(lat_a[h], lat_b[h2]) and torch.isfinite(lat_a[h]).all()
    assert img_alone.tobytes() == out[h2].tobytes()
    assert len(lat_b) == 3 and not torch.equal(lat_b[0], lat_b[h2])


@pytest.mark.parametrize("sampler", SAMPLERS)
def test_batch_of_one_equals_generate_text2img_and_mix_images(sampler):
    """max_batch = 1: the image and latent of a request equal Kandinsky2_1.generate_text2img(batch_size=1) with base_seed = the
    request's seed, bit for bit, and a request with prompt "" and image_embeds = the embedder's interpolation equals
    mix_images(batch_size=1).  max_batch = 4: three requests are within the tiny-UNet loop bound of theirs."""
    pipe = _pipe("2.1", "text2img")
    kw = dict(num_steps=5, guidance_scale=7)
    lats = {}
    b = pipe.batcher(1, 72, 60, sampler=sampler, max_steps=8)
    h = b.submit("a red cat", seed=1234, **kw)
    items, weights = ["a cat", "a dog"], [0.3, 0.7]
    hm = b.submit("", image_embeds=pipe.embedder.interpolate(items, weights, 1), seed=77, **kw)
    got = _run(b, lats)
    pipe.base_seed = 1234
    want = pipe.generate_text2img("a red cat", batch_size=1, h=72, w=60, sampler=sampler, **kw)
    assert got[h].size == (60, 72) and got[h].tobytes() == want[0].tobytes()
    assert torch.equal(lats[h], pipe.seen[-1])
    pipe.base_seed = 77
    want = pipe.mix_images(items, weights, batch_size=1, h=72, w=60, sampler=sampler, **kw)
    assert got[hm].tobytes() == want[0].tobytes()
    assert torch.equal(lats[hm], pipe.seen[-1])
    b4 = pipe.batcher(4, 64, 64, sampler=sampler, max_steps=8)
    lats4 = {}
    reqs = [("a red cat", 21, 5, 7.0), ("a blue dog", 22, 4, 4.0), ("a green bird", 23, 7, 2.5)]
    hs = [b4.submit(p, seed=sd, num_steps=n, guidance_scale=g) for p, sd, n, g in reqs]
    _run(b4, lats4)
    for hh, (p, sd, n, g) in zip(hs, reqs):
        pipe.base_seed = sd
        pipe.generate_text2img(p, batch_size=1, h=64, w=64, sampler=sampler, num_steps=n, guidance_scale=g)
        _check(lats4[hh], pipe.seen[-1], f"batcher21 max_batch 4 {sampler} {p}")


def test_one_step_is_one_graph_replay():
    """step() replays the batcher's one captured graph exactly once while a slot is occupied, and never otherwise; admitting
    and finishing requests keeps that graph and every buffer address it was captured on (the per-slot thresholds included)."""
    pipe = _pipe("2.1", "text2img")
    b = pipe.batcher(2, 64, 64, sampler="p_sampler", max_steps=8)
    g0 = b.graph
    sl = b.slots
    bufs = [sl.x, sl.state, sl.ts_tab, sl.coef_tab, sl.coef, sl.guidance, sl.noise_tab, sl.noise, sl.work, sl.sval, b.plan.x_in,
            b.plan.t_in, b.plan.out, b.plan.xf_proj] + list(b.plan.enc_kv.values())
    ptrs = [t.data_ptr() for t in bufs]
    calls = []
    orig = g0.replay
    g0.replay = lambda: (calls.append(1), orig())[1]
    assert b.step() == {} and not calls
    for i, n in enumerate((3, 5, 2)):
        b.submit(f"prompt {i}", num_steps=n, seed=i)
    steps = finished = 0
    while b.pending():
        before = len(calls)
        finished += len(b.step())
        steps += 1
        assert len(calls) == before + 1
    assert finished == 3 and steps == len(calls)
    assert b.graph is g0 and [t.data_ptr() for t in bufs] == ptrs


def test_full_size_isolation_p_sampler():
    """The isolation property at the full Kandinsky 2.1 UNet (synthetic weights), 768 x 768 images (96 x 96 latents), with the
    per-slot dynamic threshold: a request's latent is the same bits alone in slot 0 and in slot 1 next to another request
    admitted a step earlier."""
    from kandinsky2 import get_kandinsky2
    pipe = get_kandinsky2("cuda", task_type="text2img", model_version="2.1", cache_dir="/nonexistent")
    seen = []
    orig = pipe._finish
    pipe._finish = lambda lat, h, w: (seen.append(lat.clone()), orig(lat, h, w))[1]
    pipe.seen = seen
    req = dict(num_steps=3, guidance_scale=7.0, seed=3)
    la, lb = {}, {}
    alone = pipe.batcher(2, 768, 768, sampler="p_sampler", max_steps=4)
    h = alone.submit("a red cat", **req)
    _run(alone, la)
    del alone
    mixed = pipe.batcher(2, 768, 768, sampler="p_sampler", max_steps=4)
    mixed.submit("a blue dog", num_steps=4, guidance_scale=4.0, seed=9)
    _step(mixed, lb)
    h2 = mixed.submit("a red cat", **req)
    _run(mixed, lb)
    assert la[h].shape == (1, 4, 96, 96) and torch.isfinite(la[h]).all()
    assert torch.equal(la[h], lb[h2])
