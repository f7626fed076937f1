"""GPU: the continuously refilled batch (kandinsky2/batching.py) -- the slot kernels against their batch forms bit for bit and
against float64, a request's isolation from the other slots, parity with generate_text2img, and the one captured graph."""
import numpy as np
import pytest
import torch

from tests.sampler_cases import _check, _pipe

pytestmark = pytest.mark.gpu

NAN = float("nan")
SAMPLERS = ("ddpm_sampler", "dpmpp_2m_sampler", "dpmpp_2m_karras_sampler")
EPS32 = 2.0 ** -24


def _poisoned(shape, fill=None, pad=1000):
    """-> (the NaN-filled buffer, a view of `shape` inside it, holding `fill` if given)"""
    n = int(np.prod(shape))
    buf = torch.full((n + 2 * pad,), NAN, device="cuda")
    view = buf[pad:pad + n].view(shape)
    if fill is not None:
        view.copy_(fill)
    return buf, view, pad, n


def _outside_untouched(buf, pad, n):
    return bool(torch.isnan(buf[:pad]).all() and torch.isnan(buf[pad + n:]).all())


# slot -> (k_s, steps_s): active at different steps, free (-1) and past its last step
STATE = [(2, 5), (-1, 0), (0, 3), (4, 4), (1, 2)]
ACTIVE = [s for s, (k, n) in enumerate(STATE) if 0 <= k < n]


def _state(S):
    st = torch.tensor([[k for k, _ in STATE[:S]], [n for _, n in STATE[:S]]], dtype=torch.int32, device="cuda")
    return st


def test_slot_step_begin_stages_each_active_slot_and_zeroes_the_rest():
    from kandinsky2 import ops
    S, H, W, kmax = len(STATE), 5, 7, 6
    n = 4 * H * W
    g = torch.Generator(device="cuda").manual_seed(0)
    x = torch.randn(S, 4, H, W, device="cuda", generator=g)
    for s in range(S):
        if s not in ACTIVE:
            x[s] = NAN
    ts = torch.rand(S, kmax, device="cuda", generator=g) * 1000
    coef = torch.randn(S, kmax, 8, device="cuda", generator=g)
    noise_tab = torch.randn(S, kmax, 4, H, W, device="cuda", generator=g)
    bx, xin, px, nx = _poisoned((2 * S, 4, H, W))
    bt, tin, pt, nt = _poisoned((2 * S,))
    bc, cout, pc, nc = _poisoned((S, 8))
    bn, noise, pn, nn = _poisoned((S, 4, H, W))
    state = _state(S)
    ops.slot_step_begin(x, xin, tin, cout, ts, coef, noise_tab, noise, state)
    torch.cuda.synchronize()
    for s in range(S):
        k = STATE[s][0]
        if s in ACTIVE:
            assert torch.equal(xin[s], x[s]) and torch.equal(xin[S + s], x[s])
            assert tin[s].item() == ts[s, k].item() and tin[S + s].item() == ts[s, k].item()
            assert torch.equal(cout[s], coef[s, k]) and torch.equal(noise[s], noise_tab[s, k])
        else:
            assert not xin[s].any() and not xin[S + s].any() and tin[s].item() == 0 and tin[S + s].item() == 0
            assert not cout[s].any() and not noise[s].any()
    for b, p, m in ((bx, px, nx), (bt, pt, nt), (bc, pc, nc), (bn, pn, nn)):
        assert _outside_untouched(b, p, m)
    assert torch.equal(state, _state(S))
    ops.slot_step_end(state)
    torch.cuda.synchronize()
    want = [[k + 1 if s in ACTIVE else k for s, (k, _) in enumerate(STATE)], [n for _, n in STATE]]
    assert state.tolist() == want


def _ddpm64(mo, x, noise, c, g, s, S):
    """float64 k2_sampler_step of slot s (cond_first 0, clip 2, no threshold) -> (x', a bound on the fp32 error terms)"""
    mo, x, noise, c = mo.double(), x.double(), noise.double(), c.double()
    eu, ec = mo[s, :4], mo[S + s, :4]
    eps = eu + g * (ec - eu)
    x0 = (c[0] * x - c[1] * eps).clamp(-2, 2)
    mean = c[2] * x0 + c[3] * x
    frac = (mo[S + s, 4:] + 1) * 0.5
    sd = torch.exp(0.5 * (frac * c[5] + (1 - frac) * c[4]))
    term = c[6] * sd * noise if c[6] != 0 else torch.zeros_like(mean)   # the noise is not read without a noise term
    out = mean + term
    scale = (c[0] * x).abs() + (c[1] * eps).abs() + eu.abs() + abs(g) * (ec.abs() + eu.abs())
    scale = c[2].abs() * scale + (c[3] * x).abs() + term.abs() * 4
    return out, scale


def _dpm64(mo, x, hist, c, g, s, S):
    mo, x, hist, c = mo.double(), x.double(), hist.double(), c.double()
    eu, ec = mo[s, :4], mo[S + s, :4]
    eps = eu + g * (ec - eu)
    x0 = c[0] * x - c[1] * eps
    out = c[2] * x + c[3] * x0 + (c[4] * hist if c[4] != 0 else 0)
    scale = (c[0] * x).abs() + (c[1] * eps).abs() + eu.abs() + abs(g) * (ec.abs() + eu.abs())
    scale = c[3].abs() * scale + (c[2] * x).abs() + ((c[4] * hist).abs() if c[4] != 0 else 0)
    return out, x0, scale


@pytest.mark.parametrize("kind", ["ddpm", "dpmpp_2m"])
def test_slot_step_equals_the_batch_step_per_slot(kind):
    """Active slots at different steps with different guidance, idle slots whose latent, history and UNet rows are NaN, all
    operands inside NaN-poisoned memory: every active slot equals k2_sampler_step / k2_dpm_solver_step run on that slot alone,
    bit for bit, and float64 within a few fp32 ulps of its terms; idle slots and everything outside the views stay as they
    were."""
    from kandinsky2 import ops
    from kandinsky2.model.gaussian_diffusion import DPMSolverSchedule, create_ddpm_v22
    S, H, W = len(STATE), 6, 9
    g = torch.Generator(device="cuda").manual_seed(1)
    sched = create_ddpm_v22(5)
    if kind == "ddpm":
        rows = torch.from_numpy(sched.coef_table()).cuda()
    else:
        rows = torch.from_numpy(DPMSolverSchedule(sched.base_alphas_cumprod, 5).coef_table()).cuda()
    coef = rows[:S].contiguous()   # the active slots 0, 2, 4 get the last step, a middle one and the first one
    guid = torch.tensor([1.0, 4.0, 7.5, 2.0, 5.5], device="cuda")[:S]
    mo = torch.randn(2 * S, 8, H, W, device="cuda", generator=g)
    x0 = torch.randn(S, 4, H, W, device="cuda", generator=g)
    side = torch.randn(S, 4, H, W, device="cuda", generator=g)            # noise (ddpm) / history (dpm)
    for s in range(S):
        if s not in ACTIVE:
            mo[s] = mo[S + s] = x0[s] = side[s] = NAN
        elif coef[s, 4 if kind == "dpmpp_2m" else 6].item() == 0:
            side[s] = NAN   # a first-order row never reads the history, a step without noise never reads the noise
    bm, mo_v, pm, nm = _poisoned(mo.shape, mo)
    bx, x, px, nx = _poisoned(x0.shape, x0)
    bs, sd, ps, ns = _poisoned(side.shape, side)
    bc, cf, pc, nc = _poisoned(coef.shape, coef)
    bg, gv, pg, ng = _poisoned(guid.shape, guid)
    state = _state(S)
    if kind == "ddpm":
        bw, work, pw, nw = _poisoned((S, 4, H, W))
        ops.slot_sampler_step(mo_v, x, sd, cf, gv, state, work)
    else:
        ops.slot_dpm_solver_step(mo_v, x, sd, cf, gv, state)
    torch.cuda.synchronize()
    for s in range(S):
        if s not in ACTIVE:
            assert torch.isnan(x[s]).all() and torch.isnan(sd[s]).all()
            continue
        one_mo = torch.stack([mo[s], mo[S + s]]).contiguous()
        ref = x0[s:s + 1].clone()
        if kind == "ddpm":
            ops.sampler_step(one_mo, ref, side[s:s + 1].contiguous(), coef[s].contiguous(), guid[s].item(), False, clip=2.0,
                             threshold_mode=0)
            r64, scale = _ddpm64(mo, x0[s], side[s], coef[s], guid[s].item(), s, S)
        else:
            hist = side[s:s + 1].clone()
            ops.dpm_solver_step(one_mo, ref, hist, coef[s].contiguous(), guid[s].item(), False)
            r64, h64, scale = _dpm64(mo, x0[s], side[s], coef[s], guid[s].item(), s, S)
            assert torch.equal(sd[s], hist[0])
            assert ((sd[s].double() - h64).abs() <= 8 * EPS32 * scale / coef[s, 3].abs().double().clamp(min=1e-30)).all()
        torch.cuda.synchronize()
        assert torch.equal(x[s], ref[0]), (kind, s)
        assert torch.isfinite(x[s]).all()
        assert ((x[s].double() - r64).abs() <= 8 * EPS32 * scale + 1e-30).all(), (kind, s, (x[s].double() - r64).abs().max())
    assert torch.equal(state, _state(S))
    for b, p, m in ((bm, pm, nm), (bx, px, nx), (bs, ps, ns), (bc, pc, nc), (bg, pg, ng)):
        assert _outside_untouched(b, p, m)
    if kind == "ddpm":
        assert _outside_untouched(bw, pw, nw)


# ---- the batcher on the tiny 2.2 pipeline ----------------------------------------------------------------------------------
def _step(b, latents):
    """b.step(), keeping the latent each finished request handed to the decoder (pipe.seen, see sampler_cases._pipe) in
    latents[handle]."""
    pipe = b.pipe
    before = len(pipe.seen)
    done = b.step()
    for h, lat in zip(done, pipe.seen[before:]):
        latents[h] = lat
    return done


def _run(b, latents):
    out = {}
    while b.pending():
        out.update(_step(b, latents))
    return out


def _embeds(pipe, prompt):
    return pipe.embedder.image_emb(prompt, 1), pipe.embedder.zero_image_emb(1)


@pytest.mark.parametrize("sampler", SAMPLERS)
def test_request_is_isolated_from_the_other_slots(sampler):
    """A request's final latent and image are the same bits alone in the batcher (slot 0, every other slot idle) and alongside
    requests admitted at other steps, with other embeddings, guidance scales and step counts, while it sits in slot 2."""
    pipe = _pipe("2.2", "text2img")
    pos, neg = _embeds(pipe, "a red cat")
    req = dict(image_embeds=pos, negative_image_embeds=neg, decoder_steps=6, decoder_guidance_scale=4.0, seed=11)
    lat_a, lat_b = {}, {}
    alone = pipe.batcher(3, 64, 64, sampler=sampler, max_steps=12)
    h = alone.submit(**req)
    img_alone = _run(alone, lat_a)[h]
    mixed = pipe.batcher(3, 64, 64, sampler=sampler, max_steps=12)
    p2, n2 = _embeds(pipe, "a blue dog")
    mixed.submit(image_embeds=p2, negative_image_embeds=n2, decoder_steps=9, decoder_guidance_scale=7.0, seed=5)
    _step(mixed, lat_b)
    mixed.submit("a green bird", decoder_steps=4, decoder_guidance_scale=2.0, seed=7)
    _step(mixed, lat_b)
    _step(mixed, lat_b)
    h2 = mixed.submit(**req)
    out = _step(mixed, lat_b)
    assert mixed.queue.holder[2] == h2
    out.update(_run(mixed, lat_b))
    assert mixed.queue.holder == [None, None, None]
    assert torch.equal(lat_a[h], lat_b[h2]) and torch.isfinite(lat_a[h]).all()
    assert img_alone.tobytes() == out[h2].tobytes()
    assert len(lat_b) == 3 and not torch.equal(lat_b[0], lat_b[h2])


@pytest.mark.parametrize("sampler", SAMPLERS)
def test_batch_of_one_equals_generate_text2img(sampler):
    """max_batch = 1: the image and latent of a request equal generate_text2img(batch_size=1) with base_seed = the request's
    seed, bit for bit.  max_batch = 4: three requests are within the tiny-UNet loop bound of theirs."""
    pipe = _pipe("2.2", "text2img")
    kw = dict(decoder_steps=5, decoder_guidance_scale=4)
    lats = {}
    b = pipe.batcher(1, 64, 64, sampler=sampler, max_steps=8)
    h = b.submit("a red cat", seed=1234, **kw)
    got = _run(b, lats)
    pipe.base_seed = 1234
    want = pipe.generate_text2img("a red cat", batch_size=1, h=64, w=64, sampler=sampler, **kw)
    assert got[h].tobytes() == want[0].tobytes()
    assert torch.equal(lats[h], pipe.seen[-1])
    b4 = pipe.batcher(4, 64, 64, sampler=sampler, max_steps=8)
    lats4 = {}
    reqs = [("a red cat", 21, 5, 4.0), ("a blue dog", 22, 3, 6.0), ("a green bird", 23, 7, 2.5)]
    hs = [b4.submit(p, seed=sd, decoder_steps=n, decoder_guidance_scale=g) for p, sd, n, g in reqs]
    _run(b4, lats4)
    for hh, (p, sd, n, g) in zip(hs, reqs):
        pipe.base_seed = sd
        pipe.generate_text2img(p, batch_size=1, h=64, w=64, sampler=sampler, decoder_steps=n, decoder_guidance_scale=g)
        _check(lats4[hh], pipe.seen[-1], f"batcher max_batch 4 {sampler} {p}")


def test_one_step_is_one_graph_replay():
    """step() replays the batcher's one captured graph exactly once while a slot is occupied, and never otherwise; admitting
    and finishing requests keeps that graph and every buffer address it was captured on."""
    pipe = _pipe("2.2", "text2img")
    b = pipe.batcher(2, 64, 64, max_steps=8)
    g0 = b.graph
    sl = b.slots
    bufs = [sl.x, sl.state, sl.ts_tab, sl.coef_tab, sl.coef, sl.guidance, sl.noise_tab, sl.noise, sl.work, b.plan.x_in,
            b.plan.t_in, b.plan.out, b.plan.xf_proj] + list(b.plan.enc_kv.values())
    ptrs = [t.data_ptr() for t in bufs]
    calls = []
    orig = g0.replay
    g0.replay = lambda: (calls.append(1), orig())[1]
    assert b.step() == {} and not calls
    for i, n in enumerate((3, 5, 2)):
        b.submit(f"prompt {i}", decoder_steps=n, seed=i)
    steps = finished = 0
    while b.pending():
        before = len(calls)
        finished += len(b.step())
        steps += 1
        assert len(calls) == before + 1
    assert finished == 3 and steps == len(calls)
    assert b.graph is g0 and [t.data_ptr() for t in bufs] == ptrs


@pytest.mark.parametrize("sampler", ["ddpm_sampler"])
def test_full_size_isolation(sampler):
    """The isolation property at the full Kandinsky 2.2 UNet, 768 x 768 images (96 x 96 latents): a request's latent is the
    same bits alone in slot 0 and in slot 1 next to another request admitted a step earlier."""
    from kandinsky2 import get_kandinsky2
    pipe = get_kandinsky2("cuda", task_type="text2img", model_version="2.2", cache_dir="/nonexistent")
    seen = []
    orig = pipe._finish
    pipe._finish = lambda lat, h, w: (seen.append(lat.clone()), orig(lat, h, w))[1]
    pipe.seen = seen
    pos, neg = _embeds(pipe, "a red cat")
    req = dict(image_embeds=pos, negative_image_embeds=neg, decoder_steps=3, decoder_guidance_scale=4.0, seed=3)
    la, lb = {}, {}
    alone = pipe.batcher(2, 768, 768, sampler=sampler, max_steps=4)
    h = alone.submit(**req)
    _run(alone, la)
    del alone
    mixed = pipe.batcher(2, 768, 768, sampler=sampler, max_steps=4)
    p2, n2 = _embeds(pipe, "a blue dog")
    mixed.submit(image_embeds=p2, negative_image_embeds=n2, decoder_steps=4, decoder_guidance_scale=6.0, seed=9)
    _step(mixed, lb)
    h2 = mixed.submit(**req)
    _run(mixed, lb)
    assert la[h].shape == (1, 4, 96, 96) and torch.isfinite(la[h]).all()
    assert torch.equal(la[h], lb[h2])


def test_a_request_joins_at_the_next_step_and_the_host_stays_near_the_gpu():
    """A request submitted while another is mid-run holds a slot after the next step(), and after every step() every replayed
    step but the newest Batcher.RUN_AHEAD has finished on the GPU: the host cannot enqueue a request's whole run ahead of the
    device, so arrivals join the batch at the next step of the GPU's clock."""
    from kandinsky2.batching import Batcher
    pipe = _pipe("2.2", "text2img")
    b = pipe.batcher(3, 64, 64, max_steps=12)
    evs = []
    orig = b.graph.replay

    def replay():
        orig()
        ev = torch.cuda.Event()
        ev.record()
        evs.append(ev)
    b.graph.replay = replay
    h1 = b.submit("a red cat", decoder_steps=10, seed=1)
    for _ in range(3):
        b.step()
        assert all(e.query() for e in evs[:-Batcher.RUN_AHEAD])
    h2 = b.submit("a blue dog", decoder_steps=4, seed=2)
    b.step()
    assert b.queue.holder == [h1, h2, None] and b.queue.left == [6, 3, 0]
    while b.queue.busy():
        b.step()
        assert all(e.query() for e in evs[:-Batcher.RUN_AHEAD])
    assert len(evs) == 10


def test_slot_ops_refuse_operands_the_kernels_would_misread():
    """The slot wrappers raise K2Error (not an assert) on an int64 or mis-shaped state, a non-contiguous or non-fp32 operand and
    an operand of the wrong size."""
    from kandinsky2 import ops
    from kandinsky2._native import K2Error
    S, H, W, kmax = 2, 4, 4, 3
    f = lambda *s: torch.zeros(*s, device="cuda")
    state = torch.zeros(2, S, dtype=torch.int32, device="cuda")
    mo, x, coef, g, work = f(2 * S, 8, H, W), f(S, 4, H, W), f(S, 8), f(S), f(S, 4, H, W)
    with pytest.raises(K2Error, match="state"):
        ops.slot_step_end(state.long())
    with pytest.raises(K2Error, match="state"):
        ops.slot_sampler_step(mo, x, work, coef, g, torch.zeros(2, S + 1, dtype=torch.int32, device="cuda"), work)
    with pytest.raises(K2Error, match="coef"):
        ops.slot_sampler_step(mo, x, work, f(8, S).t(), g, state, work)
    with pytest.raises(K2Error, match="guidance"):
        ops.slot_dpm_solver_step(mo, x, work, coef, g.double(), state)
    with pytest.raises(K2Error, match="model_out"):
        ops.slot_dpm_solver_step(f(S, 8, H, W), x, work, coef, g, state)
    with pytest.raises(K2Error, match="coef_tab"):
        ops.slot_step_begin(x, f(2 * S, 4, H, W), f(2 * S), coef, f(S, kmax), f(S, kmax, 7), None, None, state)
    with pytest.raises(K2Error, match="noise"):
        ops.slot_step_begin(x, f(2 * S, 4, H, W), f(2 * S), coef, f(S, kmax), f(S, kmax, 8), f(S, kmax, 4, H, W), f(S, 4, H),
                            state)
