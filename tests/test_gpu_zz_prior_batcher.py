"""GPU: the Kandinsky 2.2 prior in continuously refilled slots (kandinsky2/batching.py, PriorBatcher) -- bit for bit against
PriorEmbedder22.image_emb / emb2emb at batch 1, a request's bits in any slot next to any other requests, idle slots poisoned
with NaN, both tuner settings, the weights-changed refusal, the full 2.2 prior geometry, and the decoder batcher fed by
prior slots against the one that runs the prior at submit.  The full-size tests need about 10 GB of device memory."""
import pytest
import torch

from tests import prior22_oracle as p22
from tests.test_gpu_batcher_img2img import _hint, _photo
from tests.test_gpu_batcher_lora import _lora
from tests.test_gpu_zz_emb2emb import _tiny_embedder
from tests.test_gpu_zz_prior22 import _prior_from_diffusers

pytestmark = pytest.mark.gpu

NAN = float("nan")


@pytest.fixture
def exact(monkeypatch):
    from kandinsky2 import launch_plan
    monkeypatch.setattr(launch_plan, "TUNE_SMALL_M", 0)   # bit-identical GEMM configurations only


@pytest.fixture(scope="module")
def tiny():
    cfg = p22.CONFIG_PRIOR22_TINY
    m, _ = _prior_from_diffusers(cfg, seed=5)
    D = cfg["clip_dim"]
    g = torch.Generator(device="cuda").manual_seed(9)
    mean, std = 0.1 * torch.randn(D, device="cuda", generator=g), 0.5 + torch.rand(D, device="cuda", generator=g)
    return cfg, _tiny_embedder(cfg, m, mean, std)


def _alone(emb, S, req):
    pb = emb.batcher(S)
    h = pb.submit(*req[0], **req[1])
    return pb.run()[h]


def _want(emb, req):
    """What the batch-1 call of the embedder computes for a request (prompt, [image]), kw."""
    args, kw = req
    kw = dict(kw)
    if "image" in kw:
        image = kw.pop("image")
        return emb.emb2emb(args[0], image, 1, **kw)
    return emb.image_emb(args[0], 1, **kw)


def _mixed(D):
    from PIL import Image
    vec = torch.linspace(-2, 1, D)[None]
    return [
        (("a red cat",), dict(prior_steps=10, prior_guidance_scale=4, negative_prior_prompt="ugly")),
        (("a blue dog",), dict(prior_steps=25, prior_guidance_scale=1)),
        (("a green bird",), dict(prior_steps=2, prior_guidance_scale=4)),
        (("an owl",), dict(prior_steps=25, prior_guidance_scale=4, image=vec, strength=0.85)),
        (("a fox",), dict(prior_steps=10, prior_guidance_scale=1, image=Image.new("RGB", (9, 8)), strength=0.3)),
        (("a grey wolf",), dict(prior_steps=10, prior_guidance_scale=6, image=vec[0], strength=1.0)),
    ]


def test_max_batch_1_equals_image_emb_and_emb2emb(tiny, exact):
    """One slot, reused request after request: each result, copied to the host, is image_emb(prompt, 1, ...) or
    emb2emb(prompt, image, 1, strength, ...) bit for bit -- 2 / 10 / 25 steps, guidance 4 and 1 (unguided), a negative prior
    prompt, and emb2emb at strength 0.3 / 0.85 / 1 from a tensor and from a PIL image."""
    from PIL import Image
    cfg, emb = tiny
    D = cfg["clip_dim"]
    emb.prior._step_plans.clear()   # image_emb's plan tuned as this test's batcher is
    pb = emb.batcher(1)
    reqs = [(("a red cat",), dict(prior_steps=n, prior_guidance_scale=g, negative_prior_prompt=neg))
            for n in (2, 10, 25) for g in (4.0, 1.0) for neg in ("", "low quality")]
    reqs += [(("a red cat",), dict(prior_steps=n, image=im, strength=st, negative_prior_prompt="ugly"))
             for n in (10, 25) for st in (0.3, 0.85, 1.0) for im in (torch.linspace(-1, 2, D)[None], Image.new("RGB", (8, 8)))]
    for req in reqs:
        h = pb.submit(*req[0], **req[1])
        out = pb.run()
        assert list(out) == [h]
        got = out[h]
        assert got.is_cuda and got.dtype == torch.float32 and got.shape == (1, D)
        want = _want(emb, req)
        assert torch.isfinite(want).all() and torch.equal(got.cpu(), want), req


def _isolation(emb, D, req):
    """(result of req alone in slot 0 of 4, result of req admitted into slot 2 beside requests with other prompts, step
    counts, guidance and emb2emb, with an image_emb call between the steps)."""
    alone = _alone(emb, 4, req)
    pb = emb.batcher(4)
    others = _mixed(D)
    got = {}
    hs = [pb.submit(*others[0][0], **others[0][1])]
    got.update(pb.step())
    hs.append(pb.submit(*others[3][0], **others[3][1]))
    got.update(pb.step())
    h = pb.submit(*req[0], **req[1])
    got.update(pb.step())
    assert pb.queue.holder[2] == h
    hs.append(pb.submit(*others[2][0], **others[2][1]))
    while pb.pending():
        emb.image_emb("an interleaved call", 1, prior_steps=3)   # the embedder's own batch-1 plan: no row of this batch
        got.update(pb.step())
    assert len(got) == 4 and pb.queue.holder == [None] * 4
    return alone, got[h], {hh: got[hh] for hh in hs}


def test_a_request_has_the_same_bits_in_any_slot(tiny):
    cfg, emb = tiny
    D = cfg["clip_dim"]
    for req in (_mixed(D)[1], _mixed(D)[4]):
        a, b, _ = _isolation(emb, D, req)
        assert torch.isfinite(a).all() and torch.equal(a, b), req


def test_idle_slots_poisoned_with_nan_do_not_reach_active_slots(tiny):
    cfg, emb = tiny
    D = cfg["clip_dim"]
    req = _mixed(D)[0]
    clean = _alone(emb, 4, req)
    pb = emb.batcher(4)
    p, sl = pb.plan, pb.slots
    h = pb.submit(*req[0], **req[1])
    got = pb.step()
    S = 4
    for s in range(1, S):
        for t in (sl.x[s], sl.noise[s], sl.work[s], p.model_out[s], p.model_out[S + s], sl.noise_tab[s], sl.ts_tab[s],
                  sl.coef_tab[s]):
            t.fill_(NAN)
    while pb.pending():
        got.update(pb.step())
    assert torch.isfinite(got[h]).all() and torch.equal(got[h], clean)


def test_every_request_of_a_mixed_batch_equals_the_batch_1_call(tiny, exact):
    """Under TUNE_SMALL_M = 0 the GEMMs at 2S rows sum as at 2 rows: every request of a full, refilled batch equals its
    batch-1 call bit for bit."""
    cfg, emb = tiny
    D = cfg["clip_dim"]
    emb.prior._step_plans.clear()
    reqs = _mixed(D)
    pb = emb.batcher(4)
    hs = [pb.submit(*r[0], **r[1]) for r in reqs]
    out = pb.run()
    assert sorted(out) == hs
    for h, r in zip(hs, reqs):
        assert torch.equal(out[h].cpu(), _want(emb, r)), r


def test_the_default_tuner_and_one_replay_per_step(tiny):
    """Under the default tuner too every request equals its batch-1 call bit for bit: the slot plan's GEMMs take the N tile
    and split-K factor the tuner caches for the 2-row shape.  One step() is one graph replay on buffers that never move."""
    cfg, emb = tiny
    D = cfg["clip_dim"]
    emb.prior._step_plans.clear()
    reqs = _mixed(D)
    pb = emb.batcher(4)
    calls, orig = [], pb.graph.replay
    pb.graph.replay = lambda: (calls.append(1), orig())[1]
    p, sl = pb.plan, pb.slots
    bufs = lambda: [t.data_ptr() for t in (sl.x, sl.state, sl.ts_tab, sl.coef_tab, sl.noise_tab, sl.guidance,  # noqa: E731
                                           p.seq, p.keep, p.model_out)]
    ptrs = bufs()
    hs = [pb.submit(*r[0], **r[1]) for r in reqs]
    out, steps = {}, 0
    while pb.pending():
        out.update(pb.step())
        steps += 1
    assert len(calls) == steps and ptrs == bufs()
    for h, r in zip(hs, reqs):
        assert torch.equal(out[h].cpu(), _want(emb, r)), r


def test_a_reloaded_or_adapted_prior_is_refused(tiny):
    """step() refuses once the prior's packed weights change: a reload, load_lora, and unload_lora after a batcher made with
    an adapter loaded."""
    from kandinsky2._native import K2Error
    from tests import prior_lora_oracle as plo
    cfg, emb = tiny
    m = emb.prior
    lora = plo.synth_prior_lora(cfg, rank=4, seed=2)

    def refused(change):
        pb = emb.batcher(2)
        pb.submit("a red cat", prior_steps=3)
        pb.step()
        change()
        with pytest.raises(K2Error, match="packed weights changed"):
            pb.step()

    refused(m.finalize)                     # a reload re-packs the weights
    refused(lambda: m.load_lora(lora))      # merged in place
    refused(lambda: m.load_lora(lora, 0.5))  # a new scale is a new merge
    refused(m.unload_lora)
    assert m._lora is None


# ---------------------------------------------------------------------------------------------------------------------------
# full 2.2 prior geometry, synthetic weights
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def full():
    cfg = p22.CONFIG_PRIOR22
    m, dsd = _prior_from_diffusers(cfg, seed=11, round_gemm=True)
    del dsd
    torch.cuda.empty_cache()
    D = cfg["clip_dim"]
    g = torch.Generator(device="cuda").manual_seed(3)
    mean, std = 0.1 * torch.randn(D, device="cuda", generator=g), 0.5 + torch.rand(D, device="cuda", generator=g)
    yield cfg, _tiny_embedder(cfg, m, mean, std)
    del m
    torch.cuda.empty_cache()


def test_full_size_request_alone_and_beside_three_others(full):
    """25 steps at guidance 4 at the released geometry, where the GEMM library's cycle model splits K by row count (8 x 81
    rows otherwise than 2 x 81): alone in slot 0 and in slot 2 beside requests of other lengths, guidance and emb2emb, the
    request has the bits of image_emb(prompt, 1), under TUNE_SMALL_M = 0 and under the default tuner."""
    from kandinsky2 import launch_plan
    cfg, emb = full
    D = cfg["clip_dim"]
    req = (("a red cat",), dict(prior_steps=25, prior_guidance_scale=4, negative_prior_prompt="ugly"))
    old = launch_plan.TUNE_SMALL_M
    try:
        for small_m in (0, old):
            launch_plan.TUNE_SMALL_M = small_m
            emb.prior._step_plans.clear()
            a, b, _ = _isolation(emb, D, req)
            assert torch.isfinite(a).all() and torch.equal(a, b), small_m
            assert torch.equal(a.cpu(), _want(emb, req)), small_m
    finally:
        launch_plan.TUNE_SMALL_M = old
        emb.prior._step_plans.clear()


# ---------------------------------------------------------------------------------------------------------------------------
# the decoder batcher fed by prior slots
# ---------------------------------------------------------------------------------------------------------------------------
def _prior_pipe(task):
    from kandinsky2.model.prior import PriorEmbedder22
    from oracle import synth
    from tests.test_gpu_zz_controlnet_img2img import _pipe as _cn_pipe
    cfg = dict(text_ctx=8, xf_width=128, xf_layers=2, xf_heads=2, xf_final_ln=True, xf_padding=False, clip_dim=1280,
               clip_xf_width=1280)
    dsd = synth.synth_state_dict(p22.diffusers_prior_spec(cfg), seed=13)

    def clip_text(prompts):
        outs = []
        for p in prompts:
            g = torch.Generator().manual_seed(len(p) + 17 * sum(map(ord, p)))
            outs.append((torch.randn(1280, generator=g), torch.randn(8, 1280, generator=g), torch.arange(8) < 2 + len(p) % 6))
        return tuple(torch.stack(t) for t in zip(*outs))
    clip_image = lambda img: torch.full((1, 1280), 0.25 + img.size[0] / 1000)  # noqa: E731
    emb = PriorEmbedder22.from_diffusers(dsd, clip_text, clip_image=clip_image, zero_image_emb=torch.full((1280,), -0.5))
    return _cn_pipe(task, embedder=emb)


def _serve(pipe, P, reqs, lora):
    b = pipe.batcher(2, 64, 64, max_steps=6, max_loras=1, prior_slots=P)
    b.add_lora("A", lora, 0.8)
    if P:
        emb = pipe.embedder

        def boom(*a, **k):
            raise AssertionError("a submit on a batcher with prior slots ran the prior")
        emb.image_emb = emb.emb2emb = boom
        try:
            hs = [b.submit(**r) for r in reqs]
        finally:
            del emb.image_emb, emb.emb2emb
        assert b.prior.plan.S == P
    else:
        hs = [b.submit(**r) for r in reqs]
    out = b.run()
    assert sorted(out) == hs and not b._held
    return [out[h].tobytes() for h in hs]


@pytest.mark.parametrize("task", ["text2img", "controlnet"])
def test_prior_slots_serve_the_images_of_prior_calls_at_submit(task, exact):
    """prior_slots = 1 and 3 against prior_slots = 0 on the tiny UNet and a tiny prior: the same images, bit for bit, for
    text2img with and without a decoder negative prompt, img2img, a LoRA adapter request and, on ControlNet, requests with
    and without prior_strength.  No submit calls the embedder's image_emb or emb2emb."""
    pipe = _prior_pipe(task)
    photo = _photo(64, 64, 9)
    base = dict(decoder_steps=4, prior_steps=5, negative_prior_prompt="ugly")
    if task == "controlnet":
        base["hint"] = _hint(64, 64, 10)
    reqs = [dict(base, prompt="a capybara", seed=1),
            dict(base, prompt="a red cat", negative_decoder_prompt="lowres", seed=2, prior_steps=3),
            dict(base, prompt="a blue dog", image=photo, strength=0.5, seed=3, prior_guidance_scale=1),
            dict(base, prompt="a green bird", lora="A", seed=4, negative_decoder_prompt="blurry")]
    if task == "controlnet":
        reqs += [dict(base, prompt="an owl", image=photo, strength=0.5, prior_strength=0.85, seed=5),
                 dict(base, prompt="a fox", image=photo, strength=1.0, prior_strength=0.6, negative_decoder_prompt="lowres",
                      seed=6)]
    lora = _lora(pipe.model, 4, 41)
    want = _serve(pipe, 0, reqs, lora)
    assert len(set(want)) == len(want)
    for P in (1, 3):
        assert _serve(pipe, P, reqs, lora) == want, P
