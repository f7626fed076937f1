"""GPU: the CLIP image tower (kandinsky2/model/clip_vision.py) end to end.

  - the tiny towers of tests/golden/clip_vision_tiny.pt (transformers' own outputs) within the project's per-forward bound;
  - the full ViT-bigG/14 geometry on synthetic weights, against the fp32 oracle (tests/clip_vision_oracle.py), closer than
    the oracle's own fp16 mode (the calibration of the UNet and both priors), with the fp16 residual stream's peak recorded;
  - graph replay against the eager launch list, a batch against its images one at a time, plans built over NaN-poisoned
    buffers: bit for bit;
  - the embedder wiring: PriorEmbedder22.from_diffusers(image_encoder=tower) and the pipelines that route PIL images through
    it.  The full-size tests need about 20 GB of device memory."""
import pytest
import torch

from tests import clip_vision_oracle as cvo
from tests.test_gpu_plan_poison import _Poison

pytestmark = pytest.mark.gpu


def _tower(cfg, seed, device="cuda"):
    from kandinsky2.model.clip_vision import CLIPVisionTower
    return CLIPVisionTower.from_transformers(cvo.synth_weights(cfg, seed), cfg, device=device)


def _dev(y, ref):
    return (y - ref).abs().max().item(), ((y - ref).norm() / ref.norm()).item()


@pytest.fixture(scope="module")
def bitwise():
    from kandinsky2 import launch_plan
    old = launch_plan.TUNE_SMALL_M
    launch_plan.TUNE_SMALL_M = 0     # bit-identical GEMM configurations only (as bench.py --dump-outputs)
    yield
    launch_plan.TUNE_SMALL_M = old


@pytest.fixture(scope="module")
def fx():
    return torch.load(cvo.FIXTURE)


@pytest.mark.parametrize("i", [0, 1])
def test_tiny_tower_against_transformers_golden(fx, i):
    t = fx["towers"][i]
    tower = _tower(t["cfg"], t["weight_seed"])
    hid, emb = tower.forward(cvo.tower_pixels(t).cuda())
    for got, ref, what in ((hid.float().cpu(), t["last_hidden_state"], "last_hidden_state"), (emb.cpu(), t["image_embeds"], "embeds")):
        mx, rel = _dev(got, ref)
        rms = ref.pow(2).mean().sqrt().item()
        print(f"tiny tower {i} {what}: rel-L2 {rel:.2e}, max-abs {mx / rms:.2e} RMS")
        assert rel < 2e-3 and mx < 1e-2 * rms, (what, rel, mx, rms)


def test_graph_replay_batching_and_poisoned_build(bitwise, monkeypatch):
    cfg = cvo.CONFIG_TINY
    g = torch.Generator(device="cuda").manual_seed(5)
    pix = torch.randn(4, 3, 56, 56, device="cuda", generator=g)
    tower = _tower(cfg, 7)
    h_g, e_g = tower.forward(pix, use_graph=True)
    h_e, e_e = tower.forward(pix, use_graph=False)
    assert torch.equal(h_g, h_e) and torch.equal(e_g, e_e) and torch.isfinite(e_g).all()
    assert torch.equal(tower.forward(pix)[1], e_g)                         # replayed again
    for b in range(4):
        h1, e1 = tower.forward(pix[b:b + 1])
        assert torch.equal(h1[0], h_g[b]) and torch.equal(e1[0], e_g[b]), b
    poison = _Poison(monkeypatch)
    fresh = _tower(cfg, 7)
    with poison:
        fresh._plan(4)
        fresh._plan(2)
    for use_graph in (False, True):
        h_p, e_p = fresh.forward(pix, use_graph)
        assert torch.equal(h_p, h_g) and torch.equal(e_p, e_g), use_graph


# ---------------------------------------------------------------------------------------------------------------------------
# full ViT-bigG/14 geometry, synthetic weights
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def full():
    from kandinsky2.checkpoints import transformers_clip_vision_to_k2
    from kandinsky2.model.clip_vision import CLIPVisionTower
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = cvo.CONFIG_BIGG
    sd = {k: v.cuda() for k, v in cvo.synth_weights(cfg, 21).items()}
    tower = CLIPVisionTower(transformers_clip_vision_to_k2(sd), cfg, device="cuda").finalize()
    yield cfg, sd, tower
    del sd, tower
    torch.cuda.empty_cache()


@pytest.mark.parametrize("B", [1, 4])
def test_full_size_fp16_calibration(full, B, monkeypatch):
    from kandinsky2 import ops
    cfg, sd, tower = full
    pix = torch.randn(B, 3, 224, 224, device="cuda", generator=torch.Generator(device="cuda").manual_seed(B))
    pix[0] = 0.0                                                           # the zero embedding's input
    tower._plan(B)                                                         # built (and tuned) before the GEMMs are counted
    peaks, gemm_rows = [], ops.gemm_rows

    def recording_gemm_rows(*a, **kw):
        y = gemm_rows(*a, **kw)
        if kw.get("residual") is not None:
            peaks.append(y.abs().amax())
        return y

    monkeypatch.setattr(ops, "gemm_rows", recording_gemm_rows)
    hid, emb = tower.forward(pix, use_graph=False)
    monkeypatch.undo()
    assert len(peaks) == 2 * cfg["num_hidden_layers"] + 1
    peak = torch.stack(peaks).max().item()
    assert torch.isfinite(torch.stack(peaks)).all() and torch.isfinite(emb).all(), peak
    with torch.no_grad():
        h32, e32 = cvo.forward(sd, cfg, pix)
        h16, e16 = cvo.forward(sd, cfg, pix, dtype=torch.float16)
    res = {}
    for name, got, r32, r16 in (("embeds", emb, e32, e16), ("hidden", hid.float(), h32, h16)):
        k_abs, k_rel = _dev(got, r32)
        o_abs, o_rel = _dev(r16, r32)
        res[name] = (k_abs, k_rel, o_abs, o_rel)
        print(f"CLIP ViT-bigG/14 B={B} {name}: k2 vs fp32 max-abs {k_abs:.3e} rel-L2 {k_rel:.3e} | fp16 oracle vs fp32 "
              f"max-abs {o_abs:.3e} rel-L2 {o_rel:.3e}; residual stream peak |h| {peak:.1f}")
    for name, (k_abs, k_rel, o_abs, o_rel) in res.items():
        assert k_rel <= o_rel and k_abs <= o_abs, (name, res[name])
    assert torch.equal(tower.forward(pix)[1], emb)                         # graph replay = the eager launch list


# ---------------------------------------------------------------------------------------------------------------------------
# wiring: PriorEmbedder22 and the pipelines
# ---------------------------------------------------------------------------------------------------------------------------
def _photo(w, h, seed):
    import numpy as np
    from PIL import Image
    return Image.fromarray((np.random.default_rng(seed).random((h, w, 3)) * 255).astype("uint8"))


@pytest.fixture(scope="module")
def wired(bitwise):
    """A tiny 2.2 prior (clip_dim 1280, as the decoder expects) with a tiny tower whose projection is 1280 wide."""
    from kandinsky2.model.prior import PriorEmbedder22
    from oracle import synth
    from tests import prior22_oracle as p22
    pcfg = dict(text_ctx=8, xf_width=128, xf_layers=2, xf_heads=2, xf_final_ln=True, xf_padding=False, clip_dim=1280,
                clip_xf_width=1280)
    dsd = synth.synth_state_dict(p22.diffusers_prior_spec(pcfg), seed=13)

    def clip_text(prompts):
        outs = []
        for p in prompts:
            g = torch.Generator().manual_seed(len(p) + 17 * sum(map(ord, p)))
            outs.append((torch.randn(1280, generator=g), torch.randn(8, 1280, generator=g), torch.arange(8) < 2 + len(p) % 6))
        return tuple(torch.stack(t) for t in zip(*outs))

    cfg = dict(cvo.CONFIG_TINY, image_size=224, projection_dim=1280)
    tower = _tower(cfg, 9)
    emb = PriorEmbedder22.from_diffusers(dsd, clip_text, image_encoder=tower)
    plain = PriorEmbedder22.from_diffusers(dsd, clip_text)
    return tower, emb, plain


def test_zero_image_emb_is_the_tower_on_zero_pixels(wired):
    tower, emb, plain = wired
    z = tower.image_embeds(torch.zeros(1, 3, 224, 224, device="cuda")).cpu()
    assert torch.isfinite(z).all() and z.abs().max() > 0
    assert torch.equal(emb.zero_image_emb(3), z.repeat(3, 1))
    assert torch.equal(plain.zero_image_emb(2), torch.zeros(2, 1280))
    assert plain.clip_image is None and emb.clip_image is tower


def test_emb2emb_and_interpolate_take_pil_images(wired):
    tower, emb, _ = wired
    img = _photo(300, 200, seed=4)
    kw = dict(strength=0.85, prior_steps=5)
    a = emb.emb2emb("a capybara", img, 2, **kw)
    b = emb.emb2emb("a capybara", tower(img), 2, **kw)
    assert torch.isfinite(a).all() and torch.equal(a, b)
    mix = emb.interpolate([img, "a red cat"], [0.3, 0.7], 2, prior_steps=5)
    assert mix.shape == (2, 1280) and torch.isfinite(mix).all()
    assert torch.allclose(mix, 0.3 * tower(img).repeat(2, 1) + 0.7 * emb.image_emb("a red cat", 2, prior_steps=5))


def test_controlnet_img2img_with_prior_strength_end_to_end(wired):
    from tests.test_gpu_zz_controlnet_img2img import _bytes, _pipe
    _, emb, _ = wired
    pipe = _pipe(embedder=emb)
    photo, hint = _photo(64, 64, seed=9), torch.rand(1, 3, 64, 64, generator=torch.Generator().manual_seed(10))
    kw = dict(batch_size=2, decoder_steps=4, h=64, w=64, prior_steps=5)
    a = pipe.generate_controlnet_img2img("a capybara", photo, hint, prior_strength=0.85, **kw)
    assert len(a) == 2
    assert _bytes(a) == _bytes(pipe.generate_controlnet_img2img("a capybara", photo, hint, prior_strength=0.85, **kw))
