"""GPU: truncated UnCLIP sampling and PriorEmbedder22.emb2emb (diffusers' KandinskyV22PriorEmb2EmbPipeline, restated in
tests/emb2emb_oracle.py) on the tiny diffusers-form prior and at the full 2.2 size on synthetic weights.  The full-size test
needs about 12 GB of device memory."""
import pytest
import torch

from tests import emb2emb_oracle as eo
from tests import prior22_oracle as p22
from tests.test_gpu_zz_prior22 import _cond, _dev, _prior_from_diffusers

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def tiny():
    from kandinsky2 import launch_plan
    old = launch_plan.TUNE_SMALL_M
    launch_plan.TUNE_SMALL_M = 0     # bit-identical GEMM configurations only
    cfg = p22.CONFIG_PRIOR22_TINY
    m, dsd = _prior_from_diffusers(cfg, seed=5)
    yield cfg, m, dsd
    launch_plan.TUNE_SMALL_M = old


@pytest.mark.parametrize("use_graph", [True, False])
def test_truncated_run_continues_the_full_run_bit_for_bit(tiny, use_graph):
    """N steps with x kept after N - keep of them; then keep steps from that x with the tail of the same step noise: the same
    final embedding, bit for bit."""
    from kandinsky2.model.prior import UnCLIPSchedule, sample_prior22
    cfg, m, _ = tiny
    B, D, N = 2, cfg["clip_dim"], 10
    te, tenc, mask, g = _cond(cfg, B, 4, seed=31)
    x_T = torch.randn(B, D, device="cuda", generator=g)
    noise = torch.randn(N, B, D, device="cuda", generator=g)
    mean, std = 0.1 * torch.randn(D, device="cuda", generator=g), 0.5 + torch.rand(D, device="cuda", generator=g)
    for keep in (1, 4, 9, 10):
        plan = m._step_plan(B)
        plan.bind(te, tenc, mask)
        plan.set_schedule(UnCLIPSchedule(N), x_T, noise, 4.0, use_graph)
        for _ in range(N - keep):
            plan.run(use_graph)
        x_mid = plan.x.clone()
        for _ in range(keep):
            plan.run(use_graph)
        full = plan.x * std + mean
        assert torch.equal(full, sample_prior22(m, te, tenc, mask, N, 4.0, mean, std, x_T, noise, use_graph=use_graph))
        tail = sample_prior22(m, te, tenc, mask, N, 4.0, mean, std, x_mid, noise[N - keep:], use_graph=use_graph, keep=keep)
        assert torch.isfinite(tail).all() and torch.equal(tail, full), keep


def _tiny_embedder(cfg, m, mean, std, B_max=3):
    """PriorEmbedder22 around the tiny prior, with a deterministic stand-in CLIP text tower of its width."""
    from kandinsky2.model.prior import PriorEmbedder22
    D, L, X = cfg["clip_dim"], cfg["text_ctx"], cfg["clip_xf_width"]

    def clip_text(prompts):
        outs = []
        for p in prompts:
            g = torch.Generator().manual_seed(len(p) + 17 * sum(map(ord, p)))
            outs.append((torch.randn(D, generator=g), torch.randn(L, X, generator=g), torch.arange(L) < 2 + len(p) % (L - 1)))
        return tuple(torch.stack(t) for t in zip(*outs))

    clip_image = lambda img: torch.linspace(-1, 1, D)[None] * (1 + img.size[0] % 3)  # noqa: E731
    return PriorEmbedder22(m, clip_text, mean, std, clip_image=clip_image, seed=3)


@pytest.mark.parametrize("B", [1, 3])
@pytest.mark.parametrize("guidance", [1.0, 4.0])
@pytest.mark.parametrize("strength", [0.3, 0.85, 1.0])
@pytest.mark.parametrize("N", [2, 10, 25])
def test_emb2emb_matches_the_restated_loop(tiny, N, strength, guidance, B):
    """PriorEmbedder22.emb2emb against the float64 emb2emb loop over the fp32 diffusers-form forward, with the start noise and
    step noise the embedder draws and the conditioning its text tower returns."""
    cfg, m, dsd = tiny
    D = cfg["clip_dim"]
    g = torch.Generator(device="cuda").manual_seed(N * 7 + B)
    mean, std = 0.1 * torch.randn(D, device="cuda", generator=g), 0.5 + torch.rand(D, device="cuda", generator=g)
    emb = _tiny_embedder(cfg, m, mean, std)
    image = torch.randn(1, D, device="cuda", generator=g).cpu()
    keep = eo.keep_of(N, strength)
    kw = dict(prior_steps=N, prior_guidance_scale=guidance, negative_prior_prompt="low quality")
    if keep == 0:
        with pytest.raises(ValueError, match="keeps no step"):
            emb.emb2emb("a capybara", image, B, strength=strength, **kw)
        return
    got = emb.emb2emb("a capybara", image, B, strength=strength, **kw).cuda()
    _, _, rows, gen = emb._call_args("a capybara", B, N, guidance, "low quality")
    z = torch.randn(B, D, device="cuda", generator=gen)
    noise = torch.randn(keep, B, D, device="cuda", generator=gen)
    te, tenc, mask = rows if guidance > 1.0 else (t[B:] for t in rows)

    def fn(xx, tt):
        return p22.diffusers_prior_forward(dsd, cfg, xx, tt, te, tenc, mask)
    with torch.no_grad():
        ref = eo.emb2emb_sample(fn, image.cuda().expand(B, D), z, noise, N, strength, guidance, mean, std).float()
    rel = ((got - ref).norm() / ref.norm()).item()
    print(f"tiny emb2emb N={N} strength={strength} guidance={guidance} B={B}: keep {keep}, rel-L2 {rel:.3e}")
    assert rel < 3e-2, rel   # the untruncated tiny sampling bound (tests/test_gpu_zz_prior22.py)


def test_emb2emb_inputs_determinism_and_refusals(tiny):
    from PIL import Image
    from kandinsky2._native import K2Error
    cfg, m, _ = tiny
    D = cfg["clip_dim"]
    emb = _tiny_embedder(cfg, m, torch.zeros(D, device="cuda"), torch.ones(D, device="cuda"))
    kw = dict(strength=0.85, prior_steps=10, negative_prior_prompt="ugly")
    pil = Image.new("RGB", (8, 8))
    one = emb.clip_image(pil)
    a = emb.emb2emb("a capybara", one, 3, **kw)
    assert a.shape == (3, D) and torch.isfinite(a).all() and not torch.equal(a[0], a[1])   # each row its own sample
    assert torch.equal(a, emb.emb2emb("a capybara", one.repeat(3, 1), 3, **kw))           # [B, D] as it is
    assert torch.equal(a, emb.emb2emb("a capybara", pil, 3, **kw))                        # PIL through clip_image
    assert torch.equal(a, emb.emb2emb("a capybara", one, 3, **kw))                        # deterministic
    assert not torch.equal(a, emb.emb2emb("a capybara", one * 2, 3, **kw))                # the image steers it
    assert not torch.equal(a, emb.emb2emb("a capybara", one, 3, **dict(kw, strength=0.5)))
    assert not torch.equal(a, emb.emb2emb("a capybara", Image.new("RGB", (9, 8)), 3, **kw))
    for bad in (dict(kw, strength=1.2), dict(kw, strength=-0.5), dict(kw, strength=0.05), dict(kw, prior_steps=1)):
        with pytest.raises(ValueError):
            emb.emb2emb("a capybara", one, 3, **bad)
    with pytest.raises(ValueError, match="image embedding"):
        emb.emb2emb("a capybara", one.repeat(2, 1), 3, **kw)
    emb.clip_image = None
    with pytest.raises(K2Error, match="clip_image"):
        emb.emb2emb("a capybara", pil, 3, **kw)


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


@pytest.mark.parametrize("B", [1, 4])
def test_full_size_emb2emb(full, B):
    """25 steps at strength 0.85 (the last 21 run) and guidance 4, one graph replay per step, from the noised image
    embedding, against the float64 emb2emb loop over the fp32 oracle."""
    from kandinsky2.model.prior import UnCLIPSchedule, sample_prior22
    cfg, m, dsd = full
    D, N, strength = cfg["clip_dim"], 25, 0.85
    keep = eo.keep_of(N, strength)
    te, tenc, mask, g = _cond(cfg, B, 12, seed=40 + B)
    image = torch.randn(1, D, device="cuda", generator=g).expand(B, D)
    z = torch.randn(B, D, device="cuda", generator=g)
    noise = torch.randn(keep, B, D, device="cuda", generator=g)
    mean, std = 0.1 * torch.randn(D, device="cuda", generator=g), 0.5 + torch.rand(D, device="cuda", generator=g)
    x = UnCLIPSchedule(N, keep=keep).start_latent(image, z)
    s = sample_prior22(m, te, tenc, mask, N, 4.0, mean, std, x, noise, keep=keep)
    with torch.no_grad():
        ref = eo.emb2emb_sample(lambda xx, tt: p22.diffusers_prior_forward(dsd, cfg, xx, tt, te, tenc, mask), image, z, noise,
                                N, strength, 4.0, mean, std).float()
    err, rel = _dev(s, ref)
    print(f"2.2 emb2emb full size B={B}, {keep} of {N} steps, guidance 4: rel-L2 {rel:.3e} max-abs {err:.3e}")
    assert torch.isfinite(s).all() and rel < 1e-2, rel
