"""GPU: the hybrid DPT depth estimator (MiDaS v3 DPT-Hybrid, kandinsky2/model/depth.py) end to end, and midas_hint.

  - the tiny estimator of tests/golden/dpt_hybrid_tiny.pt (transformers' outputs) at 64 x 64, 128 x 128, 64 x 96 and 80 x 80:
    rel-L2 < 5e-3 and max-abs < 3e-2 RMS (the plain DPT test's bounds);
  - the Intel/dpt-hybrid-midas geometry on synthetic weights against the fp32 oracle (tests/dpt_hybrid_oracle.py) at 384 x 384
    (B = 1, 4), 512 x 512 and 512 x 768: rel-L2 at most the oracle's fp16 mode's, max-abs within 1.5 times its, and at least as
    many uint8 depth pixels within one level of the fp32 oracle's as the fp16 mode has (with synthetic weights the map's
    min-max range is small against its mean, so neither fp16 path reaches 99.9 %); the peak |activation| of the fp16 BiT stages and residual stream;
  - graph replay against the eager list, plans built over NaN-poisoned buffers, and PDL (tuning key 4) on and off, eagerly
    and as a graph: bit for bit; a batch against its images alone within rel-L2 5e-3 (the golden bound) (not bit for bit: k2_conv_gemm picks
    split-K and its GroupNorm partial layout from the row count, so the fp32 summation order depends on the batch);
  - midas_hint fed through generate_controlnet_img2img against the same hint built by hand."""
import numpy as np
import pytest
import torch

from tests import dpt_hybrid_oracle as ho
from tests.test_gpu_plan_poison import _Poison
from tests.test_gpu_zz_depth import _photo, _pipe

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fx():
    return torch.load(ho.FIXTURE)


@pytest.fixture(scope="module")
def bitwise():
    from kandinsky2 import launch_plan
    old = launch_plan.TUNE_SMALL_M
    launch_plan.TUNE_SMALL_M = 0
    yield
    launch_plan.TUNE_SMALL_M = old


def _estimator(cfg, seed):
    from kandinsky2.model.depth import DPTDepthEstimator
    return DPTDepthEstimator.from_transformers(ho.synth_weights(cfg, seed), cfg)


def _dev(y, ref):
    return (y - ref).abs().max().item(), ((y - ref).norm() / ref.norm()).item()


def test_tiny_against_transformers_golden(fx):
    est = _estimator(fx["config"], fx["weight_seed"])
    for (h, w), g in fx["sizes"].items():
        got = est.predicted_depth(ho.fixture_pixels(g).cuda()).cpu()
        ref = g["predicted_depth"]
        assert got.shape == ref.shape, ((h, w), got.shape, ref.shape)
        mx, rel = _dev(got, ref)
        rms = ref.pow(2).mean().sqrt().item()
        plan = est._plan(1, h, w)
        for i, (m, r) in enumerate(zip(plan.bit_maps[:2], g["bit_channel_means"][:2])):   # where a mismatch starts
            mr = ((m.float().cpu().mean((0, 1, 2)) - r).norm() / r.norm()).item()
            print(f"  {h} x {w} BiT stage {i + 1} channel means rel-L2 {mr:.2e}")
        for i, (m, r) in enumerate(zip(plan.bit_maps[:2], g.get("bit_maps", [])[:2])):
            mr = ((m.float().cpu().permute(0, 3, 1, 2) - r.float()).norm() / r.float().norm()).item()
            print(f"  {h} x {w} BiT stage {i + 1} rel-L2 {mr:.2e}")
        print(f"tiny DPT-Hybrid {h} x {w}: rel-L2 {rel:.2e}, max-abs {mx / rms:.2e} RMS")
        assert rel < 5e-3 and mx < 3e-2 * rms, ((h, w), rel, mx, rms)


def test_bit_identities(fx, bitwise, monkeypatch):
    from kandinsky2 import ops
    cfg = fx["config"]
    est = _estimator(cfg, 7)
    for h, w in ((64, 96), (80, 80)):
        pix = ho.sample_pixels(h, w, seed=h + w, B=3).cuda()
        d_g = est.predicted_depth(pix)
        d_e = est.predicted_depth(pix, use_graph=False)
        assert torch.equal(d_g, d_e) and torch.isfinite(d_g).all() and (d_g > 0).float().mean() > 0.2
        assert torch.equal(est.predicted_depth(pix), d_g)
        for b in range(pix.shape[0]):   # the library's split-K choice depends on the batch: equal to fp32 summation order
            alone = est.predicted_depth(pix[b:b + 1])[0]
            rel = ((alone - d_g[b]).norm() / d_g[b].norm()).item()
            print(f"  {h} x {w} image {b}: batch vs alone rel-L2 {rel:.2e}")
            assert rel < 5e-3, ((h, w), b, rel)
        fresh = _estimator(cfg, 7)
        with _Poison(monkeypatch):
            fresh._plan(pix.shape[0], h, w)
        for use_graph in (False, True):
            assert torch.equal(fresh.predicted_depth(pix, use_graph), d_g), ((h, w), use_graph)
        try:
            ops.set_tuning(4, 1)
            pdl = _estimator(cfg, 7)
            assert torch.equal(pdl.predicted_depth(pix, use_graph=False), d_g)
            assert torch.equal(pdl.predicted_depth(pix), d_g)
        finally:
            ops.set_tuning(4, 0)


# ---------------------------------------------------------------------------------------------------------------------------
# Intel/dpt-hybrid-midas geometry, synthetic weights
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def real():
    from kandinsky2.model.depth import DPTDepthEstimator
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    sd = ho.synth_weights(ho.CFG_HYBRID, 31, last_bias=ho.REAL_LAST_BIAS)
    est = DPTDepthEstimator.from_transformers(sd, ho.CFG_HYBRID)
    yield {k: v.cuda() for k, v in sd.items()}, est
    torch.cuda.empty_cache()


@pytest.mark.parametrize("B,h,w", [(1, 384, 384), (4, 384, 384), (1, 512, 512), (1, 512, 768)])
def test_real_geometry_fp16_calibration(real, B, h, w):
    from kandinsky2.model.depth import midas_depth_u8
    sd, est = real
    pix = ho.sample_pixels(h, w, seed=B * h + w, B=B).cuda()
    got = est.predicted_depth(pix, use_graph=False)
    assert got.shape == (B, h, w) and torch.isfinite(got).all()
    r32 = ho.forward(sd, ho.CFG_HYBRID, pix)
    r16, maps16 = ho.forward(sd, ho.CFG_HYBRID, pix, dtype=torch.float16, with_maps=True)
    k_abs, k_rel = _dev(got, r32)
    o_abs, o_rel = _dev(r16, r32)
    plan = est._plan(B, h, w)
    peak_bit = max(m.abs().max().item() for m in plan.bit_maps[:2])
    peak_res = max(t.float().abs().max().item() for t in plan.vit_hidden)
    print(f"DPT-Hybrid B={B} {h}x{w}: k2 vs fp32 max-abs {k_abs:.3e} rel-L2 {k_rel:.3e} | fp16 oracle vs fp32 max-abs "
          f"{o_abs:.3e} rel-L2 {o_rel:.3e} | positive {(r32 > 0).float().mean().item():.3f} | peak |BiT| {peak_bit:.1f} "
          f"(fp16 oracle {max(m.abs().max().item() for m in maps16):.1f}), peak |residual stream| {peak_res:.1f}")
    assert np.isfinite(peak_bit) and np.isfinite(peak_res)
    assert k_rel <= o_rel and k_abs <= 1.5 * o_abs, (k_abs, k_rel, o_abs, o_rel)
    def near(a):   # the share of uint8 depth pixels within one level of the fp32 oracle's, worst image
        return min((np.abs(midas_depth_u8(a[b].cpu().numpy()).astype(int) - midas_depth_u8(r32[b].cpu().numpy()).astype(int))
                    <= 1).mean() for b in range(B))
    k_near, o_near = near(got), near(r16)
    print(f"  uint8 depth within one level: k2 {k_near:.5f}, fp16 oracle {o_near:.5f}")
    assert k_near >= o_near, (k_near, o_near)
    assert torch.equal(est.predicted_depth(pix), got)


def test_midas_hint_through_controlnet_img2img(fx, bitwise):
    from kandinsky2.model.depth import hwc3, midas_depth_u8, midas_hint, midas_pixels
    est = _estimator(fx["config"], 3)
    scene = _photo(128, 192, 4)
    hint = midas_hint(scene, est)
    img = np.array(scene)                                   # 192 x 128: already at resize_image's size
    d = est.predicted_depth(midas_pixels(img).cuda())[0].cpu().numpy()
    by_hand = torch.from_numpy(hwc3(midas_depth_u8(d)).copy()).float().div(255.0).permute(2, 0, 1)
    assert torch.equal(hint, by_hand) and hint.shape == (3, 192, 128) and hint.max() > hint.min()
    pipe = _pipe(est)
    photo = _photo(100, 70, 1)
    kw = dict(batch_size=1, decoder_steps=3, h=64, w=64)
    a = pipe.generate_controlnet_img2img("a capybara", photo, hint=midas_hint(scene, est), strength=0.5, **kw)
    b = pipe.generate_controlnet_img2img("a capybara", photo, hint=by_hand, strength=0.5, **kw)
    assert [x.tobytes() for x in a] == [x.tobytes() for x in b]
