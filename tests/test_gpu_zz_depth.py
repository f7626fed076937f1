"""GPU: the DPT depth estimator (kandinsky2/model/depth.py) end to end, and the ControlNet pipelines with a PIL hint.

  - the tiny estimators of tests/golden/dpt_tiny.pt (transformers' outputs; the even and the odd patch grid);
  - the Intel/dpt-large geometry on synthetic weights, B = 1 and 4, against the fp32 oracle (tests/dpt_oracle.py):
    predicted_depth rel-L2 at most the oracle's own fp16 mode's, max-abs within 1.5 times its (the rule of the CLIP and XLM-R
    towers), and the uint8 depth images within one level of the oracle's on at least 99.9 % of the pixels;
  - graph replay against the eager launch list, a batch against its images run alone, plans built over NaN-poisoned buffers
    (with the tuner restricted to bit-identical configurations): bit for bit;
  - generate_controlnet / generate_controlnet_img2img with a PIL hint and a tiny estimator against make_hint by hand, bit
    for bit, and the refusal of a PIL hint without an estimator."""
import numpy as np
import pytest
import torch

from tests import dpt_oracle as do
from tests.test_gpu_plan_poison import _Poison

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fx():
    return torch.load(do.FIXTURE)


@pytest.fixture(scope="module")
def bitwise():
    from kandinsky2 import launch_plan
    old = launch_plan.TUNE_SMALL_M
    launch_plan.TUNE_SMALL_M = 0     # bit-identical GEMM configurations only (as bench.py --dump-outputs)
    yield
    launch_plan.TUNE_SMALL_M = old


def _estimator(cfg, proc, seed):
    from kandinsky2.model.depth import DPTDepthEstimator
    return DPTDepthEstimator.from_transformers(do.synth_weights(cfg, seed), cfg, proc)


def _dev(y, ref):
    return (y - ref).abs().max().item(), ((y - ref).norm() / ref.norm()).item()


@pytest.mark.parametrize("name", ["even", "odd"])
def test_tiny_estimators_against_transformers_golden(fx, name):
    g = fx["configs"][name]
    est = _estimator(g["config"], g["preprocessor"], fx["weight_seed"])
    got = est.predicted_depth(g["pixel_values"].cuda()).cpu()
    ref = g["predicted_depth"]
    assert got.shape == ref.shape
    mx, rel = _dev(got, ref)
    rms = ref.pow(2).mean().sqrt().item()
    print(f"tiny DPT {name}: rel-L2 {rel:.2e}, max-abs {mx / rms:.2e} RMS")
    assert rel < 5e-3 and mx < 3e-2 * rms, (rel, mx, rms)
    images = [img for _, img in do.sample_images(fx["image_seed"])]
    assert (est.preprocess(images) - g["pixel_values"]).abs().max().item() <= 1e-6
    for img, u8, d in zip(images, g["depth_u8"], est.depth(images)):
        diff = (torch.from_numpy(np.array(d)).int() - u8.int()).abs()
        assert d.size == img.size and d.mode == "L"
        print(f"  depth image {img.size}: {(diff > 1).float().mean().item():.4f} of the pixels more than one level off")
        assert (diff <= 1).float().mean().item() >= 0.99


def test_graph_replay_batching_and_poisoned_build(fx, bitwise, monkeypatch):
    for name in ("even", "odd"):
        g = fx["configs"][name]
        est = _estimator(g["config"], g["preprocessor"], 7)
        pix = g["pixel_values"].cuda()
        d_g = est.predicted_depth(pix)
        d_e = est.predicted_depth(pix, use_graph=False)
        assert torch.equal(d_g, d_e) and torch.isfinite(d_g).all() and (d_g > 0).float().mean() > 0.5
        assert torch.equal(est.predicted_depth(pix), d_g)                          # replayed again
        for b in range(pix.shape[0]):
            assert torch.equal(est.predicted_depth(pix[b:b + 1])[0], d_g[b]), (name, b)
        fresh = _estimator(g["config"], g["preprocessor"], 7)
        with _Poison(monkeypatch):
            fresh._plan(pix.shape[0])
        for use_graph in (False, True):
            assert torch.equal(fresh.predicted_depth(pix, use_graph), d_g), (name, use_graph)


# ---------------------------------------------------------------------------------------------------------------------------
# Intel/dpt-large geometry, synthetic weights
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def large():
    from kandinsky2.model.depth import DPTDepthEstimator
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    sd = do.synth_weights(do.CFG_LARGE, 31)
    est = DPTDepthEstimator.from_transformers(sd, do.CFG_LARGE)
    yield {k: v.cuda() for k, v in sd.items()}, est
    torch.cuda.empty_cache()


@pytest.mark.parametrize("B", [1, 4])
def test_large_geometry_fp16_calibration(large, B):
    from kandinsky2.model.depth import depth_image
    sd, est = large
    pix = torch.rand(B, 3, 384, 384, device="cuda", generator=torch.Generator(device="cuda").manual_seed(B)) * 2 - 1
    got = est.predicted_depth(pix, use_graph=False)
    assert got.shape == (B, 384, 384) and torch.isfinite(got).all()
    r32 = do.forward(sd, do.CFG_LARGE, pix)
    r16 = do.forward(sd, do.CFG_LARGE, pix, dtype=torch.float16)
    k_abs, k_rel = _dev(got, r32)
    o_abs, o_rel = _dev(r16, r32)
    pos = (r32 > 0).float().mean().item()
    print(f"DPT-large B={B}: k2 vs fp32 max-abs {k_abs:.3e} rel-L2 {k_rel:.3e} | fp16 oracle vs fp32 max-abs {o_abs:.3e} "
          f"rel-L2 {o_rel:.3e} | positive {pos:.3f}")
    assert pos > 0.5
    assert k_rel <= o_rel and k_abs <= 1.5 * o_abs, (k_abs, k_rel, o_abs, o_rel)
    near = []
    for b in range(B):
        a = torch.from_numpy(np.array(depth_image(got[b].cpu(), 480, 640))).int()
        r = torch.from_numpy(np.array(depth_image(r32[b].cpu(), 480, 640))).int()
        near.append(((a - r).abs() <= 1).float().mean().item())
    print(f"  uint8 depth within one level: {min(near):.5f}")
    assert min(near) >= 0.999
    assert torch.equal(est.predicted_depth(pix), got)                              # graph replay = the eager launch list


# ---------------------------------------------------------------------------------------------------------------------------
# the ControlNet pipelines with a PIL hint
# ---------------------------------------------------------------------------------------------------------------------------
def _pipe(depth_estimator):
    import copy

    from kandinsky2.configs import CONFIG_2_2
    from kandinsky2.pipelines import Kandinsky2_2
    from tests.test_gpu_movq_sampler import _tiny_overrides
    config = copy.deepcopy(CONFIG_2_2)
    for k, v in _tiny_overrides().items():
        config[k].update(v)
    return Kandinsky2_2(config, "cuda", task_type="controlnet", depth_estimator=depth_estimator)


def _photo(w, h, seed):
    from PIL import Image
    return Image.fromarray((np.random.default_rng(seed).random((h, w, 3)) * 255).astype("uint8"))


def test_pil_hint_equals_make_hint_by_hand(fx, bitwise):
    from kandinsky2.model.depth import make_hint
    g = fx["configs"]["even"]
    est = _estimator(g["config"], g["preprocessor"], 3)
    pipe = _pipe(est)
    photo, scene = _photo(100, 70, 1), _photo(90, 60, 2)
    hint = make_hint(scene, est)
    assert hint.shape == (3, 60, 90) and 0 <= hint.min() and hint.max() <= 1 and hint.max() > hint.min()
    kw = dict(batch_size=2, decoder_steps=3, h=64, w=64)
    a = pipe.generate_controlnet("a capybara", scene, **kw)
    b = pipe.generate_controlnet("a capybara", hint[None], **kw)
    assert [x.tobytes() for x in a] == [x.tobytes() for x in b]
    c = pipe.generate_controlnet_img2img("a capybara", photo, scene, strength=0.5, **kw)
    d = pipe.generate_controlnet_img2img("a capybara", photo, hint, strength=0.5, **kw)
    assert [x.tobytes() for x in c] == [x.tobytes() for x in d]
    with pytest.raises(ValueError, match="depth_estimator="):
        _pipe(None).generate_controlnet("a capybara", scene, **kw)
    with pytest.raises(ValueError, match="depth_estimator="):
        _pipe(None).generate_controlnet_img2img("a capybara", photo, scene, **kw)
