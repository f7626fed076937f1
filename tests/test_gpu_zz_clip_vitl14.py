"""GPU: the Kandinsky 2.1 CLIP ViT-L/14 towers (kandinsky2/model/clip_vitl14.py) end to end.

  - the tiny towers of tests/golden/openai_clip_tiny.pt (transformers' CLIPModel with quick_gelu and argmax pooling);
  - the full ViT-L/14 geometry on synthetic weights against the fp32 oracle (tests/openai_clip_oracle.py): rel-L2 at most
    the oracle's own fp16 mode's, max-abs within 1.5 times its (the bars of the bigG towers and XLM-R);
  - graph replay against the eager launch list, a batch against its rows one at a time, plans built over NaN-poisoned
    buffers: bit for bit;
  - PriorEmbedder.from_pretrained on a tiny 2.1 folder (prior, CLIP, BPE, M-CLIP, stats) driving Kandinsky2_1's
    generate_text2img and mix_images with a PIL image, against the same pieces composed by hand, and its refusals."""
import json
import os

import pytest
import torch

from tests import openai_clip_oracle as oo
from tests.test_gpu_plan_poison import _Poison

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fx():
    return torch.load(oo.FIXTURE)


@pytest.fixture(scope="module")
def bitwise():
    from kandinsky2 import launch_plan
    old = launch_plan.TUNE_SMALL_M
    launch_plan.TUNE_SMALL_M = 0     # bit-identical GEMM configurations only (as bench.py --dump-outputs)
    yield
    launch_plan.TUNE_SMALL_M = old


def _towers(geo, seed, bpe=None):
    from kandinsky2.model.clip_vitl14 import load_openai_clip
    return load_openai_clip(oo.synth_weights(geo, seed), "cuda", bpe)


def _dev(y, ref):
    return (y - ref).abs().max().item(), ((y - ref).norm() / ref.norm()).item()


def test_tiny_towers_against_transformers_golden(fx):
    text, image = _towers(fx["geo"], fx["weight_seed"])
    hid, temb = text.forward(fx["tokens"])
    pix = oo.sample_pixels(fx["geo"], fx["pixel_seed"])
    assert oo.sha256(pix) == fx["pixel_sha256"]
    iemb = image.image_embeds(pix.cuda())
    for got, ref, what in ((hid.float().cpu(), fx["txt_feat_seq"], "txt_feat_seq"), (temb.cpu(), fx["txt_feat"], "txt_feat"),
                           (iemb.cpu(), fx["image_emb"], "image_emb")):
        mx, rel = _dev(got, ref)
        rms = ref.pow(2).mean().sqrt().item()
        print(f"tiny ViT {what}: rel-L2 {rel:.2e}, max-abs {mx / rms:.2e} RMS")
        assert rel < 2e-3 and mx < 1e-2 * rms, (what, rel, mx, rms)


def test_graph_replay_batching_and_poisoned_build(fx, bitwise, monkeypatch):
    geo = fx["geo"]
    text, image = _towers(geo, 7)
    tok = oo.sample_tokens(geo, 8, n=4)
    pix = torch.randn(4, 3, 56, 56, device="cuda", generator=torch.Generator(device="cuda").manual_seed(5))
    runs = ((text, lambda t, x, g: t.forward(x, g), tok), (image, lambda t, x, g: t.forward(x, g), pix))
    for tower, fwd, x in runs:
        h_g, e_g = fwd(tower, x, True)
        h_e, e_e = fwd(tower, x, False)
        assert torch.equal(h_g, h_e) and torch.equal(e_g, e_e) and torch.isfinite(e_g).all()
        assert torch.equal(fwd(tower, x, True)[1], e_g)                    # replayed again
        for b in range(4):
            h1, e1 = fwd(tower, x[b:b + 1], True)
            assert torch.equal(h1[0], h_g[b]) and torch.equal(e1[0], e_g[b]), b
    poison = _Poison(monkeypatch)
    fresh_t, fresh_i = _towers(geo, 7)
    with poison:
        fresh_t._plan(4)
        fresh_i._plan(4)
    for use_graph in (False, True):
        assert torch.equal(fresh_t.forward(tok, use_graph)[1], text.forward(tok)[1])
        assert torch.equal(fresh_i.forward(pix, use_graph)[1], image.forward(pix)[1])


# ---------------------------------------------------------------------------------------------------------------------------
# full ViT-L/14 geometry, synthetic weights
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def full():
    from kandinsky2.checkpoints import openai_clip_to_k2
    from kandinsky2.model.clip_vitl14 import OpenAICLIPTextTower, OpenAICLIPVisionTower
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    sd = {k: v.cuda() for k, v in oo.synth_weights(oo.GEO_L14, 31).items()}
    t, v, geo = openai_clip_to_k2(sd)
    yield sd, OpenAICLIPTextTower(t, geo["text"]).finalize(), OpenAICLIPVisionTower(v, geo["vision"]).finalize()
    del sd
    torch.cuda.empty_cache()


def _calibrate(name, got, r32, r16):
    """rel-L2 at most the fp16 oracle's; max-abs within 1.5 times its (the XLM-R precedent: both end in an fp16 rounding of
    the largest outputs, so the single largest error is one rounding either way)."""
    k_abs, k_rel = _dev(got, r32)
    o_abs, o_rel = _dev(r16, r32)
    print(f"CLIP ViT-L/14 {name}: k2 vs fp32 max-abs {k_abs:.3e} rel-L2 {k_rel:.3e} | fp16 oracle vs fp32 max-abs "
          f"{o_abs:.3e} rel-L2 {o_rel:.3e}")
    assert k_rel <= o_rel and k_abs <= 1.5 * o_abs, (name, k_abs, k_rel, o_abs, o_rel)


@pytest.mark.parametrize("n", [2, 4])
def test_full_size_text_tower_fp16_calibration(full, n):
    sd, text, _ = full
    tok = oo.sample_tokens(oo.GEO_L14, 40 + n, n=n).cuda()
    hid, emb = text.forward(tok, use_graph=False)
    assert torch.isfinite(hid).all() and torch.isfinite(emb).all()
    with torch.no_grad():
        s32, e32 = oo.text_forward(sd, tok)
        s16, e16 = oo.text_forward(sd, tok, dtype=torch.float16)
    _calibrate(f"text n={n} txt_feat", emb, e32, e16)
    _calibrate(f"text n={n} txt_feat_seq", hid.float(), s32, s16)
    assert torch.equal(text.forward(tok)[1], emb)                          # graph replay = the eager launch list


@pytest.mark.parametrize("B", [1, 4])
def test_full_size_image_tower_fp16_calibration(full, B):
    sd, _, image = full
    pix = torch.randn(B, 3, 224, 224, device="cuda", generator=torch.Generator(device="cuda").manual_seed(B))
    pix[0] = 0.0                                                           # create_zero_img_emb's input
    hid, emb = image.forward(pix, use_graph=False)
    assert torch.isfinite(emb).all()
    with torch.no_grad():
        h32, e32 = oo.vision_forward(sd, pix)
        h16, e16 = oo.vision_forward(sd, pix, dtype=torch.float16)
    _calibrate(f"image B={B} embedding", emb, e32, e16)
    _calibrate(f"image B={B} last hidden", hid.float(), h32, h16)
    assert torch.equal(image.forward(pix)[1], emb)


# ---------------------------------------------------------------------------------------------------------------------------
# PriorEmbedder.from_pretrained on a tiny 2.1 folder
# ---------------------------------------------------------------------------------------------------------------------------
GEO_E2E = dict(oo.GEO_TINY, embed_dim=768)     # the tiny 2.1 decoder takes 768-wide image embeddings


def _write_folder(path):
    from kandinsky2.model.prior import PriorTransformer
    from oracle import synth
    from tests import xlmr_oracle as xo
    from tests.test_cpu_clip_vitl14 import _synthetic_bpe
    geo = GEO_E2E
    spec = PriorTransformer(text_ctx=geo["context"], xf_width=128, xf_layers=1, xf_heads=2, xf_final_ln=True, xf_padding=False,
                            clip_dim=geo["embed_dim"], clip_xf_width=geo["text_width"], device="meta").state_dict()
    prior = synth.synth_state_dict([(k, tuple(v.shape)) for k, v in spec.items()], seed=3)
    torch.save({"model." + k: v.half() for k, v in prior.items()}, path / "prior_fp16.ckpt")
    g = torch.Generator().manual_seed(4)
    torch.save((0.1 * torch.randn(geo["embed_dim"], generator=g), 0.5 + torch.rand(geo["embed_dim"], generator=g)),
               path / "ViT-L-14_stats.th")
    torch.save({k: v.half() for k, v in oo.synth_weights(geo, 5).items()}, path / "ViT-L-14.pt")
    _synthetic_bpe(path)                                                   # writes bpe_simple_vocab_16e6.txt.gz
    xfx = torch.load(xo.FIXTURE)
    t0 = xfx["towers"][0]
    te = path / "text_encoder"
    te.mkdir()
    torch.save({k: v.half() for k, v in xo.synth_weights(t0["cfg"], t0["out_features"], 9).items()}, te / "pytorch_model.bin")
    (te / "config.json").write_text(json.dumps(dict(t0["cfg"], architectures=["MultilingualCLIP"])))
    (te / "tokenizer.json").write_text(xo.fixture_json(xfx), encoding="utf-8")
    return t0


@pytest.fixture(scope="module")
def folder(tmp_path_factory):
    path = tmp_path_factory.mktemp("k21")
    return path, _write_folder(path)


def _photo(w, h, seed):
    import numpy as np
    from PIL import Image
    return Image.fromarray((np.random.default_rng(seed).random((h, w, 3)) * 255).astype("uint8"))


def test_from_pretrained_drives_the_21_pipeline(folder, bitwise):
    from kandinsky2 import get_kandinsky2
    from kandinsky2.model.prior import PriorEmbedder, sample_prior
    from kandinsky2.model.gaussian_diffusion import space_timesteps
    from tests.test_gpu_movq_sampler import _tiny_overrides
    path, t0 = folder
    emb = PriorEmbedder.from_pretrained(str(path), prior_steps="5")
    assert emb.clip_text.act == emb.clip_image.act == "quick_gelu"
    over = _tiny_overrides()
    over["model_config"] = dict(over["model_config"], text_encoder_in_dim1=t0["cfg"]["hidden_size"],
                                text_encoder_in_dim2=t0["out_features"])
    pipe = get_kandinsky2("cuda", task_type="text2img", model_version="2.1", cache_dir="/nonexistent", embedder=emb,
                          config_overrides=over)
    kw = dict(num_steps=3, batch_size=2, guidance_scale=4, h=64, w=64, sampler="p_sampler")
    a = pipe.generate_text2img("a red cat", **kw)
    assert len(a) == 2 and [x.tobytes() for x in a] == [x.tobytes() for x in pipe.generate_text2img("a red cat", **kw)]
    # by hand: the CLIP text tower -> the prior's sampling (PriorEmbedder.image_emb's generator) -> the decoder with the
    # image tower's zero embedding as the negative
    import hashlib
    feat, seq, mask = emb.clip_text(["a red cat"] * 2 + [""] * 2)
    assert feat.dtype == seq.dtype == torch.float32 and mask.dtype == torch.bool and seq.shape == (4, 16, 128)
    steps = sorted(space_timesteps(1000, [5]))
    g = torch.Generator(device="cuda").manual_seed(
        int.from_bytes(hashlib.sha256(b"0:a red cat").digest()[:7], "little"))
    x_T = torch.randn(2, 768, device="cuda", generator=g)
    noise = torch.randn(len(steps), 2, 768, device="cuda", generator=g)
    pos = sample_prior(emb.prior, feat, seq, mask, steps, 4.0, emb.clip_mean, emb.clip_std, x_T, noise).float().cpu()
    zero = emb.clip_image.zero_embed().float().cpu()
    assert torch.isfinite(pos).all() and torch.isfinite(zero).all()
    hand = pipe.generate_img("a red cat", torch.cat([pos, zero.repeat(2, 1)]), batch_size=2, guidance_scale=4, h=64, w=64,
                             sampler="p_sampler", num_steps=3, diffusion=pipe._diffusion("p_sampler", 3))
    assert [x.tobytes() for x in hand] == [x.tobytes() for x in a]
    # mix_images with a text and a PIL image
    img = _photo(90, 70, 1)
    kw1 = dict(kw, batch_size=1)
    m = pipe.mix_images(["a red cat", img], [0.4, 0.6], **kw1)
    assert [x.tobytes() for x in m] == [x.tobytes() for x in pipe.mix_images(["a red cat", img], [0.4, 0.6], **kw1)]
    e_img = emb.clip_image(img)
    assert e_img.shape == (1, 768) and torch.equal(e_img, emb.clip_image.image_embeds(
        emb.clip_image.preprocess(img).cuda()).cpu())
    mixed = emb.image_emb("a red cat", 1) * 0.4 + e_img * 0.6
    hand = pipe.generate_img("", torch.cat([mixed, zero]), batch_size=1, guidance_scale=4, h=64, w=64, sampler="p_sampler",
                             num_steps=3, diffusion=pipe._diffusion("p_sampler", 3))
    assert [x.tobytes() for x in hand] == [x.tobytes() for x in m]


@pytest.mark.parametrize("name", ["prior_fp16.ckpt", "ViT-L-14_stats.th", "text_encoder", "ViT-L-14.pt",
                                  "bpe_simple_vocab_16e6.txt.gz"])
def test_from_pretrained_names_each_missing_file(folder, tmp_path, name):
    import shutil

    from kandinsky2._native import K2Error
    from kandinsky2.model.prior import PriorEmbedder
    src, _ = folder
    for f in os.listdir(src):
        if f != name and f != "tok":
            (shutil.copytree if os.path.isdir(src / f) else shutil.copy)(src / f, tmp_path / f)
    with pytest.raises(K2Error, match=name.replace(".", r"\.")):
        PriorEmbedder.from_pretrained(str(tmp_path))


def test_from_pretrained_refuses_a_mismatched_clip(folder, tmp_path):
    import shutil

    from kandinsky2._native import K2Error
    from kandinsky2.model.prior import PriorEmbedder
    src, _ = folder
    torch.save(oo.synth_weights(dict(GEO_E2E, context=20), 5), tmp_path / "other.pt")
    with pytest.raises(K2Error, match=r"\(128, 768, 20\).*\(128, 768, 16\)"):
        PriorEmbedder.from_pretrained(str(src), clip_path=str(tmp_path / "other.pt"))
    shutil.rmtree(tmp_path, ignore_errors=True)
