"""GPU: the CLIP text tower (kandinsky2/model/clip_text.py) end to end.

  - the tiny towers of tests/golden/clip_text_tiny.pt (transformers' own outputs, both pooling rules) within the image
    tower's bound;
  - the full ViT-bigG/14 text geometry on synthetic weights, against the fp32 oracle (tests/clip_text_oracle.py): rel-L2
    closer than the oracle's own fp16 mode (the calibration of the UNet, both priors and the image tower), max-abs within
    1.5x of it, with the fp16 residual stream's peak recorded;
  - graph replay against the eager launch list, a batch against its rows one at a time, plans built over NaN-poisoned
    buffers, repeated prompts against the distinct ones: bit for bit;
  - the embedder wiring: PriorEmbedder22.from_diffusers(text_encoder=tower) and from_pretrained on a folder written here,
    driving Kandinsky2_2.generate_text2img.  The full-size tests need about 12 GB of device memory."""
import json
import os

import pytest
import torch

from tests import clip_text_oracle as cto
from tests.test_gpu_plan_poison import _Poison

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fx():
    return torch.load(cto.FIXTURE)


def _tokenizer(fx):
    from kandinsky2.model.clip_text import CLIPTokenizer
    return CLIPTokenizer(cto.synthetic_vocab(fx["merges"]), [tuple(m) for m in fx["merges"]], model_max_length=fx["max_length"])


def _tower(cfg, seed, tokenizer=None):
    from kandinsky2.model.clip_text import CLIPTextTower
    return CLIPTextTower.from_transformers(cto.synth_weights(cfg, seed), cfg, device="cuda", tokenizer=tokenizer)


def _dev(y, ref):
    return (y - ref).abs().max().item(), ((y - ref).norm() / ref.norm()).item()


@pytest.fixture(scope="module")
def bitwise():
    from kandinsky2 import launch_plan
    old = launch_plan.TUNE_SMALL_M
    launch_plan.TUNE_SMALL_M = 0     # bit-identical GEMM configurations only (as bench.py --dump-outputs)
    yield
    launch_plan.TUNE_SMALL_M = old


@pytest.mark.parametrize("i", [0, 1])
def test_tiny_tower_against_transformers_golden(fx, i):
    t = fx["towers"][i]
    tower = _tower(t["cfg"], t["weight_seed"])
    hid, emb = tower.forward(t["input_ids"].long())
    for got, ref, what in ((hid.float().cpu(), t["last_hidden_state"], "last_hidden_state"), (emb.cpu(), t["text_embeds"], "embeds")):
        mx, rel = _dev(got, ref)
        rms = ref.pow(2).mean().sqrt().item()
        print(f"tiny text tower {i} {what}: rel-L2 {rel:.2e}, max-abs {mx / rms:.2e} RMS")
        assert rel < 2e-3 and mx < 1e-2 * rms, (what, rel, mx, rms)
    plan = tower._plan(*t["input_ids"].shape)
    idx = cto.pooled_index(t["input_ids"].long(), t["cfg"]["eos_token_id"])
    assert plan.index.cpu().tolist() == idx.tolist()


def _tiny_cfg(fx, eos=None, projection_dim=32):
    V = len(cto.synthetic_vocab(fx["merges"]))
    return dict(cto.tiny_config(V, V - 1 if eos is None else eos), projection_dim=projection_dim)


def test_graph_replay_batching_poisoned_build_and_prompts(fx, bitwise, monkeypatch):
    cfg = _tiny_cfg(fx)
    tok = _tokenizer(fx)
    prompts = ["a red cat", "A capybara, 4k photo", "", "a <|endoftext|> b"]
    ids = tok(prompts)["input_ids"]
    tower = _tower(cfg, 7, tok)
    h_g, e_g = tower.forward(ids, use_graph=True)
    h_e, e_e = tower.forward(ids, use_graph=False)
    assert torch.equal(h_g, h_e) and torch.equal(e_g, e_e) and torch.isfinite(e_g).all()
    assert torch.equal(tower.forward(ids)[1], e_g)                         # replayed again
    for b in range(4):
        h1, e1 = tower.forward(ids[b:b + 1])
        assert torch.equal(h1[0], h_g[b]) and torch.equal(e1[0], e_g[b]), b
    poison = _Poison(monkeypatch)
    fresh = _tower(cfg, 7, tok)
    with poison:
        fresh._plan(4)
        fresh._plan(2)
    for use_graph in (False, True):
        h_p, e_p = fresh.forward(ids, use_graph)
        assert torch.equal(h_p, h_g) and torch.equal(e_p, e_g), use_graph
    # the clip_text protocol: repeated prompts are encoded once and gathered back
    calls = []
    fwd = type(tower).forward
    monkeypatch.setattr(type(tower), "forward", lambda self, x, use_graph=True: (calls.append(x.shape[0]), fwd(self, x))[1])
    e, h, m = tower(["a red cat", "a red cat", "", "a red cat", ""])
    assert calls == [2]
    e2, h2, m2 = tower(["a red cat", ""])
    assert torch.equal(e, e2[[0, 0, 1, 0, 1]]) and torch.equal(h, h2[[0, 0, 1, 0, 1]]) and torch.equal(m, m2[[0, 0, 1, 0, 1]])
    assert torch.equal(e2[0], e_g[0]) and torch.equal(h2[1], h_g[2])
    assert m.dtype == torch.bool and m2.sum(1).tolist() == tok(["a red cat", ""])["attention_mask"].sum(1).tolist()


# ---------------------------------------------------------------------------------------------------------------------------
# full ViT-bigG/14 text geometry, synthetic weights
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def full():
    from kandinsky2.checkpoints import transformers_clip_text_to_k2
    from kandinsky2.model.clip_text import CLIPTextTower
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = cto.CONFIG_BIGG
    sd = {k: v.cuda() for k, v in cto.synth_weights(cfg, 21).items()}
    tower = CLIPTextTower(transformers_clip_text_to_k2(sd), cfg, device="cuda").finalize()
    yield cfg, sd, tower
    del sd, tower
    torch.cuda.empty_cache()


def bigg_ids(n, seed, lengths=(3, 20, 77)):
    """n rows of 77: bos, random ids below bos, eos, then pad (id 0), with the rows' real lengths cycling through `lengths`."""
    V = cto.CONFIG_BIGG["vocab_size"]
    bos, eos = V - 2, V - 1
    g = torch.Generator().manual_seed(seed)
    ids = torch.zeros(n, 77, dtype=torch.long)
    for r in range(n):
        L = lengths[r % len(lengths)]
        ids[r, 0], ids[r, L - 1] = bos, eos
        ids[r, 1:L - 1] = torch.randint(1, bos, (L - 2,), generator=g)
    return ids


@pytest.mark.parametrize("n", [2, 8])
def test_full_size_fp16_calibration(full, n, monkeypatch):
    from kandinsky2 import ops
    cfg, sd, tower = full
    ids = bigg_ids(n, seed=n)
    tower._plan(n)                                                         # built (and tuned) before the GEMMs are counted
    peaks, gemm_rows = [], ops.gemm_rows

    def recording_gemm_rows(*a, **kw):
        y = gemm_rows(*a, **kw)
        if kw.get("residual") is not None:
            peaks.append(y.abs().amax())
        return y

    monkeypatch.setattr(ops, "gemm_rows", recording_gemm_rows)
    hid, emb = tower.forward(ids, use_graph=False)
    monkeypatch.undo()
    assert len(peaks) == 2 * cfg["num_hidden_layers"]
    peak = torch.stack(peaks).max().item()
    assert torch.isfinite(torch.stack(peaks)).all() and torch.isfinite(emb).all(), peak
    assert tower._plan(n).index.cpu().tolist() == cto.pooled_index(ids, 2).tolist()
    with torch.no_grad():
        h32, e32 = cto.forward(sd, cfg, ids.cuda())
        h16, e16 = cto.forward(sd, cfg, ids.cuda(), dtype=torch.float16)
    res = {}
    for name, got, r32, r16 in (("embeds", emb, e32, e16), ("hidden", hid.float(), h32, h16)):
        k_abs, k_rel = _dev(got, r32)
        o_abs, o_rel = _dev(r16, r32)
        res[name] = (k_abs, k_rel, o_abs, o_rel)
        print(f"CLIP ViT-bigG/14 text n={n} {name}: k2 vs fp32 max-abs {k_abs:.3e} rel-L2 {k_rel:.3e} | fp16 oracle vs fp32 "
              f"max-abs {o_abs:.3e} rel-L2 {o_rel:.3e}; residual stream peak |h| {peak:.1f}")
    # rel-L2 is the calibration: below the fp16 mode's.  The max-abs is one element's rounding (of n x 1280 pooled values, or
    # of fp16 outputs where 2 ulp ~ 0.0156): on an H100 it fell either side of the fp16 mode's, within 1.27x; held to 1.5x.
    for name, (k_abs, k_rel, o_abs, o_rel) in res.items():
        assert k_rel <= o_rel and k_abs <= 1.5 * o_abs, (name, res[name])
    assert torch.equal(tower.forward(ids)[1], emb)                         # graph replay = the eager launch list


# ---------------------------------------------------------------------------------------------------------------------------
# wiring: PriorEmbedder22 and the pipeline
# ---------------------------------------------------------------------------------------------------------------------------
PRIOR_CFG = dict(text_ctx=77, xf_width=128, xf_layers=2, xf_heads=2, xf_final_ln=True, xf_padding=False, clip_dim=1280,
                 clip_xf_width=128)


@pytest.fixture(scope="module")
def wired(fx, bitwise):
    """A tiny 2.2 prior (77 text tokens, clip_dim 1280 as the decoder expects) and a tiny tower whose projection is 1280
    wide."""
    from oracle import synth
    from tests import prior22_oracle as p22
    dsd = synth.synth_state_dict(p22.diffusers_prior_spec(PRIOR_CFG), seed=13)
    cfg = _tiny_cfg(fx, projection_dim=1280)
    return dsd, cfg, _tower(cfg, 9, _tokenizer(fx))


@pytest.mark.parametrize("guidance", [4.0, 1.0])
def test_text_encoder_is_the_clip_text_callable(wired, guidance):
    from kandinsky2.model.prior import PriorEmbedder22
    dsd, cfg, tower = wired
    a = PriorEmbedder22.from_diffusers(dsd, text_encoder=tower)
    assert a.clip_text is tower
    same = lambda prompts: tuple(t.clone() for t in tower(prompts))   # noqa: E731  the tower's own outputs, as a callable
    b = PriorEmbedder22.from_diffusers(dsd, same)
    kw = dict(prior_steps=5, prior_guidance_scale=guidance, negative_prior_prompt="low quality")
    x = a.image_emb("a red cat", 2, **kw)
    assert x.shape == (2, 1280) and torch.isfinite(x).all()
    assert torch.equal(x, b.image_emb("a red cat", 2, **kw))
    if guidance > 1:
        assert not torch.equal(x, a.image_emb("a blue cat", 2, **kw))


def test_from_diffusers_refusals(wired, fx):
    from kandinsky2._native import K2Error
    from kandinsky2.model.prior import PriorEmbedder22
    from oracle import synth
    from tests import prior22_oracle as p22
    dsd, cfg, tower = wired
    with pytest.raises(ValueError, match="exactly one"):
        PriorEmbedder22.from_diffusers(dsd, lambda p: None, text_encoder=tower)
    with pytest.raises(ValueError, match="exactly one"):
        PriorEmbedder22.from_diffusers(dsd)
    for change in (dict(text_ctx=8), dict(clip_xf_width=256), dict(clip_dim=32)):
        bad = synth.synth_state_dict(p22.diffusers_prior_spec(dict(PRIOR_CFG, **change)), seed=13)
        with pytest.raises(K2Error, match="text_ctx, clip_xf_width, clip_dim"):
            PriorEmbedder22.from_diffusers(bad, text_encoder=tower)


def _write_folder(root, fx, dsd, cfg, seed, fmt):
    """A kandinsky-2-2-prior-shaped folder: prior/, text_encoder/, tokenizer/ (fmt "bin": torch.save, "safetensors")."""
    def save(sd, sub, stem):
        os.makedirs(os.path.join(root, sub), exist_ok=True)
        if fmt == "bin":
            torch.save(sd, os.path.join(root, sub, stem + ".bin"))
        else:
            from safetensors.torch import save_file
            save_file({k: v.contiguous() for k, v in sd.items()}, os.path.join(root, sub, stem + ".safetensors"))
    save(dsd, "prior", "diffusion_pytorch_model")
    save({k: v.half() for k, v in cto.synth_weights(cfg, seed).items()}, "text_encoder", "model")
    with open(os.path.join(root, "text_encoder", "config.json"), "w") as f:
        json.dump(dict(cfg, architectures=["CLIPTextModelWithProjection"], torch_dtype="float16"), f)
    os.makedirs(os.path.join(root, "tokenizer"))
    with open(os.path.join(root, "tokenizer", "vocab.json"), "w") as f:
        json.dump(cto.synthetic_vocab(fx["merges"]), f)
    with open(os.path.join(root, "tokenizer", "merges.txt"), "w") as f:
        f.write("#version: 0.2\n" + "\n".join(" ".join(m) for m in fx["merges"]) + "\n")
    with open(os.path.join(root, "tokenizer", "tokenizer_config.json"), "w") as f:
        json.dump(dict(model_max_length=77, pad_token="<|endoftext|>"), f)


@pytest.mark.parametrize("fmt", ["bin", "safetensors"])
def test_from_pretrained_drives_text2img(wired, fx, tmp_path, fmt):
    from kandinsky2 import get_kandinsky2
    from kandinsky2._native import K2Error
    from kandinsky2.model.prior import PriorEmbedder22
    from tests.test_gpu_movq_sampler import _tiny_overrides
    if fmt == "safetensors":
        pytest.importorskip("safetensors")
    dsd, cfg, _ = wired
    root = str(tmp_path / "kandinsky-2-2-prior")
    _write_folder(root, fx, dsd, cfg, 9, fmt)
    emb = PriorEmbedder22.from_pretrained(root, prior_steps=3)
    assert emb.clip_image is None
    pipe = get_kandinsky2("cuda", task_type="text2img", model_version="2.2", cache_dir="/nonexistent", embedder=emb,
                          config_overrides=_tiny_overrides())
    kw = dict(batch_size=2, decoder_steps=2, h=64, w=64)
    a = pipe.generate_text2img("a red cat", **kw)
    assert len(a) == 2 and a[0].size == (64, 64)
    assert [x.tobytes() for x in a] == [x.tobytes() for x in pipe.generate_text2img("a red cat", **kw)]
    # the folder's fp16 text encoder equals a tower built from the same fp16 weights
    from kandinsky2.model.clip_text import CLIPTextTower
    ref = CLIPTextTower.from_transformers({k: v.half() for k, v in cto.synth_weights(cfg, 9).items()}, cfg,
                                          tokenizer=_tokenizer(fx))
    assert torch.equal(emb.clip_text(["a red cat"])[0], ref(["a red cat"])[0])
    os.remove(os.path.join(root, "tokenizer", "merges.txt"))
    with pytest.raises(K2Error, match="merges.txt"):
        PriorEmbedder22.from_pretrained(root)
    os.remove(os.path.join(root, "text_encoder", "config.json"))
    with pytest.raises(K2Error, match="config.json"):
        PriorEmbedder22.from_pretrained(root)
