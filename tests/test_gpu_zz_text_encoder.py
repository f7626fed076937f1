"""GPU: the Kandinsky 2.1 text encoder (kandinsky2/model/text_encoders.py) end to end.

  - the tiny towers of tests/golden/xlmr_tiny.pt (transformers' own outputs) within the CLIP towers' bound;
  - XLM-RoBERTa-large (24 x 1024, vocabulary 250002, 514 positions) on synthetic weights against the fp32 oracle
    (tests/xlmr_oracle.py): rel-L2 no worse than the oracle's own fp16 mode, max-abs within 1.5x of it, the residual stream
    finite;
  - graph replay against the eager launch list, a batch against its rows one at a time, plans built over NaN-poisoned
    buffers, tower(prompt, B) against forward of the tokenized [prompt x B | "" x B]: bit for bit;
  - the embedder wiring: PriorEmbedder(text_encoder=tower) driving a tiny Kandinsky2_1's generate_text2img and
    generate_inpainting, and TextEncoder on a folder written here.  The full-size tests need about 8 GB of device memory."""
import json
import os

import pytest
import torch

from tests import xlmr_oracle as xo
from tests.test_gpu_plan_poison import _Poison

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def fx():
    return torch.load(xo.FIXTURE)


def _tokenizer(fx):
    return xo.k2_tokenizer(xo.fixture_json(fx))


def _tower(cfg, out, seed, tokenizer=None):
    from kandinsky2.model.text_encoders import MultilingualCLIP
    return MultilingualCLIP.from_state_dict(xo.synth_weights(cfg, out, seed), cfg, tokenizer=tokenizer, device="cuda")


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
    tower = _tower(t["cfg"], t["out_features"], t["weight_seed"])
    hid, pooled = tower.forward(t["input_ids"].long(), t["attention_mask"].long())
    for got, ref, what in ((hid.float().cpu(), t["last_hidden_state"], "last_hidden_state"), (pooled.cpu(), t["pooled"], "pooled")):
        mx, rel = _dev(got, ref)
        rms = ref.pow(2).mean().sqrt().item()
        print(f"tiny M-CLIP tower {i} {what}: rel-L2 {rel:.2e}, max-abs {mx / rms:.2e} RMS")
        assert rel < 2e-3 and mx < 1e-2 * rms, (what, rel, mx, rms)


def test_graph_replay_batching_poisoned_build_and_prompts(fx, bitwise, monkeypatch):
    t0 = fx["towers"][0]
    cfg, out = t0["cfg"], t0["out_features"]
    tok = _tokenizer(fx)
    prompts = ["a red cat", "A capybara, 4k photo", "", "a <mask> b <pad> c"]
    e = tok(prompts)
    ids, mask = e["input_ids"], e["attention_mask"]
    tower = _tower(cfg, out, 7, tok)
    h_g, p_g = tower.forward(ids, mask, use_graph=True)
    h_e, p_e = tower.forward(ids, mask, use_graph=False)
    assert torch.equal(h_g, h_e) and torch.equal(p_g, p_e) and torch.isfinite(p_g).all() and torch.isfinite(h_g).all()
    assert torch.equal(tower.forward(ids, mask)[1], p_g)                    # replayed again
    for b in range(4):
        h1, p1 = tower.forward(ids[b:b + 1], mask[b:b + 1])
        assert torch.equal(h1[0], h_g[b]) and torch.equal(p1[0], p_g[b]), b
    poison = _Poison(monkeypatch)
    fresh = _tower(cfg, out, 7, tok)
    with poison:
        fresh._plan(4)
        fresh._plan(1)
    for use_graph in (False, True):
        h_p, p_p = fresh.forward(ids, mask, use_graph)
        assert torch.equal(h_p, h_g) and torch.equal(p_p, p_g), use_graph
    # the text_encoder protocol: [prompt x B | "" x B], each distinct prompt encoded once
    calls = []
    fwd = type(tower).forward
    monkeypatch.setattr(type(tower), "forward",
                        lambda self, x, m, use_graph=True: (calls.append(x.shape[0]), fwd(self, x, m))[1])
    full, pooled = tower("a red cat", 3)
    assert calls == [2] and full.shape == (6, 77, cfg["hidden_size"]) and pooled.shape == (6, out)
    ref = tok(["a red cat"] * 3 + [""] * 3)
    h_r, p_r = fwd(tower, ref["input_ids"], ref["attention_mask"])
    assert torch.equal(full, h_r) and torch.equal(pooled, p_r)
    assert torch.equal(full[0], h_g[0]) and torch.equal(pooled[5], p_g[2])
    assert len(calls) == 1 and tower("", 2)[0].shape[0] == 4 and calls[-1] == 1


# ---------------------------------------------------------------------------------------------------------------------------
# XLM-RoBERTa-large, synthetic weights
# ---------------------------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def full():
    from kandinsky2.checkpoints import mclip_to_k2
    from kandinsky2.model.text_encoders import MultilingualCLIP
    torch.backends.cuda.matmul.allow_tf32 = False
    torch.backends.cudnn.allow_tf32 = False
    cfg = xo.CONFIG_LARGE
    sd = {k: v.cuda() for k, v in xo.synth_weights(cfg, xo.OUT_LARGE, 21).items()}
    tower = MultilingualCLIP(mclip_to_k2(sd, cfg["num_hidden_layers"]), cfg, device="cuda").finalize()
    yield cfg, sd, tower
    del sd, tower
    torch.cuda.empty_cache()


def large_ids(n, seed, lengths=(2, 9, 40, 77)):
    """n rows of 77: <s>, random ids, </s>, then <pad>, the rows' real lengths cycling through `lengths` (2 is the empty
    prompt)."""
    V = xo.CONFIG_LARGE["vocab_size"]
    g = torch.Generator().manual_seed(seed)
    ids = torch.full((n, 77), xo.PAD_ID, dtype=torch.long)
    for r in range(n):
        L = lengths[r % len(lengths)]
        ids[r, 0], ids[r, L - 1] = 0, 2
        ids[r, 1:L - 1] = torch.randint(3, V, (L - 2,), generator=g)
    return ids, (ids != xo.PAD_ID).long()


@pytest.mark.parametrize("n", [2, 8])
def test_full_size_fp16_calibration(full, n, monkeypatch):
    from kandinsky2 import ops
    cfg, sd, tower = full
    ids, mask = large_ids(n, seed=n)
    tower._plan(n)                                                         # built (and tuned) before the GEMMs are counted
    peaks, gemm_rows = [], ops.gemm_rows

    def recording_gemm_rows(*a, **kw):
        y = gemm_rows(*a, **kw)
        if kw.get("residual") is not None:
            peaks.append(y.abs().amax())
        return y

    monkeypatch.setattr(ops, "gemm_rows", recording_gemm_rows)
    hid, pooled = tower.forward(ids, mask, use_graph=False)
    monkeypatch.undo()
    assert len(peaks) == 2 * cfg["num_hidden_layers"]
    peak = torch.stack(peaks).max().item()
    assert torch.isfinite(torch.stack(peaks)).all() and torch.isfinite(hid).all() and torch.isfinite(pooled).all(), peak
    with torch.no_grad():
        h32, p32 = xo.forward(sd, cfg, ids.cuda(), mask.cuda())
        h16, p16 = xo.forward(sd, cfg, ids.cuda(), mask.cuda(), dtype=torch.float16)
    res = {}
    for name, got, r32, r16 in (("pooled", pooled, p32, p16), ("full", hid.float(), h32, h16)):
        k_abs, k_rel = _dev(got, r32)
        o_abs, o_rel = _dev(r16, r32)
        res[name] = (k_abs, k_rel, o_abs, o_rel)
        print(f"XLM-R-large n={n} {name}: k2 vs fp32 max-abs {k_abs:.3e} rel-L2 {k_rel:.3e} | fp16 oracle vs fp32 max-abs "
              f"{o_abs:.3e} rel-L2 {o_rel:.3e}; residual stream peak |h| {peak:.1f}")
    for name, (k_abs, k_rel, o_abs, o_rel) in res.items():
        assert k_rel <= o_rel and k_abs <= 1.5 * o_abs, (name, res[name])
    h_g, p_g = tower.forward(ids, mask)                                    # graph replay = the eager launch list
    assert torch.equal(h_g, hid) and torch.equal(p_g, pooled)


# ---------------------------------------------------------------------------------------------------------------------------
# wiring: PriorEmbedder, Kandinsky2_1 and TextEncoder
# ---------------------------------------------------------------------------------------------------------------------------
def _tiny_pipeline(tower, task):
    from kandinsky2 import get_kandinsky2
    from kandinsky2.model.prior import PriorEmbedder
    from kandinsky2.pipelines import SyntheticEmbedder
    from tests.test_gpu_movq_sampler import _tiny_overrides
    syn = SyntheticEmbedder(768)

    class _Prior:            # the prior is not under test: the synthetic image embedding stands in for its sampling
        clip_dim = 768

    emb = PriorEmbedder(_Prior(), None, clip_mean=torch.zeros(768, device="cuda"), clip_std=torch.ones(768, device="cuda"),
                        text_encoder=tower)
    emb.image_emb = syn.image_emb
    over = _tiny_overrides()
    over["model_config"] = dict(over["model_config"], text_encoder_in_dim1=tower.cfg["hidden_size"],
                                text_encoder_in_dim2=tower.out_features)
    return get_kandinsky2("cuda", task_type=task, model_version="2.1", cache_dir="/nonexistent", embedder=emb,
                          config_overrides=over)


def test_prior_embedder_drives_text2img_and_inpainting(fx, bitwise):
    from PIL import Image
    t0 = fx["towers"][0]
    tower = _tower(t0["cfg"], t0["out_features"], 9, _tokenizer(fx))
    pipe = _tiny_pipeline(tower, "text2img")
    kw = dict(num_steps=3, batch_size=2, guidance_scale=4, h=64, w=64, sampler="p_sampler")
    a = pipe.generate_text2img("a red cat", **kw)
    assert len(a) == 2 and a[0].size == (64, 64)
    assert [x.tobytes() for x in a] == [x.tobytes() for x in pipe.generate_text2img("a red cat", **kw)]
    assert [x.tobytes() for x in a] != [x.tobytes() for x in pipe.generate_text2img("a blue dog", **kw)]
    pipe = _tiny_pipeline(tower, "inpainting")
    img = Image.fromarray((torch.arange(64 * 64 * 3) % 251).reshape(64, 64, 3).to(torch.uint8).numpy())
    m = torch.ones(64, 64).numpy()
    m[16:48, 16:48] = 0
    b = pipe.generate_inpainting("a red cat", img, m, **kw)
    assert len(b) == 2 and [x.tobytes() for x in b] == [x.tobytes() for x in pipe.generate_inpainting("a red cat", img, m, **kw)]


def test_text_encoder_reads_a_folder(fx, tmp_path):
    from kandinsky2._native import K2Error
    from kandinsky2.model.text_encoders import MultilingualCLIP, TextEncoder
    t0 = fx["towers"][0]
    cfg, out = t0["cfg"], t0["out_features"]
    sd = {k: v.half() for k, v in xo.synth_weights(cfg, out, 9).items()}
    torch.save(dict(sd, **{"transformer.embeddings.position_ids": torch.arange(cfg["max_position_embeddings"])[None]}),
               tmp_path / "pytorch_model.bin")
    (tmp_path / "config.json").write_text(json.dumps(dict(cfg, architectures=["MultilingualCLIP"])))
    (tmp_path / "tokenizer.json").write_text(xo.fixture_json(fx), encoding="utf-8")
    enc = TextEncoder(str(tmp_path), "multiclip", in_features=cfg["hidden_size"], out_features=out)
    e = _tokenizer(fx)(["a red cat", ""])
    full, pooled = enc.forward(e["input_ids"], e["attention_mask"])
    ref = MultilingualCLIP.from_state_dict(sd, cfg, tokenizer=_tokenizer(fx))
    assert torch.equal(full, ref.forward(e["input_ids"], e["attention_mask"])[0])
    assert torch.equal(pooled, enc.model("a red cat", 1)[1])
    with pytest.raises(K2Error, match="768"):
        TextEncoder(str(tmp_path), "multiclip")
    os.remove(tmp_path / "tokenizer.json")
    with pytest.raises(K2Error, match="tokenizer.json"):
        TextEncoder(str(tmp_path), "multiclip", in_features=cfg["hidden_size"], out_features=out)
