"""CPU: the CLIP text tower's host side.  kandinsky2's CLIPTokenizer against transformers' input_ids and attention masks in
tests/golden/clip_text_tiny.pt, the restated forward (tests/clip_text_oracle.py) against transformers' own tower outputs, the
state-dict remap through the network, the config / id / tokenizer refusals, and the two new C-ABI entry points' argument
checks (no device needed: nothing is launched).  Where transformers is importable, a second seed runs against it live."""
import json

import pytest
import torch

from tests import clip_text_oracle as cto
from tests.test_cpu_vector_arg_checks import A, P, _refused, _with


@pytest.fixture(scope="module")
def fx():
    return torch.load(cto.FIXTURE)


@pytest.fixture(scope="module")
def tok(fx):
    from kandinsky2.model.clip_text import CLIPTokenizer
    return CLIPTokenizer(cto.synthetic_vocab(fx["merges"]), [tuple(m) for m in fx["merges"]], model_max_length=fx["max_length"])


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


def test_tokenizer_reproduces_every_fixture_text(fx, tok):
    ids, mask = cto.unpack_ids(fx["ids"], fx["lengths"], tok.pad_token_id)
    assert len(fx["texts"]) == ids.shape[0] > 200
    got = tok(fx["texts"])
    bad = [t for i, t in enumerate(fx["texts"]) if not torch.equal(got["input_ids"][i], ids[i])]
    assert not bad, bad[:5]
    assert torch.equal(got["attention_mask"], mask)


def test_tokenizer_edge_cases(fx, tok):
    """The cases the fixture was built around, spelled out."""
    L = fx["max_length"]
    enc = lambda t: tok([t])["input_ids"][0]  # noqa: E731
    bos, eos = tok.bos_token_id, tok.eos_token_id
    assert eos == max(tok.vocab.values()) and bos == eos - 1          # the specials come last
    assert enc("").tolist()[:2] == [bos, eos] and tok([""])["attention_mask"][0].sum() == 2
    assert enc(" \t\n ").tolist()[:3] == [bos, eos, eos]            # whitespace only: no token
    assert enc("\x1c").tolist()[2] == eos and enc("\x1c")[1] != eos   # a token for the backend, whitespace for Python
    assert (enc("a <|endoftext|> b") == eos).nonzero()[0].item() == 2  # a literal eos in the raw text
    assert (enc("<|ENDOFTEXT|>") == eos).nonzero()[0].item() > 3       # not a special once lowercased
    assert not torch.equal(enc("ΟΔΟΣ"), enc("οδος"))                 # no final-sigma rule
    assert torch.equal(enc("ΟΔΟΣ"), enc("οδοσ"))
    x75 = tok(["x " * 75])
    assert x75["attention_mask"][0].sum() == L and x75["input_ids"][0, -1] == eos
    assert torch.equal(tok(["x " * 80 + "tail"])["input_ids"], x75["input_ids"])   # truncated to 75 tokens + eos


def test_tokenizer_from_dir(fx, tmp_path):
    from kandinsky2.model.clip_text import CLIPTokenizer
    vocab = cto.synthetic_vocab(fx["merges"])
    (tmp_path / "vocab.json").write_text(json.dumps(vocab))
    (tmp_path / "merges.txt").write_text("#version: 0.2\n" + "\n".join(" ".join(m) for m in fx["merges"]) + "\n")
    t = CLIPTokenizer.from_dir(str(tmp_path))
    assert t.model_max_length == 77 and t.pad_token_id == t.eos_token_id
    ref = t(fx["texts"][:40])
    (tmp_path / "special_tokens_map.json").write_text(json.dumps({"pad_token": {"content": "!"}}))
    (tmp_path / "tokenizer_config.json").write_text(json.dumps({"model_max_length": 20}))
    t2 = CLIPTokenizer.from_dir(str(tmp_path))
    assert t2.model_max_length == 20 and t2.pad_token_id == vocab["!"]
    e = t2(["hi!!"])
    assert e["input_ids"].shape == (1, 20) and e["input_ids"][0, -1] == vocab["!"]
    assert t2.tokenize_ids("hi!!")[-2:] == [vocab["!"]] * 2         # the pad token is matched in the raw text, like eos
    assert torch.equal(t(fx["texts"][:40])["input_ids"], ref["input_ids"])
    (tmp_path / "merges.txt").unlink()
    from kandinsky2._native import K2Error
    with pytest.raises(K2Error, match="merges.txt"):
        CLIPTokenizer.from_dir(str(tmp_path))


@pytest.mark.parametrize("i", [0, 1])
def test_oracle_equals_transformers_golden(fx, i):
    t = fx["towers"][i]
    sd = cto.synth_weights(t["cfg"], t["weight_seed"])
    hid, emb = cto.forward(sd, t["cfg"], t["input_ids"].long())
    assert _rel(hid, t["last_hidden_state"]) <= 1e-5 and _rel(emb, t["text_embeds"]) <= 1e-5


def test_golden_towers_cover_both_pooling_rules(fx, tok):
    a, b = fx["towers"]
    assert a["cfg"]["eos_token_id"] == 2 and b["cfg"]["eos_token_id"] == tok.eos_token_id
    assert torch.equal(tok(b["prompts"])["input_ids"], b["input_ids"].long())
    idx = cto.pooled_index(b["input_ids"].long(), b["cfg"]["eos_token_id"])
    assert idx.tolist() == [2]                                          # the literal eos, not the final one


@pytest.mark.parametrize("i", [0, 1])
def test_remapped_forward_equals_transformers_names(fx, i):
    from kandinsky2.checkpoints import transformers_clip_text_to_k2
    t = fx["towers"][i]
    sd = cto.synth_weights(t["cfg"], t["weight_seed"])
    sd_pos = dict(sd, **{"text_model.embeddings.position_ids": torch.arange(77)[None]})   # a stray buffer is ignored
    k2 = transformers_clip_text_to_k2(sd_pos)
    a = cto.forward(sd, t["cfg"], t["input_ids"].long())
    b = cto.forward_k2(k2, t["cfg"], t["input_ids"].long())
    for x, y in zip(a, b):
        assert _rel(x, y) <= 1e-6


def test_remap_refuses_missing_and_unexpected_keys(fx):
    from kandinsky2._native import K2Error
    from kandinsky2.checkpoints import transformers_clip_text_to_k2
    sd = cto.synth_weights(fx["towers"][0]["cfg"], 0)
    gone = "text_model.encoder.layers.1.mlp.fc2.bias"
    with pytest.raises(K2Error, match=gone.replace(".", r"\.")):
        transformers_clip_text_to_k2({k: v for k, v in sd.items() if k != gone})
    with pytest.raises(K2Error, match="visual_projection"):
        transformers_clip_text_to_k2(dict(sd, **{"visual_projection.weight": torch.zeros(2, 2)}))
    with pytest.raises(K2Error, match="text_projection"):
        transformers_clip_text_to_k2({k: v for k, v in sd.items() if k != "text_projection.weight"})


@pytest.mark.parametrize("change,msg", [
    (dict(hidden_act="quick_gelu"), "hidden_act"),
    (dict(hidden_act=None), "hidden_act"),
    (dict(hidden_size=1664, num_attention_heads=16), "head width 104"),
    (dict(num_attention_heads=4), "head width 32"),
    (dict(max_position_embeddings=129), "at most 128"),
    (dict(hidden_size=132, num_attention_heads=1, intermediate_size=256), "head width 132"),
    (dict(vocab_size=None), "missing"),
])
def test_from_transformers_refuses_unimplemented_configs(fx, change, msg):
    from kandinsky2._native import K2Error
    from kandinsky2.model.clip_text import CLIPTextTower
    base = fx["towers"][0]["cfg"]
    cfg = dict(base, **change)
    for k in [k for k, v in cfg.items() if v is None]:
        del cfg[k]                         # transformers' default (hidden_act: quick_gelu)
    with pytest.raises(K2Error, match=msg):
        CLIPTextTower.from_transformers(cto.synth_weights(base, 0), cfg, device="cpu")


def test_config_pooling_rule():
    from kandinsky2.model.clip_text import text_tower_config
    cfg = dict(cto.CONFIG_BIGG)
    assert text_tower_config(cfg)["pool_eos"] == -1                   # eos_token_id 2: the argmax rule
    assert text_tower_config(dict(cfg, eos_token_id=49407))["pool_eos"] == 49407
    del cfg["eos_token_id"]
    assert text_tower_config(cfg)["pool_eos"] == 49407                 # transformers' default


def test_tower_refuses_weights_that_do_not_fit_the_config(fx):
    from kandinsky2._native import K2Error
    from kandinsky2.checkpoints import transformers_clip_text_to_k2
    from kandinsky2.model.clip_text import CLIPTextTower
    cfg = fx["towers"][0]["cfg"]
    sd = transformers_clip_text_to_k2(cto.synth_weights(cfg, 0))
    with pytest.raises(K2Error, match="mlp.fc1.weight"):
        CLIPTextTower(sd, dict(cfg, intermediate_size=512), device="cpu")
    with pytest.raises(K2Error, match="token_embedding"):
        CLIPTextTower(sd, dict(cfg, vocab_size=cfg["vocab_size"] + 1), device="cpu")


def test_tower_refuses_bad_ids_and_tokenizers(fx, tok):
    from kandinsky2._native import K2Error
    from kandinsky2.checkpoints import transformers_clip_text_to_k2
    from kandinsky2.model.clip_text import CLIPTextTower, CLIPTokenizer
    cfg = fx["towers"][0]["cfg"]
    sd = transformers_clip_text_to_k2(cto.synth_weights(cfg, 0))
    tower = CLIPTextTower(sd, cfg, device="cpu", tokenizer=tok)       # not finalized: nothing touches a device
    V = cfg["vocab_size"]
    for ids, msg in ((torch.tensor([[0, V]]), r"\[0, 814\)"), (torch.tensor([[-1, 3]]), "must lie in"),
                     (torch.zeros(2, 78, dtype=torch.long), "T <= 77"), (torch.zeros(3, dtype=torch.long), r"\[n, T\]"),
                     (torch.zeros(1, 5), "integers")):
        with pytest.raises(K2Error, match=msg):
            tower.forward(ids)
    with pytest.raises(K2Error, match="tokenizer="):
        CLIPTextTower(sd, cfg, device="cpu")(["a cat"])
    long_tok = CLIPTokenizer(tok.vocab, list(tok.ranks), model_max_length=78)
    with pytest.raises(K2Error, match="model_max_length 78"):
        CLIPTextTower(sd, cfg, device="cpu", tokenizer=long_tok)
    with pytest.raises(K2Error, match="beyond the vocabulary"):
        CLIPTextTower(sd, dict(cfg, vocab_size=V - 1), device="cpu", tokenizer=tok)


# k2_clip_text_embed(ids, ldi, B, T, tok, V, pos, H, out, ldo, stream)
EMBED = dict(ids=P(A), ldi=77, B=2, T=77, tok=P(A), V=49408, pos=P(A), H=1280, out=P(A), ldo=1280, stream=None)


@pytest.mark.parametrize("change,msg", [
    (dict(ids=None), "bad arguments"),
    (dict(tok=None), "bad arguments"),
    (dict(pos=None), "bad arguments"),
    (dict(out=None), "bad arguments"),
    (dict(B=0), "bad arguments"),
    (dict(T=0), "bad arguments"),
    (dict(V=0), "bad arguments"),
    (dict(H=1284, ldo=1288), "multiple of 8"),
    (dict(ldi=76), "row strides"),
    (dict(ldo=1272), "row strides"),
    (dict(ldo=1284), "row strides"),
    (dict(ids=P(A + 2)), "alignment"),
    (dict(tok=P(A + 8)), "alignment"),
    (dict(pos=P(A + 4)), "alignment"),
    (dict(out=P(A + 2)), "alignment"),
])
def test_clip_text_embed_refuses(change, msg):
    _refused("k2_clip_text_embed", list(_with(EMBED, **change).values()), msg)


# k2_clip_text_pool(ids, ldi, B, T, eos_id, hidden, ldh, H, out, ldo, index_out, stream)
POOL = dict(ids=P(A), ldi=77, B=2, T=77, eos_id=49407, hidden=P(A), ldh=1280, H=1280, out=P(A), ldo=1280, index_out=None,
            stream=None)


@pytest.mark.parametrize("change,msg", [
    (dict(ids=None), "bad arguments"),
    (dict(hidden=None), "bad arguments"),
    (dict(out=None), "bad arguments"),
    (dict(B=0), "bad arguments"),
    (dict(T=0), "bad arguments"),
    (dict(H=0), "bad arguments"),
    (dict(ldi=10), "row strides"),
    (dict(ldh=1279), "row strides"),
    (dict(ldo=100), "row strides"),
    (dict(ids=P(A + 2)), "alignment"),
    (dict(out=P(A + 2)), "alignment"),
    (dict(index_out=P(A + 1)), "alignment"),
    (dict(hidden=P(A + 1)), "alignment"),
])
def test_clip_text_pool_refuses(change, msg):
    _refused("k2_clip_text_pool", list(_with(POOL, **change).values()), msg)


def test_live_transformers_second_seed(fx, tok):
    pytest.importorskip("transformers")
    hf = cto.hf_tokenizer(fx["merges"])
    texts = cto.random_prompts(2000, seed=2)
    ids, mask = cto.hf_encode(hf, texts)
    got = tok(texts)
    bad = [t for i, t in enumerate(texts) if not torch.equal(got["input_ids"][i], ids[i])]
    assert not bad, bad[:5]
    assert torch.equal(got["attention_mask"], mask)
    for i in (0, 1):
        cfg = fx["towers"][i]["cfg"]
        sd = cto.synth_weights(cfg, 17)
        x = torch.randint(0, cfg["vocab_size"] - 2, (2, 77), generator=torch.Generator().manual_seed(17))
        x[:, 9], x[1, 4] = cfg["vocab_size"] - 1, cfg["vocab_size"] - 1
        ref = cto.transformers_outputs(dict(sd), cfg, x)
        got = cto.forward(sd, cfg, x)
        assert all(_rel(g, r) <= 1e-5 for g, r in zip(got, ref))
