"""CPU: the Kandinsky 2.1 text encoder's host side.  kandinsky2's XLMRobertaTokenizer against transformers' input_ids and
attention masks in tests/golden/xlmr_tiny.pt (and tokenizers' for the legacy tokenizer.json layout), the restated forward
(tests/xlmr_oracle.py) against transformers' own outputs, the M-CLIP state-dict remap through the network, the config / remap /
tokenizer refusals, K2Error without a device, and the two new C-ABI entry points' argument checks (nothing is launched).  Where
transformers and tokenizers are importable, 2000 more strings and a second weight seed run against them live."""
import json

import pytest
import torch

from tests import xlmr_oracle as xo
from tests.test_cpu_vector_arg_checks import A, P, _refused, _with


@pytest.fixture(scope="module")
def fx():
    return torch.load(xo.FIXTURE)


@pytest.fixture(scope="module")
def tok(fx):
    return xo.k2_tokenizer(xo.fixture_json(fx))


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


@pytest.mark.parametrize("legacy", [False, True])
def test_tokenizer_reproduces_every_fixture_text(fx, legacy):
    t = xo.k2_tokenizer(xo.fixture_json(fx, legacy))
    ids, mask = xo.unpack_ids(*((fx["legacy_ids"], fx["legacy_lengths"]) if legacy else (fx["ids"], fx["lengths"])))
    assert len(fx["texts"]) == ids.shape[0] > 230
    got = t(fx["texts"])
    bad = [repr(x) for i, x in enumerate(fx["texts"]) if not torch.equal(got["input_ids"][i], ids[i])]
    assert not bad, bad[:5]
    assert torch.equal(got["attention_mask"], mask)


def test_tokenizer_edge_cases(fx, tok):
    """The cases the fixture was built around, spelled out."""
    enc = lambda t: tok([t])["input_ids"][0]  # noqa: E731
    mask_id = tok.added["<mask>"][0]
    assert enc("").tolist()[:3] == [0, 2, xo.PAD_ID] and tok([""])["attention_mask"][0].sum() == 2
    assert enc(" \t\n ").tolist()[:2] == [0, 2]                              # whitespace only: no token
    assert mask_id in enc("a <mask> b").tolist() and mask_id in enc("a<mask>b").tolist()
    assert enc("<s>").tolist()[:3] == [0, 0, 2]                              # a literal special in the raw text
    x75 = tok(["x " * 75])
    assert x75["attention_mask"][0].sum() == 77 and x75["input_ids"][0, -1] == 2
    assert torch.equal(tok(["x " * 80 + "tail"])["input_ids"], x75["input_ids"])   # truncated to 75 tokens + </s>
    legacy = xo.k2_tokenizer(xo.fixture_json(fx, legacy=True))
    assert legacy.added["<mask>"][1] and not tok.added["<mask>"][1]               # lstrip in the legacy layout only
    assert legacy.tokenize_ids("a  <mask>") == legacy.tokenize_ids("a<mask>")     # lstrip takes the white space


def test_grapheme_clusters():
    from kandinsky2.model.text_encoders import _graphemes
    assert _graphemes("a\r\nb") == ["a", "\r\n", "b"]
    assert _graphemes("e\u0301x") == ["e\u0301", "x"]
    assert _graphemes("\x01\u0301") == ["\x01", "\u0301"]                          # no extending a control
    assert _graphemes("\U0001f469\u200d\U0001f469\u200d\U0001f467!") == ["\U0001f469\u200d\U0001f469\u200d\U0001f467", "!"]
    assert _graphemes("\U0001f1ef\U0001f1f5\U0001f1fa\U0001f1f8\U0001f1e9") == [
        "\U0001f1ef\U0001f1f5", "\U0001f1fa\U0001f1f8", "\U0001f1e9"]
    assert _graphemes("\u1100\u1161\u11a8\uac01") == ["\u1100\u1161\u11a8", "\uac01"]     # jamo L V T, then LVT
    assert _graphemes("\u0600a") == ["\u0600a"] and _graphemes("a\u0903") == ["a\u0903"]   # Prepend, SpacingMark


def test_tokenizer_from_dir(fx, tmp_path):
    from kandinsky2._native import K2Error
    from kandinsky2.model.text_encoders import XLMRobertaTokenizer
    (tmp_path / "tokenizer.json").write_text(xo.fixture_json(fx), encoding="utf-8")
    t = XLMRobertaTokenizer.from_dir(str(tmp_path))
    assert t.model_max_length == 77 and t.pad_token_id == xo.PAD_ID and t.prefix == [0] and t.suffix == [2]
    ref = xo.k2_tokenizer(xo.fixture_json(fx))(fx["texts"][:40])
    assert torch.equal(t(fx["texts"][:40])["input_ids"], ref["input_ids"])
    (tmp_path / "special_tokens_map.json").write_text(json.dumps({"pad_token": {"content": "</s>"}}))
    assert XLMRobertaTokenizer.from_dir(str(tmp_path)).pad_token_id == 2
    (tmp_path / "special_tokens_map.json").write_text(json.dumps({"pad_token": "<nope>"}))
    with pytest.raises(K2Error, match="<nope>"):
        XLMRobertaTokenizer.from_dir(str(tmp_path))
    (tmp_path / "tokenizer.json").unlink()
    with pytest.raises(K2Error, match="tokenizer.json"):
        XLMRobertaTokenizer.from_dir(str(tmp_path))


@pytest.mark.parametrize("path,value,msg", [
    (("normalizer",), {"type": "NFKC"}, "normalizer 'NFKC'"),
    (("normalizer",), {"type": "Replace", "pattern": {"Other": "x"}, "content": ""}, "Replace pattern"),
    (("pre_tokenizer",), {"type": "ByteLevel"}, "pre-tokenizer 'ByteLevel'"),
    (("pre_tokenizer", "pretokenizers", 1, "prepend_scheme"), "first", "prepend_scheme 'first'"),
    (("model", "type"), "BPE", "model 'BPE'"),
    (("model", "byte_fallback"), True, "byte_fallback"),
    (("post_processor",), {"type": "BertProcessing"}, "post-processor 'BertProcessing'"),
    (("added_tokens", 4, "single_word"), True, "single_word"),
])
def test_tokenizer_refuses_unimplemented_kinds(fx, path, value, msg):
    from kandinsky2._native import K2Error
    from kandinsky2.model.text_encoders import XLMRobertaTokenizer
    spec = json.loads(xo.fixture_json(fx))
    node = spec
    for k in path[:-1]:
        node = node[k]
    node[path[-1]] = value
    with pytest.raises(K2Error, match=msg):
        XLMRobertaTokenizer(spec)


@pytest.mark.parametrize("i", [0, 1])
def test_oracle_equals_transformers_golden(fx, i):
    t = fx["towers"][i]
    sd = xo.synth_weights(t["cfg"], t["out_features"], t["weight_seed"])
    hid, pooled = xo.forward(sd, t["cfg"], t["input_ids"].long(), t["attention_mask"].long())
    assert _rel(hid, t["last_hidden_state"]) <= 1e-5 and _rel(pooled, t["pooled"]) <= 1e-5


def test_golden_towers_use_the_tokenizer(fx, tok):
    for t in fx["towers"]:
        e = tok(t["prompts"])
        assert torch.equal(e["input_ids"], t["input_ids"].long()) and torch.equal(e["attention_mask"], t["attention_mask"].long())
    assert (fx["towers"][1]["input_ids"][0] == xo.PAD_ID).sum() > (1 - fx["towers"][1]["attention_mask"][0]).sum()  # a literal <pad>


@pytest.mark.parametrize("i", [0, 1])
def test_remapped_forward_equals_reference_names(fx, i):
    from kandinsky2.checkpoints import mclip_to_k2
    t = fx["towers"][i]
    sd = xo.synth_weights(t["cfg"], t["out_features"], t["weight_seed"])
    sd_pos = dict(sd, **{"transformer.embeddings.position_ids": torch.arange(80)[None]})   # ignored, as the pooler
    k2 = mclip_to_k2(sd_pos, t["cfg"]["num_hidden_layers"])
    ids, mask = t["input_ids"].long(), t["attention_mask"].long()
    for x, y in zip(xo.forward(sd, t["cfg"], ids, mask), xo.forward_k2(k2, t["cfg"], ids, mask)):
        assert _rel(y, x) <= 1e-6


def test_remap_refuses_missing_and_unexpected_keys(fx):
    from kandinsky2._native import K2Error
    from kandinsky2.checkpoints import mclip_to_k2
    cfg = fx["towers"][0]["cfg"]
    sd = xo.synth_weights(cfg, 32, 0)
    gone = "transformer.encoder.layer.1.output.LayerNorm.bias"
    with pytest.raises(K2Error, match=gone.replace(".", r"\.")):
        mclip_to_k2({k: v for k, v in sd.items() if k != gone}, 2)
    with pytest.raises(K2Error, match="LinearTransformation.weight"):
        mclip_to_k2({k: v for k, v in sd.items() if k != "LinearTransformation.weight"}, 2)
    with pytest.raises(K2Error, match=r"encoder\.layer\.1\."):
        mclip_to_k2(sd, 1)                                                  # a layer beyond the config
    with pytest.raises(K2Error, match="lm_head"):
        mclip_to_k2(dict(sd, **{"lm_head.bias": torch.zeros(2)}), 2)


@pytest.mark.parametrize("change,msg", [
    (dict(hidden_act="gelu_new"), "hidden_act"),
    (dict(hidden_size=96, intermediate_size=256), "head width 48"),
    (dict(position_embedding_type="relative_key"), "position_embedding_type"),
    (dict(type_vocab_size=2), "type_vocab_size 2"),
    (dict(type_vocab_size=None), "type_vocab_size 2"),                      # transformers' default
    (dict(vocab_size=None), "missing"),
    (dict(max_position_embeddings=40), "at most 38"),
])
def test_from_state_dict_refuses_unimplemented_configs(fx, tok, change, msg):
    from kandinsky2._native import K2Error
    from kandinsky2.model.text_encoders import MultilingualCLIP
    base = fx["towers"][0]["cfg"]
    cfg = dict(base, **change)
    for k in [k for k, v in cfg.items() if v is None]:
        del cfg[k]
    with pytest.raises(K2Error, match=msg):
        MultilingualCLIP.from_state_dict(xo.synth_weights(base, 32, 0), cfg, tokenizer=tok, device="cpu")


def test_config_reads_the_large_geometry():
    from kandinsky2.model.text_encoders import xlmr_config
    c = xlmr_config(xo.CONFIG_LARGE)
    assert (c["max_tokens"], c["pad_token_id"], c["layer_norm_eps"], c["head_dim"]) == (128, 1, 1e-5, 64)


def test_tower_refusals_without_a_device(fx, tok):
    from kandinsky2._native import K2Error
    from kandinsky2.checkpoints import mclip_to_k2
    from kandinsky2.model.text_encoders import MultilingualCLIP, TextEncoder
    cfg = fx["towers"][0]["cfg"]
    sd = mclip_to_k2(xo.synth_weights(cfg, 32, 0), 2)
    with pytest.raises(K2Error, match="mlp.fc1.weight"):
        MultilingualCLIP(sd, dict(cfg, intermediate_size=512), device="cpu")
    tower = MultilingualCLIP(sd, cfg, device="cpu", tokenizer=tok)        # not finalized: nothing touches a device
    assert tower.out_features == 32 and tower.tokens == 77
    V = cfg["vocab_size"]
    one = torch.ones(1, 2, dtype=torch.long)
    for ids, mask, msg in ((torch.tensor([[0, V]]), one, rf"\[0, {V}\)"), (torch.tensor([[-1, 3]]), one, "must lie in"),
                           (torch.zeros(2, 129, dtype=torch.long), torch.ones(2, 129), r"T <= 79"),
                           (torch.zeros(3, dtype=torch.long), one, r"\[n, T\]"), (torch.zeros(1, 2), one, "integers"),
                           (torch.zeros(1, 2, dtype=torch.long), torch.ones(1, 3), "attention_mask"),
                           (torch.zeros(1, 2, dtype=torch.long), torch.ones(1, 2), "attention_mask")):
        with pytest.raises(K2Error, match=msg):
            tower.forward(ids, mask)
    with pytest.raises(K2Error, match="tokenizer="):
        MultilingualCLIP(sd, cfg, device="cpu")("a cat", 1)
    with pytest.raises(K2Error, match="beyond the vocabulary"):
        MultilingualCLIP(mclip_to_k2(xo.synth_weights(dict(cfg, vocab_size=V - 1), 32, 0), 2), dict(cfg, vocab_size=V - 1),
                         device="cpu", tokenizer=tok)
    with pytest.raises(K2Error, match="pads with 1"):
        MultilingualCLIP(sd, dict(cfg, pad_token_id=0), device="cpu", tokenizer=tok)
    with pytest.raises(K2Error, match="model_name 'clip'"):
        TextEncoder("/nonexistent", model_name="clip")
    with pytest.raises(K2Error, match="config.json"):
        TextEncoder("/nonexistent")


# k2_xlmr_embed(ids, ldi, B, T, pad_id, word, V, pos, P, type_row, gamma, beta, eps, out, ldo, H, stream)
EMBED = dict(ids=P(A), ldi=77, B=2, T=77, pad_id=1, word=P(A), V=250002, pos=P(A), P=514, type_row=P(A), gamma=P(A),
             beta=P(A), eps=1e-5, out=P(A), ldo=1024, H=1024, stream=None)


@pytest.mark.parametrize("change,msg", [
    (dict(ids=None), "bad arguments"),
    (dict(word=None), "bad arguments"),
    (dict(pos=None), "bad arguments"),
    (dict(type_row=None), "bad arguments"),
    (dict(gamma=None), "bad arguments"),
    (dict(beta=None), "bad arguments"),
    (dict(out=None), "bad arguments"),
    (dict(B=0), "bad arguments"),
    (dict(T=0), "bad arguments"),
    (dict(V=0), "bad arguments"),
    (dict(P=0), "bad arguments"),
    (dict(H=0), "bad arguments"),
    (dict(pad_id=-1), "pad_id"),
    (dict(H=8200, ldo=8200), "at most 8192"),
    (dict(ldi=76), "row strides"),
    (dict(ldo=1000), "row strides"),
    (dict(eps=0.0), "eps"),
    (dict(ids=P(A + 2)), "alignment"),
    (dict(gamma=P(A + 2)), "alignment"),
    (dict(beta=P(A + 2)), "alignment"),
    (dict(word=P(A + 1)), "alignment"),
    (dict(pos=P(A + 1)), "alignment"),
    (dict(type_row=P(A + 1)), "alignment"),
    (dict(out=P(A + 1)), "alignment"),
])
def test_xlmr_embed_refuses(change, msg):
    _refused("k2_xlmr_embed", list(_with(EMBED, **change).values()), msg)


# k2_masked_mean_f16(hidden, ldh, mask, ldm, B, T, H, out, ldo, stream)
MEAN = dict(hidden=P(A), ldh=1024, mask=P(A), ldm=77, B=2, T=77, H=1024, out=P(A), ldo=1024, stream=None)


@pytest.mark.parametrize("change,msg", [
    (dict(hidden=None), "bad arguments"),
    (dict(mask=None), "bad arguments"),
    (dict(out=None), "bad arguments"),
    (dict(B=0), "bad arguments"),
    (dict(T=0), "bad arguments"),
    (dict(H=0), "bad arguments"),
    (dict(ldh=1000), "row strides"),
    (dict(ldm=76), "row strides"),
    (dict(ldo=1000), "row strides"),
    (dict(B=65536), "65535"),
    (dict(hidden=P(A + 1)), "alignment"),
    (dict(out=P(A + 2)), "alignment"),
])
def test_masked_mean_refuses(change, msg):
    _refused("k2_masked_mean_f16", list(_with(MEAN, **change).values()), msg)


def test_live_transformers_more_strings(fx, tok):
    pytest.importorskip("transformers")
    pytest.importorskip("tokenizers")
    texts = xo.random_prompts(2000, seed=2)
    text = xo.fixture_json(fx)
    for layout in (text, xo.legacy_json(text)):
        ids, mask = xo.tokenizers_encode(layout, texts)
        got = xo.k2_tokenizer(layout)(texts)
        bad = [repr(t) for i, t in enumerate(texts) if not torch.equal(got["input_ids"][i], ids[i])]
        assert not bad, bad[:5]
        assert torch.equal(got["attention_mask"], mask)
    for t in fx["towers"]:
        cfg = t["cfg"]
        sd = xo.synth_weights(cfg, t["out_features"], 17)
        e = tok(["a red cat " * 3, "", "x <pad> y"])
        ref = xo.transformers_outputs(sd, cfg, e["input_ids"], e["attention_mask"])
        got = xo.forward(sd, cfg, e["input_ids"], e["attention_mask"])
        assert all(_rel(g, r) <= 1e-5 for g, r in zip(got, ref))
