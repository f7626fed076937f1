"""CPU: the Kandinsky 2.1 CLIP ViT-L/14 pieces that need no GPU (kandinsky2/model/clip_vitl14.py, checkpoints.openai_clip_to_k2):
the oracle against transformers' CLIPModel (tests/golden/openai_clip_tiny.pt), the OpenAI -> kandinsky2 remap through the
network, the loader's refusals and geometry, both checkpoint forms, the reference's CustomizedTokenizer restated (BPE,
padded_tokens_and_mask, text cleaning), the clip image transform against torchvision's output, and k2_quick_gelu_f16's
argument checks."""
import gzip
import json
import os

import pytest
import torch

from tests import openai_clip_oracle as oo
from tests.test_cpu_vector_arg_checks import A, P, _refused


@pytest.fixture(scope="module")
def fx():
    return torch.load(oo.FIXTURE)


def _rel(a, b):
    return ((a - b).norm() / b.norm()).item()


# ---------------------------------------------------------------------------------------------------------------------------
# oracle and remap
# ---------------------------------------------------------------------------------------------------------------------------
def test_oracle_matches_the_transformers_golden(fx):
    sd = oo.synth_weights(fx["geo"], fx["weight_seed"])
    assert torch.equal(oo.sample_tokens(fx["geo"], fx["token_seed"]), fx["tokens"])
    pix = oo.sample_pixels(fx["geo"], fx["pixel_seed"])
    assert oo.sha256(pix) == fx["pixel_sha256"]
    seq, temb = oo.text_forward(sd, fx["tokens"])
    _, iemb = oo.vision_forward(sd, pix)
    for got, ref in ((seq, fx["txt_feat_seq"]), (temb, fx["txt_feat"]), (iemb, fx["image_emb"])):
        assert _rel(got, ref) <= 1e-5


def test_remap_through_the_network(fx):
    """in_proj split and re-packed per head, out_proj / c_fc / c_proj renamed, the projections transposed: the kandinsky2-name
    forward equals the OpenAI-name forward."""
    from kandinsky2.checkpoints import openai_clip_to_k2
    sd = oo.synth_weights(fx["geo"], fx["weight_seed"])
    text, vision, geo = openai_clip_to_k2(dict(sd, logit_scale=torch.tensor(4.6), input_resolution=torch.tensor(56),
                                               context_length=torch.tensor(16), vocab_size=torch.tensor(1000)))
    tok, pix = fx["tokens"], oo.sample_pixels(fx["geo"], fx["pixel_seed"])
    for a, b in zip(oo.text_forward_k2(text, tok), oo.text_forward(sd, tok)):
        assert _rel(a, b) <= 1e-6
    for a, b in zip(oo.vision_forward_k2(vision, pix), oo.vision_forward(sd, pix)):
        assert _rel(a, b) <= 1e-6
    assert torch.equal(text["proj.weight"], sd["text_projection"].t())
    w = text["layers.0.attn.qkv.weight"]
    assert torch.equal(w[64:128], sd["transformer.resblocks.0.attn.in_proj_weight"][128:192])   # head 0's k rows


def test_geometry_from_shapes(fx):
    from kandinsky2.checkpoints import openai_clip_geometry
    g = openai_clip_geometry(oo.synth_weights(fx["geo"], 0))
    assert g["text"] == dict(width=128, layers=2, heads=2, mlp=512, context=16, vocab=1000, embed_dim=96)
    assert g["vision"] == dict(width=128, layers=2, heads=2, mlp=512, patch=14, grid=4, tokens=17, image_size=56, embed_dim=96)
    spec = dict(oo.openai_spec(oo.GEO_L14))
    big = openai_clip_geometry({k: torch.empty(()).expand(*s) for k, s in spec.items()})
    assert big["text"] == dict(width=768, layers=12, heads=12, mlp=3072, context=77, vocab=49408, embed_dim=768)
    assert big["vision"] == dict(width=1024, layers=24, heads=16, mlp=4096, patch=14, grid=16, tokens=257, image_size=224,
                                 embed_dim=768)


@pytest.mark.parametrize("edit,name", [
    (lambda sd: sd.pop("visual.ln_post.bias"), "visual.ln_post.bias"),
    (lambda sd: sd.pop("transformer.resblocks.1.mlp.c_fc.weight"), "transformer.resblocks.1.mlp.c_fc.weight"),
    (lambda sd: sd.update({"visual.attnpool.weight": torch.zeros(1)}), "visual.attnpool.weight"),
    (lambda sd: sd.update({"transformer.resblocks.3.ln_1.weight": torch.zeros(1)}), "transformer.resblocks.3.ln_1.weight"),
    (lambda sd: sd.pop("ln_final.weight"), "ln_final.weight"),
    (lambda sd: sd.pop("text_projection"), "text_projection"),
])
def test_refusals_name_the_key(fx, edit, name):
    from kandinsky2._native import K2Error
    from kandinsky2.checkpoints import openai_clip_to_k2
    sd = oo.synth_weights(fx["geo"], 0)
    edit(sd)
    with pytest.raises(K2Error, match=name.replace(".", r"\.")):
        openai_clip_to_k2(sd)


def test_both_checkpoint_forms_load(fx, tmp_path):
    """A TorchScript archive (what the clip package downloads) and a plain torch.save'd state dict give the same dict."""
    from kandinsky2._native import K2Error
    from kandinsky2.checkpoints import load_openai_clip
    sd = oo.synth_weights(fx["geo"], 5)

    class Holder(torch.nn.Module):
        def __init__(self):
            super().__init__()
            for k, v in sd.items():
                mod = self
                *path, leaf = k.split(".")
                for p in path:
                    if not hasattr(mod, p):
                        mod.add_module(p, torch.nn.Module())
                    mod = getattr(mod, p)
                mod.register_parameter(leaf, torch.nn.Parameter(v.clone(), requires_grad=False))

        def forward(self, x):
            return x

    torch.jit.save(torch.jit.script(Holder()), str(tmp_path / "ViT-tiny.pt"))
    torch.save(sd, tmp_path / "plain.pt")
    for f in ("ViT-tiny.pt", "plain.pt"):
        got = load_openai_clip(str(tmp_path / f))
        assert set(got) == set(sd) and all(torch.equal(got[k], sd[k]) for k in sd), f
    with pytest.raises(K2Error, match="missing.pt"):
        load_openai_clip(str(tmp_path / "missing.pt"))


# ---------------------------------------------------------------------------------------------------------------------------
# tokenizer
# ---------------------------------------------------------------------------------------------------------------------------
WORDS = ("a", "red", "cat", "sitting", "on", "the", "mat", "photo", "of", "dog", "blue", "sky", "4k", "hello", "world")


def _synthetic_bpe(tmp_path):
    """A bpe_simple_vocab-style .txt.gz (a version line, then merges) and the equivalent vocab.json / merges.txt folder."""
    from kandinsky2.model.clip_text import bytes_to_unicode
    merges, have = [], set()
    for w in WORDS:
        syms = list(w[:-1]) + [w[-1] + "</w>"]
        while len(syms) > 1:
            m = (syms[0], syms[1])
            if m not in have:
                have.add(m)
                merges.append(m)
            syms = [syms[0] + syms[1]] + syms[2:]
    chars = list(bytes_to_unicode().values())
    vocab = chars + [c + "</w>" for c in chars] + ["".join(m) for m in merges] + ["<|startoftext|>", "<|endoftext|>"]
    lines = ["\"bpe_simple_vocab_16e6.txt#version: 0.2"] + [" ".join(m) for m in merges]
    gz = tmp_path / "bpe_simple_vocab_16e6.txt.gz"
    with gzip.open(gz, "wb") as fh:
        fh.write(("\n".join(lines) + "\n").encode("utf-8"))
    d = tmp_path / "tok"
    d.mkdir()
    (d / "vocab.json").write_text(json.dumps({v: i for i, v in enumerate(vocab)}), encoding="utf-8")
    (d / "merges.txt").write_text("#version: 0.2\n" + "\n".join(" ".join(m) for m in merges) + "\n", encoding="utf-8")
    return gz, d


def test_from_bpe_matches_clip_tokenizer_on_plain_text(tmp_path):
    from kandinsky2.model.clip_text import CLIPTokenizer
    from kandinsky2.model.clip_vitl14 import OpenAICLIPTokenizer
    gz, d = _synthetic_bpe(tmp_path)
    ours, folder, hf = OpenAICLIPTokenizer.from_bpe(str(gz)), OpenAICLIPTokenizer.from_bpe(str(d)), CLIPTokenizer.from_dir(str(d))
    assert ours.vocab == folder.vocab
    assert len(ours.vocab) == 512 + len(ours.ranks) + 2 and ours.eot_token == len(ours.vocab) - 1
    for text in ("a red cat sitting on the mat", "Photo of a blue dog, 4k!", "hello   world", "sky's", "unknownword 123"):
        assert ours.tokenize_ids(text) == hf.tokenize_ids(text) == folder.tokenize_ids(text), text
    assert ours.tokenize_ids("a cat") == [ours.vocab["a</w>"], ours.vocab["cat</w>"]]


def test_padded_tokens_and_mask(tmp_path):
    from kandinsky2.model.clip_vitl14 import OpenAICLIPTokenizer
    tok = OpenAICLIPTokenizer.from_bpe(str(_synthetic_bpe(tmp_path)[0]))
    sot, eot, cat = tok.sot_token, tok.eot_token, tok.vocab["cat</w>"]
    ids, mask = tok.padded_tokens_and_mask(["", "cat " * 75, "cat " * 80], 77)
    assert ids.dtype == torch.int32 and mask.dtype == torch.bool and ids.shape == mask.shape == (3, 77)
    assert ids[0, :2].tolist() == [sot, eot] and (ids[0, 2:] == 0).all()                     # empty prompt, pads are 0
    assert mask[0].tolist() == [True] * 2 + [False] * 75
    assert ids[1].tolist() == [sot] + [cat] * 75 + [eot] and mask[1].all()                   # exactly 75 tokens fill 77
    assert ids[2].tolist() == [sot] + [cat] * 75 + [eot] and mask[2].all()                   # over-long: eot at 76
    ids, mask = tok.padded_tokens_and_mask(["cat cat"], 3)
    assert ids.tolist() == [[sot, cat, eot]] and mask.tolist() == [[True] * 3]
    assert tok.padded_tokens_and_mask(["<|endoftext|> cat"], 5)[0].tolist() == [[sot, eot, cat, eot, 0]]


@pytest.mark.parametrize("text,want", [
    ("  A  Red\tCAT \n", "a red cat"),
    ("“Quoted” ‘text’ it’s", "\"quoted\" 'text' it's"),
    ("ﬁne ﬂow ĳ", "fine flow ij"),
    ("ＡＢＣ　１２３", "abc 123"),
    ("line\r\nbreak here", "line break here"),
    ("ctrl\x00\x0bchars﻿", "ctrlchars"),
    ("\x1b[31mred\x1b[0m", "red"),
    ("café", "café"),
    ("&amp;amp; &lt;b&gt;", "& <b>"),
    ("\x93c1\x94", "\"c1\""),
])
def test_cleaning(text, want):
    from kandinsky2.model.clip_vitl14 import clean_text
    assert clean_text(text) == want


# ---------------------------------------------------------------------------------------------------------------------------
# preprocessing and argument checks
# ---------------------------------------------------------------------------------------------------------------------------
def test_preprocess_is_torchvisions_clip_transform(fx):
    from kandinsky2.model.clip_vitl14 import preprocess_openai
    for name, img in oo.sample_images():
        x = preprocess_openai(img)[0]
        assert x.dtype == torch.float32 and x.shape == (3, 224, 224)
        assert oo.sha256(x) == fx["preprocess_sha256"][name], name
        assert torch.equal(x[:, :1], fx["preprocess_rows"][name]), name


@pytest.mark.parametrize("x,y,n,msg", [
    (A, A, 7, "even element count"),
    (A, A, 0, "even element count"),
    (A, A, -2, "even element count"),
    (None, A, 8, "even element count"),
    (A + 2, A, 8, "alignment"),
    (A, A + 2, 8, "alignment"),
])
def test_quick_gelu_f16_refuses(x, y, n, msg):
    _refused("k2_quick_gelu_f16", [P(x) if x is not None else None, P(y), n, None], msg)


def test_ops_refuse_cpu_tensors():
    from kandinsky2 import ops
    from kandinsky2._native import K2Error
    with pytest.raises(K2Error, match="no CPU fallback"):
        ops.quick_gelu_f16_(torch.zeros(4, dtype=torch.float16))


def test_prior_embedder_from_pretrained_names_a_missing_file(tmp_path):
    from kandinsky2._native import K2Error
    from kandinsky2.model.prior import PriorEmbedder
    with pytest.raises(K2Error, match=os.path.join(str(tmp_path), "prior_fp16.ckpt")):
        PriorEmbedder.from_pretrained(str(tmp_path), device="cpu")
