"""TEST INFRASTRUCTURE (oracle): the Kandinsky 2.1 text encoder -- the reference's MultilingualCLIP (transformers'
XLMRobertaModel + LinearTransformation) restated from the math in torch, a tiny SentencePiece tokenizer loaded through
transformers, and the writer of the golden fixture tests/golden/xlmr_tiny.pt:

    python -m tests.xlmr_oracle

  train_spm            <- a unigram SentencePiece model over CORPUS (nmt_nfkc, fixed seed, one thread)
  hf_tokenizer_json    <- the tokenizer.json transformers 5 writes for it (XLMRobertaTokenizer.from_pretrained)
  legacy_json          <- the older layout of the same tokenizer: normalizer Sequence[Precompiled, Replace(" {2,}" -> " ")],
                          a bare Metaspace with add_prefix_space, <mask> with lstrip
  mclip_spec           <- the reference's MultilingualCLIP state dict of a config (key names as torch writes them)
  forward              <- MultilingualCLIP.forward from those names: word + token type + position embedding (positions from
                          the ids, transformers' create_position_ids_from_input_ids), LayerNorm, post-LN encoder layers
                          (eager attention, padded keys masked, exact GELU), the masked mean and the Linear.
                          dtype=torch.float16 rounds where the halved reference model does (fp16 inputs to every op, softmax
                          in fp32 then rounded, the pooling in fp16).
  forward_k2           <- the same network from kandinsky2's names (checkpoints.mclip_to_k2), fp32

The fixture holds the tokenizer.json (xz-compressed: almost all of it is the charsmap; legacy_json derives the other
layout from it), transformers' ids for every text
(fixed edge cases and seeded random strings), tokenizers' ids for the legacy layout, and for two tiny towers their config,
weight seed, ids / mask and transformers' fp32 outputs.  Before writing, the generator asserts that kandinsky2's
XLMRobertaTokenizer reproduces both layouts and that the oracle is within 1e-5 of transformers."""
import io
import json
import lzma
import os
import random
import tempfile

import torch
import torch.nn.functional as F

from oracle import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "xlmr_tiny.pt")
MAX_LENGTH = 77
PAD_ID = 1

# XLM-RoBERTa-large as the M-CLIP text encoder is expected to configure it (not checked against the released file)
CONFIG_LARGE = dict(vocab_size=250002, hidden_size=1024, intermediate_size=4096, num_hidden_layers=24, num_attention_heads=16,
                    max_position_embeddings=514, type_vocab_size=1, hidden_act="gelu", layer_norm_eps=1e-5, pad_token_id=1,
                    bos_token_id=0, eos_token_id=2, position_embedding_type="absolute")
OUT_LARGE = 768

CORPUS = (
    "a photo of a red cat sitting on the table, 4k, highly detailed, trending on artstation",
    "A capybara, 4k photo. The capybara's fur is wet; it's raining and we'll see the sunset.",
    "lowres, text, error, cropped, worst quality, low quality, jpeg artifacts, ugly, duplicate, blurry, watermark",
    "portrait of an old man with a beard, oil painting, dramatic lighting, by a famous painter",
    "ein Hund läuft über die Straße und bellt laut, schöne Grüße aus München",
    "une maison près de la mer, été, lumière dorée, peinture à l'huile",
    "красивый пейзаж с горами и озером на закате, фотография",
    "η οδός του ήλιου, ΟΔΟΣ, φως και θάλασσα",
    "一只猫坐在桌子上，高清照片，日落时分的城市",
    "富士山と桜の花、美しい風景写真",
    "한국어 문장입니다 고양이가 탁자 위에 앉아 있다",
    "🐱🐶 emoji party 🎉🎉 with 123 balloons and 4567 stars!!!",
    "numbers 0 1 2 3 4 5 6 7 8 9 10 100 1000 2023 3.14159",
    "cyberpunk city at night, neon lights, rain, reflections, cinematic, 8k, unreal engine",
    "watercolor painting of a fox in the forest, soft colors, misty morning",
    "मेज पर बैठी एक बिल्ली की तस्वीर",
    "صورة قطة تجلس على الطاولة",
)


# ---------------------------------------------------------------------------------------------------------------------------
# tokenizer
# ---------------------------------------------------------------------------------------------------------------------------
def train_spm():
    import sentencepiece as spm
    buf = io.BytesIO()
    spm.SentencePieceTrainer.train(sentence_iterator=iter(CORPUS * 4), model_writer=buf, vocab_size=400,
                                   model_type="unigram", normalization_rule_name="nmt_nfkc", num_threads=1,
                                   hard_vocab_limit=False, character_coverage=1.0, minloglevel=2)
    return buf.getvalue()


def hf_tokenizer(model_bytes):
    """transformers 5's XLMRobertaTokenizer over the SentencePiece model, read as the reference reads its folder."""
    from transformers import XLMRobertaTokenizer
    d = tempfile.mkdtemp()
    with open(os.path.join(d, "sentencepiece.bpe.model"), "wb") as f:
        f.write(model_bytes)
    return XLMRobertaTokenizer.from_pretrained(d)


def hf_tokenizer_json(tok):
    d = tempfile.mkdtemp()
    tok.save_pretrained(d)
    with open(os.path.join(d, "tokenizer.json"), encoding="utf-8") as f:
        return f.read()


def legacy_json(text):
    """The older tokenizer.json layout of the same model (transformers 4's XLM-R converter)."""
    j = json.loads(text)
    pre = j["normalizer"]
    assert pre["type"] == "Precompiled", pre["type"]
    j["normalizer"] = {"type": "Sequence", "normalizers": [pre, {"type": "Replace", "pattern": {"Regex": " {2,}"},
                                                                 "content": " "}]}
    j["pre_tokenizer"] = {"type": "Metaspace", "replacement": "▁", "add_prefix_space": True}
    for t in j["added_tokens"]:
        if t["content"] == "<mask>":
            t["lstrip"] = True
    return json.dumps(j, ensure_ascii=False)


def fixed_prompts():
    return [
        "", " ", "\t\n  \t", "a\t\tb\n\nc   d", "a\r\nb\rc\n", "\x00\x01a\x7f\x1c\x1f", "a\u0085b\u2028c", "\u200b\u200c\u200d",
        "a\u200db", "a\u200cb", "\u00a0x\u3000y\u2003z", "A RED CAT", "ΟΔΟΣ οδος", "İstanbul İ ı",
        "e\u0301 cafe\u0301 CAFE\u0301 é", "a\u0301\u0302\u0303\u0304", "Ａ\u0301 ａ\u0308", "n\u0303 ñ",
        "一只猫坐在桌子上", "한국어 각 한", "🐱🐶🎉 emoji 👩\u200d👩\u200d👧 👍🏽 ❤\ufe0f #\ufe0f\u20e3",
        "🇯🇵🇺🇸🇩", "ﬁne ｆｕｌｌｗｉｄｔｈ Ⅻ ½ ² ㍿ ㈱ ℌ", "ｶﾞｷﾞ ｱﾞ", "1234567890 3.14159 2023 ①②",
        "it's we'll they're", "wow!!! ... ?!?! --- (()) [[]] {{}}", "a <mask> b", "a<mask>b", "<mask>", "  <mask>  x",
        "<s> x </s> <pad> <unk>", "<S> <MASK> ＜s＞", "\u0600a क\u094dष กำ", "म\u0947ज पर ब\u0948ठी",
        "صورة قطة", "x " * 75, "x " * 80 + "tail", "A capybara, 4k photo", "red cat",
        "lowres, text, error, cropped, worst quality, low quality, jpeg artifacts, ugly, duplicate, morbid, mutilated, out of "
        "frame, extra fingers, mutated hands, poorly drawn hands, poorly drawn face, mutation, deformed, blurry, dehydrated, "
        "bad anatomy, bad proportions, extra limbs, cloned face, disfigured, gross proportions, malformed limbs, missing arms",
    ]


_PIECES = (list("abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789") + list(" \t\n\r  ") +
           list(".,!?;:'\"-()[]{}<>|/\\@#$%^&*_+=~`") + list("äöüßéèêàçñåøÄÖÜÉ") + list("αβγδεζηθΣσςΩΟΔ") +
           list("абвгдеёжзийклмнопрстуфхцчшщъыьэюяЖЯ") + list("猫狗日本語中文漢字かなカナ한국어") + ["🐱", "🎉", "👩\u200d👩\u200d👧", "🇯🇵", "👍🏽"] +
           ["\x00", "\x1c", "\x1f", "\x7f", "\u0085", "\u200b", "\u200c", "\u200d", "\u00a0", "\u3000", "\u0301", "\u0308",
            "\u20e3", "\ufe0f", "İ", "ﬁ", "Ⅻ", "½", "ｱ", "ﾞ", "Ａ", "ᄀ", "ᅡ", "ᆨ", "क", "\u094d",
            "ำ", "\u0600", "힣", "\U0001d400"] +
           ["<mask>", "<s>", "</s>", "<pad>", "cat", "the ", "photo", "capybara", "  ", "\r\n"])


def random_prompts(n, seed):
    rng = random.Random(seed)
    return ["".join(rng.choice(_PIECES) for _ in range(rng.randint(0, 40))) for _ in range(n)]


def hf_encode(tok, texts):
    """transformers: encode_text's call (max_length 77, padding to it, truncation)."""
    e = tok(texts, padding="max_length", max_length=MAX_LENGTH, truncation=True, return_tensors="pt")
    return e["input_ids"].long(), e["attention_mask"].long()


def tokenizers_encode(text_json, texts):
    """tokenizers directly on a tokenizer.json, truncated and padded as encode_text asks."""
    from tokenizers import Tokenizer
    t = Tokenizer.from_str(text_json)
    t.enable_truncation(MAX_LENGTH)
    t.enable_padding(length=MAX_LENGTH, pad_id=PAD_ID, pad_token="<pad>")
    enc = t.encode_batch(texts)
    return (torch.tensor([e.ids for e in enc], dtype=torch.long),
            torch.tensor([e.attention_mask for e in enc], dtype=torch.long))


def k2_tokenizer(text_json):
    from kandinsky2.model.text_encoders import XLMRobertaTokenizer
    return XLMRobertaTokenizer(json.loads(text_json), model_max_length=MAX_LENGTH)


def pack_ids(ids, mask):
    """[n, L] ids and mask -> (concatenated rows up to their mask's length, int16; lengths, int16)."""
    lengths = mask.sum(1)
    assert torch.equal(mask, (torch.arange(ids.shape[1])[None] < lengths[:, None]).long())
    return torch.cat([ids[i, :lengths[i]] for i in range(ids.shape[0])]).to(torch.int16), lengths.to(torch.int16)


def unpack_ids(flat, lengths, pad_id=PAD_ID, L=MAX_LENGTH):
    """Inverse of pack_ids -> (input_ids int64 [n, L], attention_mask int64 [n, L])."""
    n = lengths.shape[0]
    ids = torch.full((n, L), pad_id, dtype=torch.int64)
    mask = torch.zeros(n, L, dtype=torch.int64)
    at = 0
    for i, ln in enumerate(lengths.tolist()):
        ids[i, :ln] = flat[at:at + ln].long()
        mask[i, :ln] = 1
        at += ln
    return ids, mask


def fixture_json(fx, legacy=False):
    """The fixture's tokenizer.json text, or its legacy_json layout."""
    text = lzma.decompress(fx["tokenizer_json"]).decode("utf-8")
    return legacy_json(text) if legacy else text


# ---------------------------------------------------------------------------------------------------------------------------
# tower
# ---------------------------------------------------------------------------------------------------------------------------
def tiny_config(vocab_size, layers=2, eps=1e-5):
    return dict(vocab_size=vocab_size, hidden_size=128, intermediate_size=256, num_hidden_layers=layers, num_attention_heads=2,
                max_position_embeddings=MAX_LENGTH + PAD_ID + 3, type_vocab_size=1, hidden_act="gelu", layer_norm_eps=eps,
                pad_token_id=PAD_ID, bos_token_id=0, eos_token_id=2, position_embedding_type="absolute")


def mclip_spec(cfg, out_features, pooler=True):
    H, I = cfg["hidden_size"], cfg["intermediate_size"]
    p = "transformer."
    spec = [(p + "embeddings.word_embeddings.weight", (cfg["vocab_size"], H)),
            (p + "embeddings.position_embeddings.weight", (cfg["max_position_embeddings"], H)),
            (p + "embeddings.token_type_embeddings.weight", (cfg["type_vocab_size"], H)),
            (p + "embeddings.LayerNorm.weight", (H,)), (p + "embeddings.LayerNorm.bias", (H,))]
    for i in range(cfg["num_hidden_layers"]):
        lp = f"{p}encoder.layer.{i}."
        for n in ("attention.self.query", "attention.self.key", "attention.self.value", "attention.output.dense"):
            spec += [(f"{lp}{n}.weight", (H, H)), (f"{lp}{n}.bias", (H,))]
        spec += [(lp + "attention.output.LayerNorm.weight", (H,)), (lp + "attention.output.LayerNorm.bias", (H,)),
                 (lp + "intermediate.dense.weight", (I, H)), (lp + "intermediate.dense.bias", (I,)),
                 (lp + "output.dense.weight", (H, I)), (lp + "output.dense.bias", (H,)),
                 (lp + "output.LayerNorm.weight", (H,)), (lp + "output.LayerNorm.bias", (H,))]
    if pooler:
        spec += [(p + "pooler.dense.weight", (H, H)), (p + "pooler.dense.bias", (H,))]
    return spec + [("LinearTransformation.weight", (out_features, H)), ("LinearTransformation.bias", (out_features,))]


def synth_weights(cfg, out_features, seed, pooler=True):
    return synth.synth_state_dict(mclip_spec(cfg, out_features, pooler), seed=seed)


def position_ids(ids, pad_id):
    """transformers' create_position_ids_from_input_ids."""
    m = ids.ne(pad_id).long()
    return torch.cumsum(m, dim=1) * m + pad_id


def _tower(emb, mask, layers, proj, cfg, dtype):
    """emb [B, T, H] (embedding LayerNorm output); layers: per layer ((wq, bq), (wk, bk), (wv, bv), (wo, bo), ln1, fc1, fc2,
    ln2) -> (last_hidden_state, pooled), fp32."""
    H, eps, heads = cfg["hidden_size"], cfg["layer_norm_eps"], cfg["num_attention_heads"]
    B, T, _ = emb.shape
    d = H // heads
    keep = mask.to(emb.device).bool()
    h = emb
    for q, k, v, o, ln1, fc1, fc2, ln2 in layers:
        qh, kh, vh = (F.linear(h, *w).view(B, T, heads, d).transpose(1, 2) for w in (q, k, v))
        w = torch.matmul(qh, kh.transpose(-1, -2)) * d ** -0.5
        w = torch.softmax(w.float().masked_fill(~keep[:, None, None, :], float("-inf")), dim=-1).to(dtype)
        a = torch.matmul(w, vh).transpose(1, 2).reshape(B, T, H)
        h = F.layer_norm(h + F.linear(a, *o), (H,), *ln1, eps=eps)
        h = F.layer_norm(h + F.linear(F.gelu(F.linear(h, *fc1)), *fc2), (H,), *ln2, eps=eps)
    m = mask.to(h.device).to(dtype)
    pooled = (h * m[..., None]).sum(dim=1) / m.sum(dim=1)[:, None]
    return h.float(), F.linear(pooled, *proj).float()


def forward(sd, cfg, ids, mask, dtype=torch.float32):
    """The reference's names, ids / mask [B, T] -> (last_hidden_state [B, T, H], pooled [B, out]), both fp32."""
    sd = {k: v.to(dtype) for k, v in sd.items()}
    p = "transformer."
    g = lambda n: (sd[n + ".weight"], sd[n + ".bias"])  # noqa: E731
    dev = sd[p + "embeddings.word_embeddings.weight"].device
    ids = ids.to(dev).long()
    pos = position_ids(ids, cfg["pad_token_id"])
    emb = sd[p + "embeddings.word_embeddings.weight"][ids] + sd[p + "embeddings.token_type_embeddings.weight"][0]
    emb = emb + sd[p + "embeddings.position_embeddings.weight"][pos]
    emb = F.layer_norm(emb, (cfg["hidden_size"],), *g(p + "embeddings.LayerNorm"), eps=cfg["layer_norm_eps"])
    layers = []
    for i in range(cfg["num_hidden_layers"]):
        lp = f"{p}encoder.layer.{i}."
        layers.append((g(lp + "attention.self.query"), g(lp + "attention.self.key"), g(lp + "attention.self.value"),
                       g(lp + "attention.output.dense"), g(lp + "attention.output.LayerNorm"), g(lp + "intermediate.dense"),
                       g(lp + "output.dense"), g(lp + "output.LayerNorm")))
    return _tower(emb, mask, layers, g("LinearTransformation"), cfg, dtype)


def forward_k2(sd, cfg, ids, mask):
    """kandinsky2 names (attn.qkv packed per head [q_h | k_h | v_h]) -> the same outputs as forward, fp32."""
    H, heads = cfg["hidden_size"], cfg["num_attention_heads"]
    d = H // heads
    g = lambda n: (sd[n + ".weight"].float(), sd[n + ".bias"].float())  # noqa: E731
    ids = ids.long()
    pos = position_ids(ids, cfg["pad_token_id"])
    emb = sd["word_embedding"].float()[ids] + sd["token_type_embedding"].float()[0] + sd["position_embedding"].float()[pos]
    emb = F.layer_norm(emb, (H,), *g("emb_ln"), eps=cfg["layer_norm_eps"])
    layers = []
    for i in range(cfg["num_hidden_layers"]):
        w, b = g(f"layers.{i}.attn.qkv")
        wq, wk, wv = (w.view(heads, 3, d, H)[:, j].reshape(H, H) for j in range(3))
        bq, bk, bv = (b.view(heads, 3, d)[:, j].reshape(H) for j in range(3))
        p = f"layers.{i}."
        layers.append(((wq, bq), (wk, bk), (wv, bv), g(p + "attn.proj"), g(p + "ln_1"), g(p + "mlp.fc1"), g(p + "mlp.fc2"),
                       g(p + "ln_2")))
    return _tower(emb, mask, layers, g("proj"), cfg, torch.float32)


def transformers_outputs(sd, cfg, ids, mask):
    """transformers' own XLMRobertaModel (eager attention, fp32) + the Linear, as MultilingualCLIP.forward runs them."""
    from transformers import XLMRobertaConfig, XLMRobertaModel
    model = XLMRobertaModel(XLMRobertaConfig(**cfg, attn_implementation="eager")).eval()
    model.load_state_dict({k[len("transformer."):]: v for k, v in sd.items() if k.startswith("transformer.")}, strict=True)
    lin = torch.nn.Linear(cfg["hidden_size"], sd["LinearTransformation.weight"].shape[0])
    lin.load_state_dict({"weight": sd["LinearTransformation.weight"], "bias": sd["LinearTransformation.bias"]})
    with torch.no_grad():
        embs = model(input_ids=ids, attention_mask=mask)[0]
        pooled = (embs * mask.unsqueeze(2)).sum(dim=1) / mask.sum(dim=1)[:, None]
        return embs.float(), lin(pooled).float()


TOWERS = ((dict(layers=2, eps=1e-5), 32, ("A capybara, 4k photo", "red cat", "")),
          (dict(layers=3, eps=1e-12), 48, ("a <mask> b <pad> c", "ein Hund läuft über die Straße")))


def write_fixture():
    import tokenizers
    import transformers
    model = train_spm()
    assert model == train_spm(), "SentencePiece training is not byte-stable"
    hf = hf_tokenizer(model)
    text = hf_tokenizer_json(hf)
    legacy = legacy_json(text)
    texts = fixed_prompts() + random_prompts(200, seed=1)
    ids, mask = hf_encode(hf, texts)
    lids, lmask = tokenizers_encode(legacy, texts)
    assert torch.equal(tokenizers_encode(text, texts)[0], ids)
    for layout, (ri, rm) in ((text, (ids, mask)), (legacy, (lids, lmask))):
        got = k2_tokenizer(layout)(texts)
        bad = [t for i, t in enumerate(texts) if not torch.equal(got["input_ids"][i], ri[i])]
        assert not bad and torch.equal(got["attention_mask"], rm), [repr(t) for t in bad[:5]]
    assert not torch.equal(lids, ids)                      # the layouts differ on some text
    V = len(hf)
    towers = []
    for n, (kw, out, prompts) in enumerate(TOWERS):
        cfg, wseed = tiny_config(V, **kw), 5 + n
        sd = synth_weights(cfg, out, wseed)
        tid, tmask = hf_encode(hf, list(prompts))
        hid, emb = transformers_outputs(sd, cfg, tid, tmask)
        ohid, oemb = forward(sd, cfg, tid, tmask)
        rel = max(((ohid - hid).norm() / hid.norm()).item(), ((oemb - emb).norm() / emb.norm()).item())
        assert rel <= 1e-5, f"oracle deviates from transformers by rel {rel}"
        towers.append(dict(cfg=cfg, out_features=out, weight_seed=wseed, prompts=list(prompts),
                           input_ids=tid.to(torch.int16), attention_mask=tmask.to(torch.int8), last_hidden_state=hid,
                           pooled=emb))
    flat, lengths = pack_ids(ids, mask)
    lflat, llengths = pack_ids(lids, lmask)
    torch.save(dict(transformers_version=transformers.__version__, tokenizers_version=tokenizers.__version__,
                    tokenizer_json=lzma.compress(text.encode("utf-8"), preset=9),
                    max_length=MAX_LENGTH, texts=texts, ids=flat, lengths=lengths, legacy_ids=lflat, legacy_lengths=llengths,
                    towers=towers), FIXTURE)
    print(f"wrote {FIXTURE} (transformers {transformers.__version__}, tokenizers {tokenizers.__version__}, vocabulary {V}, "
          f"{len(texts)} texts, {os.path.getsize(FIXTURE)} bytes)")


if __name__ == "__main__":
    import sys
    sys.path.insert(0, os.path.join(ROOT, "kandinsky-2_b200"))
    write_fixture()
