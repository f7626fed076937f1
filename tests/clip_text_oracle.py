"""TEST INFRASTRUCTURE (oracle): the CLIP text side of the Kandinsky 2.2 prior pipeline -- transformers'
`CLIPTextModelWithProjection` restated from the math in torch, a synthetic CLIP BPE tokenizer, and the writer of the golden
fixture tests/golden/clip_text_tiny.pt:

    python -m tests.clip_text_oracle

  clip_text_spec       <- the transformers state dict of a config (key names as transformers writes them)
  synth_weights        <- oracle/synth.py synthetic weights for it
  forward              <- CLIPTextModelWithProjection.forward from transformers names: token + position embedding, pre-LN
                          encoder layers (eager causal attention, exact GELU), final_layer_norm over every row, the pooled row
                          (eos_token_id == 2: the first argmax of the ids; else the first eos), text_projection.
                          dtype=torch.float16 rounds where transformers' fp16 model does (fp16 inputs to every op, softmax in
                          fp32 then rounded).
  forward_k2           <- the same network from kandinsky2's names (checkpoints.transformers_clip_text_to_k2), fp32
  train_merges         <- a tiny deterministic BPE trainer over CORPUS: the synthetic tokenizer's merges
  synthetic_vocab      <- its vocabulary: the 256 byte symbols, the same with "</w>", the merges, then the two specials (eos
                          last, so it has the highest id as in the real vocabulary; the argmax pooling rule depends on it)
  fixed_prompts / random_prompts <- the texts whose tokenization the fixture pins

The fixture holds the merges (the vocabulary follows from them), transformers' input_ids for every text (each row up to its
eos; the rest is padding, its length is the attention mask), and for two tiny towers (hidden 128, 2 heads of 64, MLP 256,
projection 32, 77 positions; one with eos_token_id 2, one with the tokenizer's eos id) their weight seeds, ids and
transformers' fp32 last_hidden_state / text_embeds.  Before writing, the generator asserts that the oracle and
kandinsky2's CLIPTokenizer reproduce transformers."""
import os
import random

import torch
import torch.nn.functional as F

from oracle import synth

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
FIXTURE = os.path.join(ROOT, "tests", "golden", "clip_text_tiny.pt")
MAX_LENGTH = 77
N_MERGES = 300

# ViT-bigG/14 text as kandinsky-2-2-prior/text_encoder is expected to configure it (not checked against the real file)
CONFIG_BIGG = dict(vocab_size=49408, hidden_size=1280, intermediate_size=5120, num_hidden_layers=32, num_attention_heads=20,
                   max_position_embeddings=77, projection_dim=1280, hidden_act="gelu", layer_norm_eps=1e-5, bos_token_id=0,
                   eos_token_id=2, pad_token_id=1)

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
    "🐱🐶 emoji party 🎉🎉 with 123 balloons and 4567 stars!!!",
    "numbers 0 1 2 3 4 5 6 7 8 9 10 100 1000 2023 3.14159",
    "cyberpunk city at night, neon lights, rain, reflections, cinematic, 8k, unreal engine",
    "watercolor painting of a fox in the forest, soft colors, misty morning",
)


# ---------------------------------------------------------------------------------------------------------------------------
# tokenizer
# ---------------------------------------------------------------------------------------------------------------------------
def _words(text):
    """The byte-level pre-tokens of a text, as kandinsky2's CLIPTokenizer forms them (specials aside)."""
    from kandinsky2.model.clip_text import CLIPTokenizer, _byte_level_split, _clip_split, bytes_to_unicode
    bmap = bytes_to_unicode()
    return ["".join(bmap[b] for b in w.encode("utf-8")) for p in _clip_split(CLIPTokenizer.normalize(text))
            for w in _byte_level_split(p)]


def train_merges(n=N_MERGES):
    """Greedy BPE over CORPUS: the most frequent adjacent pair (ties: the smallest pair) is merged, a pair whose result is
    already a token is skipped, until n merges or no pair is left."""
    from kandinsky2.model.clip_text import bytes_to_unicode
    freq = {}
    for line in CORPUS:
        for w in _words(line):
            syms = tuple(w[:-1]) + (w[-1] + "</w>",)
            freq[syms] = freq.get(syms, 0) + 1
    have = set(bytes_to_unicode().values()) | {s + "</w>" for s in bytes_to_unicode().values()}
    merges = []
    while len(merges) < n:
        counts = {}
        for syms, f in freq.items():
            for a, b in zip(syms, syms[1:]):
                if a + b not in have:
                    counts[(a, b)] = counts.get((a, b), 0) + f
        if not counts:
            break
        pair = min(counts, key=lambda p: (-counts[p], p))
        merges.append(pair)
        have.add(pair[0] + pair[1])
        new = {}
        for syms, f in freq.items():
            out, i = [], 0
            while i < len(syms):
                if i + 1 < len(syms) and (syms[i], syms[i + 1]) == pair:
                    out.append(syms[i] + syms[i + 1])
                    i += 2
                else:
                    out.append(syms[i])
                    i += 1
            new[tuple(out)] = new.get(tuple(out), 0) + f
        freq = new
    return merges


def synthetic_vocab(merges):
    from kandinsky2.model.clip_text import bytes_to_unicode
    syms = list(bytes_to_unicode().values())
    tokens = syms + [s + "</w>" for s in syms] + [a + b for a, b in merges] + ["<|startoftext|>", "<|endoftext|>"]
    return {t: i for i, t in enumerate(tokens)}


def fixed_prompts():
    return [
        "", " ", "\t\n  \t", "a\t\tb\n\nc   d", "\x1c", "a\x1cb", "\u0085", "a\u0085b", "\u200b", "a\u200bb", "\u00a0x\u3000y",
        "A RED CAT", "ΟΔΟΣ", "İstanbul İ", "e\u0301 cafe\u0301 CAFE\u0301", "一只猫坐在桌子上", "🐱🐶🎉 emoji 👩\u200d👩\u200d👧",
        "1234567890 3.14159 2023", "it's we'll they're I've I'm you'd can't IT'S", "wow!!! ... ?!?! --- (()) [[]] {{}}",
        "a <|endoftext|> b", "<|ENDOFTEXT|> <|startoftext|>x", "<|endoftext|>", "x " * 75, "x " * 80 + "tail",
        "A capybara, 4k photo",
        "lowres, text, error, cropped, worst quality, low quality, jpeg artifacts, ugly, duplicate, morbid, mutilated, out of "
        "frame, extra fingers, mutated hands, poorly drawn hands, poorly drawn face, mutation, deformed, blurry, dehydrated, "
        "bad anatomy, bad proportions, extra limbs, cloned face, disfigured, gross proportions, malformed limbs, missing arms, "
        "missing legs, extra arms, extra legs, fused fingers, too many fingers, long neck, username, watermark, signature",
        "red cat", "ﬁne ｆｕｌｌｗｉｄｔｈ Ⅻ ½ ²",
    ]


_PIECES = (list("abcdefghijklmnopqrstuvwxyzABCDEFGHIJKLMNOPQRSTUVWXYZ0123456789") + list(" \t\n  ") +
           list(".,!?;:'\"-()[]{}<>|/\\@#$%^&*_+=~`") + list("äöüßéèêàçñåøÄÖÜÉ") + list("αβγδεζηθΣσςΩΟΔ") +
           list("абвгдеёжзийклмнопрстуфхцчшщъыьэюяЖЯ") + list("猫狗日本語中文漢字かなカナ한국어") + ["🐱", "🎉", "👩\u200d👩\u200d👧", "🇯🇵"] +
           ["\x1c", "\x1f", "\u0085", "\u200b", "\u00a0", "\u3000", "\u0301", "\u0308", "İ", "ﬁ", "Ⅻ", "½"] +
           ["'s", "'t", "'re", "'ll", "<|endoftext|>", "<|startoftext|>", "cat", "the ", "photo", "capybara"])


def random_prompts(n, seed):
    rng = random.Random(seed)
    return ["".join(rng.choice(_PIECES) for _ in range(rng.randint(0, 40))) for _ in range(n)]


def hf_tokenizer(merges):
    """transformers' own CLIPTokenizer over the synthetic vocabulary, model_max_length MAX_LENGTH."""
    from transformers import CLIPTokenizer
    return CLIPTokenizer(vocab=synthetic_vocab(merges), merges=[tuple(m) for m in merges], model_max_length=MAX_LENGTH)


def k2_tokenizer(merges):
    from kandinsky2.model.clip_text import CLIPTokenizer
    return CLIPTokenizer(synthetic_vocab(merges), merges, model_max_length=MAX_LENGTH)


def hf_encode(tok, texts):
    e = tok(texts, padding="max_length", max_length=MAX_LENGTH, truncation=True, return_tensors="pt")
    return e["input_ids"].long(), e["attention_mask"].long()


def pack_ids(ids, mask):
    """[n, L] ids and mask -> (concatenated rows up to their mask's length, int16; lengths, int16)."""
    lengths = mask.sum(1)
    assert torch.equal(mask, (torch.arange(ids.shape[1])[None] < lengths[:, None]).long())
    return torch.cat([ids[i, :lengths[i]] for i in range(ids.shape[0])]).to(torch.int16), lengths.to(torch.int16)


def unpack_ids(flat, lengths, pad_id, L=MAX_LENGTH):
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


# ---------------------------------------------------------------------------------------------------------------------------
# tower
# ---------------------------------------------------------------------------------------------------------------------------
def tiny_config(vocab_size, eos_token_id):
    return dict(vocab_size=vocab_size, hidden_size=128, intermediate_size=256, num_hidden_layers=2, num_attention_heads=2,
                max_position_embeddings=MAX_LENGTH, projection_dim=32, hidden_act="gelu", layer_norm_eps=1e-5,
                bos_token_id=vocab_size - 2, eos_token_id=eos_token_id, pad_token_id=vocab_size - 1)


def clip_text_spec(cfg):
    H, I = cfg["hidden_size"], cfg["intermediate_size"]
    p = "text_model."
    spec = [(p + "embeddings.token_embedding.weight", (cfg["vocab_size"], H)),
            (p + "embeddings.position_embedding.weight", (cfg["max_position_embeddings"], H))]
    for i in range(cfg["num_hidden_layers"]):
        lp = f"{p}encoder.layers.{i}."
        for n in ("q_proj", "k_proj", "v_proj", "out_proj"):
            spec += [(f"{lp}self_attn.{n}.weight", (H, H)), (f"{lp}self_attn.{n}.bias", (H,))]
        spec += [(lp + "layer_norm1.weight", (H,)), (lp + "layer_norm1.bias", (H,)), (lp + "mlp.fc1.weight", (I, H)),
                 (lp + "mlp.fc1.bias", (I,)), (lp + "mlp.fc2.weight", (H, I)), (lp + "mlp.fc2.bias", (H,)),
                 (lp + "layer_norm2.weight", (H,)), (lp + "layer_norm2.bias", (H,))]
    return spec + [(p + "final_layer_norm.weight", (H,)), (p + "final_layer_norm.bias", (H,)),
                   ("text_projection.weight", (cfg["projection_dim"], H))]


def synth_weights(cfg, seed):
    return synth.synth_state_dict(clip_text_spec(cfg), seed=seed)


def _attention(q, k, v, heads, dtype):
    B, T, H = q.shape
    d = H // heads
    q, k, v = (t.view(B, T, heads, d).transpose(1, 2) for t in (q, k, v))
    w = torch.matmul(q, k.transpose(-1, -2)) * d ** -0.5
    causal = torch.ones(T, T, dtype=torch.bool, device=q.device).triu(1)
    w = torch.softmax(w.float().masked_fill(causal, float("-inf")), dim=-1).to(dtype)
    return torch.matmul(w, v).transpose(1, 2).reshape(B, T, H)


def pooled_index(ids, eos_token_id):
    """transformers' pooled position per row: eos_token_id == 2 -> the first argmax of the ids; else the first position equal
    to eos_token_id (0 if none)."""
    if eos_token_id == 2:
        return ids.to(torch.int).argmax(-1)
    return (ids.to(torch.int) == eos_token_id).int().argmax(-1)


def _tower(emb, ids, layers, final, proj, cfg, dtype):
    """emb [B, T, H] (token + position embedding); layers: per layer (ln1, (wq, bq), (wk, bk), (wv, bv), (wo, bo), ln2, fc1,
    fc2) with ln = (weight, bias) -> (last_hidden_state, text_embeds), fp32."""
    H, eps, heads = cfg["hidden_size"], cfg["layer_norm_eps"], cfg["num_attention_heads"]
    h = emb
    for ln1, q, k, v, o, ln2, fc1, fc2 in layers:
        y = F.layer_norm(h, (H,), *ln1, eps=eps)
        a = _attention(F.linear(y, *q), F.linear(y, *k), F.linear(y, *v), heads, dtype)
        h = h + F.linear(a, *o)
        y = F.layer_norm(h, (H,), *ln2, eps=eps)
        h = h + F.linear(F.gelu(F.linear(y, *fc1)), *fc2)
    h = F.layer_norm(h, (H,), *final, eps=eps)
    idx = pooled_index(ids, cfg.get("eos_token_id", 49407)).to(h.device)
    pooled = h[torch.arange(h.shape[0], device=h.device), idx]
    return h.float(), F.linear(pooled, proj).float()


def forward(sd, cfg, ids, dtype=torch.float32):
    """transformers names, ids [B, T] -> (last_hidden_state [B, T, H], text_embeds [B, projection_dim]), both fp32."""
    sd = {k: v.to(dtype) for k, v in sd.items()}
    p = "text_model."
    g = lambda n: (sd[n + ".weight"], sd[n + ".bias"])  # noqa: E731
    ids = ids.to(sd[p + "embeddings.token_embedding.weight"].device).long()
    emb = sd[p + "embeddings.token_embedding.weight"][ids] + sd[p + "embeddings.position_embedding.weight"][:ids.shape[1]][None]
    layers = []
    for i in range(cfg["num_hidden_layers"]):
        lp = f"{p}encoder.layers.{i}."
        layers.append((g(lp + "layer_norm1"), g(lp + "self_attn.q_proj"), g(lp + "self_attn.k_proj"), g(lp + "self_attn.v_proj"),
                       g(lp + "self_attn.out_proj"), g(lp + "layer_norm2"), g(lp + "mlp.fc1"), g(lp + "mlp.fc2")))
    return _tower(emb, ids, layers, g(p + "final_layer_norm"), sd["text_projection.weight"], cfg, dtype)


def forward_k2(sd, cfg, ids):
    """kandinsky2 names (attn.qkv packed per head [q_h | k_h | v_h]) -> the same outputs as forward, fp32."""
    H, heads = cfg["hidden_size"], cfg["num_attention_heads"]
    d = H // heads
    g = lambda n: (sd[n + ".weight"].float(), sd[n + ".bias"].float())  # noqa: E731
    ids = ids.long()
    emb = sd["token_embedding"].float()[ids] + sd["position_embedding"].float()[:ids.shape[1]][None]
    layers = []
    for i in range(cfg["num_hidden_layers"]):
        w, b = g(f"layers.{i}.attn.qkv")
        wq, wk, wv = (w.view(heads, 3, d, H)[:, j].reshape(H, H) for j in range(3))
        bq, bk, bv = (b.view(heads, 3, d)[:, j].reshape(H) for j in range(3))
        p = f"layers.{i}."
        layers.append((g(p + "ln_1"), (wq, bq), (wk, bk), (wv, bv), g(p + "attn.proj"), g(p + "ln_2"), g(p + "mlp.fc1"),
                       g(p + "mlp.fc2")))
    return _tower(emb, ids, layers, g("final_ln"), sd["proj.weight"].float(), cfg, torch.float32)


def transformers_outputs(sd, cfg, ids):
    """transformers' own CLIPTextModelWithProjection (eager attention, fp32) on sd, called without an attention mask (as
    diffusers' _encode_prompt calls it)."""
    from transformers import CLIPTextConfig, CLIPTextModelWithProjection
    model = CLIPTextModelWithProjection(CLIPTextConfig(**cfg, attn_implementation="eager")).eval()
    model.load_state_dict(sd, strict=True)
    with torch.no_grad():
        o = model(input_ids=ids)
    return o.last_hidden_state.float(), o.text_embeds.float()


TOWER_PROMPTS = (("A capybara, 4k photo", "red cat"), ("a <|endoftext|> b",))


def write_fixture():
    import tokenizers
    import transformers
    merges = train_merges()
    hf = hf_tokenizer(merges)
    mine = k2_tokenizer(merges)
    texts = fixed_prompts() + random_prompts(200, seed=1)
    ids, mask = hf_encode(hf, texts)
    for i, t in enumerate(texts):
        got = mine([t])
        assert torch.equal(got["input_ids"], ids[i:i + 1]) and torch.equal(got["attention_mask"], mask[i:i + 1]), repr(t)
    flat, lengths = pack_ids(ids, mask)
    V = len(synthetic_vocab(merges))
    towers = []
    for n, (eos, prompts) in enumerate(zip((2, hf.eos_token_id), TOWER_PROMPTS)):
        cfg, wseed = tiny_config(V, eos), 5 + n
        sd = synth_weights(cfg, wseed)
        tid, _ = hf_encode(hf, list(prompts))
        hid, emb = transformers_outputs(sd, cfg, tid)
        ohid, oemb = forward(sd, cfg, tid)
        rel = max(((ohid - hid).norm() / hid.norm()).item(), ((oemb - emb).norm() / emb.norm()).item())
        assert rel <= 1e-5, f"oracle deviates from transformers by rel {rel}"
        towers.append(dict(cfg=cfg, weight_seed=wseed, prompts=list(prompts), input_ids=tid.to(torch.int16),
                           last_hidden_state=hid, text_embeds=emb))
    torch.save(dict(transformers_version=transformers.__version__, tokenizers_version=tokenizers.__version__,
                    merges=[list(m) for m in merges], max_length=MAX_LENGTH, texts=texts, ids=flat, lengths=lengths,
                    towers=towers), FIXTURE)
    print(f"wrote {FIXTURE} (transformers {transformers.__version__}, tokenizers {tokenizers.__version__}, {len(merges)} "
          f"merges, vocabulary {V}, {len(texts)} texts, {os.path.getsize(FIXTURE)} bytes)")


if __name__ == "__main__":
    import sys
    sys.path.insert(0, os.path.join(ROOT, "kandinsky-2_b200"))
    write_fixture()
