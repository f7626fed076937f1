"""The CLIP text side of the Kandinsky 2.2 prior pipeline: the tokenizer and the transformers `CLIPTextModelWithProjection`
(ViT-bigG/14 text in `kandinsky-2-2-prior/text_encoder`) that diffusers' `KandinskyV22PriorPipeline._encode_prompt` runs for
every prompt of every 2.2 method.

The tower is read from the checkpoint's `config.json` (hidden 1280, 32 layers, 20 heads of 64, MLP 5120, 77 positions,
vocabulary 49408, projection 1280, exact GELU expected for ViT-bigG/14); what is not implemented is refused with K2Error: any
`hidden_act` but "gelu", any head width but 64 (so the hidden size is a multiple of 8), more than 128 positions.  Compute, per
(row count, length) one LaunchPlan replayed as one CUDA graph:
    k2_clip_text_embed (token + position embedding, one fp16 rounding), then the pre-LayerNorm layers of model/encoder.py
    (q / k / v packed per head) with k2_attention_small as the attention (causal, no key mask: diffusers calls the encoder
    without attention_mask),
    final_layer_norm over every row (last_hidden_state), k2_clip_text_pool (the pooled row, chosen on the device from the ids
    by the config's eos_token_id rule, widened to fp32) and the bias-free text_projection in fp32 (ops.linear).
fp16 storage, fp32 accumulation, the prior's LayerNorm statistics and attention.

CLIPTokenizer restates transformers 5's CLIPTokenizer (the `tokenizers` backend) in the standard library only.

Parity: tests/test_cpu_clip_text.py pins the oracle (tests/clip_text_oracle.py) and the tokenizer to transformers
(tests/golden/clip_text_tiny.pt); tests/test_gpu_zz_clip_text.py runs the tower against the golden and, at full size on
synthetic weights, against the fp32 oracle.
"""
import os
import unicodedata

import torch

from .. import ops
from .._native import K2Error
from ..checkpoints import read_json
from ..launch_plan import LaunchPlan
from .encoder import Tower, clip_config, f16, f32, layer_shapes, pack_layers, record_layers

_REQUIRED = ("hidden_size", "intermediate_size", "num_hidden_layers", "num_attention_heads", "max_position_embeddings",
             "vocab_size", "projection_dim")
MAX_TOKENS = 128   # k2_attention_small's sequence limit


def text_tower_config(config):
    """The transformers CLIPTextConfig dict -> the geometry this module implements; K2Error for anything else.  A key that is
    absent takes transformers' default (hidden_act "quick_gelu", layer_norm_eps 1e-5, eos_token_id 49407).  "pool_eos" is the
    pooling rule: -1 for eos_token_id == 2 (the first argmax of the ids, pre-#24773 configs), else the eos id."""
    # heads of 64 make hidden_size a multiple of 8, which k2_clip_text_embed's 16-byte rows need
    c = clip_config(config, _REQUIRED, "text", 64)
    if not 0 < c["max_position_embeddings"] <= MAX_TOKENS:
        raise K2Error(f"CLIP text tower: max_position_embeddings {c['max_position_embeddings']} is not implemented "
                      f"(at most {MAX_TOKENS} tokens)")
    c["eos_token_id"] = int(config.get("eos_token_id", 49407))
    c["pool_eos"] = -1 if c["eos_token_id"] == 2 else c["eos_token_id"]
    return c


# ---------------------------------------------------------------------------------------------------------------------------
# tokenizer
# ---------------------------------------------------------------------------------------------------------------------------
# Unicode White_Space (what the tokenizers regex engine's \s matches; Python's str.isspace adds U+001C..U+001F)
_WS = frozenset("\t\n\x0b\x0c\r \x85\xa0\u1680\u2000\u2001\u2002\u2003\u2004\u2005\u2006\u2007\u2008\u2009"
                "\u200a\u2028\u2029\u202f\u205f\u3000")
_CONTRACTIONS = ("'s", "'t", "'re", "'ve", "'m", "'ll", "'d")
_CLIP_SPECIALS = ("<|startoftext|>", "<|endoftext|>")


def bytes_to_unicode():
    """GPT-2's reversible byte -> printable character map (the ByteLevel pre-tokenizer's alphabet)."""
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs = bs[:]
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return dict(zip(bs, map(chr, cs)))


def _is_letter(ch):
    return unicodedata.category(ch)[0] == "L"


def _is_number(ch):
    return unicodedata.category(ch)[0] == "N"


def _clip_split(text):
    """The CLIP pre-tokenizer's Split (matches kept, the rest removed):
    <|startoftext|>|<|endoftext|>|'s|'t|'re|'ve|'m|'ll|'d|[\\p{L}]+|[\\p{N}]|[^\\s\\p{L}\\p{N}]+  (leftmost-first)."""
    out, i, n = [], 0, len(text)
    while i < n:
        m = next((s for s in _CLIP_SPECIALS + _CONTRACTIONS if text.startswith(s, i)), None)
        if m is not None:
            out.append(m)
            i += len(m)
            continue
        ch = text[i]
        if _is_letter(ch):
            j = i + 1
            while j < n and _is_letter(text[j]):
                j += 1
        elif _is_number(ch):
            j = i + 1
        elif ch not in _WS:
            j = i + 1
            while j < n and not (text[j] in _WS or _is_letter(text[j]) or _is_number(text[j])):
                j += 1
        else:
            i += 1
            continue
        out.append(text[i:j])
        i = j
    return out


def _byte_level_split(piece):
    """The ByteLevel pre-tokenizer's own GPT-2 split of one CLIP piece (no whitespace inside):
    's|'t|'re|'ve|'m|'ll|'d| ?\\p{L}+| ?\\p{N}+| ?[^\\s\\p{L}\\p{N}]+.  It only changes the special-token pieces:
    "<|endoftext|>" -> "<|", "endoftext", "|>"."""
    out, i, n = [], 0, len(piece)
    while i < n:
        m = next((s for s in _CONTRACTIONS if piece.startswith(s, i)), None)
        if m is not None:
            out.append(m)
            i += len(m)
            continue
        cls = _is_letter if _is_letter(piece[i]) else _is_number if _is_number(piece[i]) else None
        j = i + 1
        if cls is not None:
            while j < n and cls(piece[j]):
                j += 1
        else:
            while j < n and not (piece[j] in _WS or _is_letter(piece[j]) or _is_number(piece[j])):
                j += 1
        out.append(piece[i:j])
        i = j
    return out


class CLIPTokenizer:
    """transformers 5's CLIPTokenizer (the `tokenizers` backend: tokenization_clip.py), restated with the standard library:
      1. added (special) tokens are matched in the raw text first, leftmost-longest, case-sensitively;
      2. the rest is normalised: NFC, runs of Unicode White_Space -> " ", then each character lowercased on its own (no
         final-sigma rule);
      3. split by the CLIP pattern, then by ByteLevel's GPT-2 pattern; each piece's UTF-8 bytes are mapped to
         bytes_to_unicode characters;
      4. BPE per piece with "</w>" on its last symbol, merging the lowest-ranked adjacent pair (leftmost first) until none
         is left; a symbol missing from the vocabulary becomes unk;
      5. [bos] + tokens[:max_length - 2] + [eos], right-padded with pad to max_length, and the attention mask.
    vocab: {token: id}; merges: [(a, b)] in rank order."""

    def __init__(self, vocab, merges, bos_token="<|startoftext|>", eos_token="<|endoftext|>", unk_token="<|endoftext|>",
                 pad_token="<|endoftext|>", model_max_length=77, added_tokens=()):
        self.vocab = dict(vocab)
        self.ranks = {tuple(m): r for r, m in enumerate(merges)}
        self.model_max_length = int(model_max_length)
        for name, tok in (("bos", bos_token), ("eos", eos_token), ("unk", unk_token), ("pad", pad_token)):
            if tok not in self.vocab:
                raise K2Error(f"CLIPTokenizer: the {name} token {tok!r} is not in the vocabulary")
        self.bos_token_id, self.eos_token_id = self.vocab[bos_token], self.vocab[eos_token]
        self.unk_token_id, self.pad_token_id = self.vocab[unk_token], self.vocab[pad_token]
        self.special = sorted({bos_token, eos_token, unk_token, pad_token, *added_tokens}, key=len, reverse=True)
        self.byte_map = bytes_to_unicode()
        self._cache = {}

    @classmethod
    def from_dir(cls, path):
        """A transformers tokenizer folder: vocab.json, merges.txt, and special_tokens_map.json / tokenizer_config.json when
        present (special tokens, the pad token, model_max_length; without one, model_max_length is 77)."""
        vocab = read_json(path, "vocab.json", "CLIPTokenizer")
        mf = os.path.join(path, "merges.txt")
        if not os.path.exists(mf):
            raise K2Error(f"CLIPTokenizer: {mf} not found")
        with open(mf, encoding="utf-8") as fh:
            lines = fh.read().split("\n")
        merges = [tuple(ln.split(" ")) for ln in lines if ln and not ln.startswith("#version")]
        kw = {}
        cfg = read_json(path, "tokenizer_config.json", "CLIPTokenizer", False) or {}
        cfg.update(read_json(path, "special_tokens_map.json", "CLIPTokenizer", False) or {})
        for k in ("bos_token", "eos_token", "unk_token", "pad_token"):
            v = cfg.get(k)
            if v is not None:
                kw[k] = v["content"] if isinstance(v, dict) else v
        if cfg.get("model_max_length") is not None and int(cfg["model_max_length"]) <= 1 << 20:
            kw["model_max_length"] = int(cfg["model_max_length"])
        added = [v["content"] for v in cfg.get("added_tokens_decoder", {}).values() if isinstance(v, dict) and "content" in v]
        return cls(vocab, merges, added_tokens=added, **kw)

    # -- steps ------------------------------------------------------------------------------------------------------------
    @staticmethod
    def normalize(text):
        text = unicodedata.normalize("NFC", text)
        out, prev_ws = [], False
        for ch in text:
            if ch in _WS:
                if not prev_ws:
                    out.append(" ")
                prev_ws = True
            else:
                out.append(ch.lower())
                prev_ws = False
        return "".join(out)

    def _bpe(self, word):
        """One pre-token (byte-level characters) -> vocabulary ids."""
        hit = self._cache.get(word)
        if hit is not None:
            return hit
        syms = list(word)
        syms[-1] += "</w>"
        while len(syms) > 1:
            best, at = None, -1
            for i in range(len(syms) - 1):
                r = self.ranks.get((syms[i], syms[i + 1]))
                if r is not None and (best is None or r < best):
                    best, at = r, i
            if best is None:
                break
            syms[at:at + 2] = [syms[at] + syms[at + 1]]
        ids = [self.vocab.get(s, self.unk_token_id) for s in syms]
        self._cache[word] = ids
        return ids

    def _split_special(self, text):
        """[(segment, is_special)] with the added tokens matched leftmost-longest in the raw text."""
        out, i, start, n = [], 0, 0, len(text)
        while i < n:
            m = next((s for s in self.special if text.startswith(s, i)), None)
            if m is None:
                i += 1
                continue
            if i > start:
                out.append((text[start:i], False))
            out.append((m, True))
            i += len(m)
            start = i
        if start < n:
            out.append((text[start:], False))
        return out

    def tokenize_ids(self, text):
        """The token ids of one text, without bos / eos."""
        ids = []
        for seg, special in self._split_special(text):
            if special:
                ids.append(self.vocab[seg])
                continue
            for piece in _clip_split(self.normalize(seg)):
                for word in _byte_level_split(piece):
                    ids += self._bpe("".join(self.byte_map[b] for b in word.encode("utf-8")))
        return ids

    def __call__(self, texts, max_length=None):
        """texts: str or list[str] -> dict(input_ids int64 [n, L], attention_mask int64 [n, L]) on the CPU, L = max_length
        (default model_max_length): padding="max_length", truncation=True."""
        if isinstance(texts, str):
            texts = [texts]
        L = self.model_max_length if max_length is None else int(max_length)
        if L < 2:
            raise K2Error(f"CLIPTokenizer: max_length {L} leaves no room for bos and eos")
        ids = torch.full((len(texts), L), self.pad_token_id, dtype=torch.int64)
        mask = torch.zeros(len(texts), L, dtype=torch.int64)
        for r, t in enumerate(texts):
            row = [self.bos_token_id] + self.tokenize_ids(t)[:L - 2] + [self.eos_token_id]
            ids[r, :len(row)] = torch.tensor(row)
            mask[r, :len(row)] = 1
        return {"input_ids": ids, "attention_mask": mask}


# ---------------------------------------------------------------------------------------------------------------------------
# tower
# ---------------------------------------------------------------------------------------------------------------------------
class CLIPTextTower(Tower):
    """CLIPTextModelWithProjection on this package's kernels.  sd: state dict in this module's names
    (checkpoints.transformers_clip_text_to_k2); config: the transformers config.json dict; tokenizer: a CLIPTokenizer (needed
    by __call__ only).  `tokens` is the sequence length __call__ produces: the tokenizer's model_max_length, or
    max_position_embeddings without a tokenizer."""

    what = "CLIP text tower"
    act = "gelu"   # the layers' MLP activation (encoder.ACTIVATIONS)

    def __init__(self, sd, config, device="cuda", tokenizer=None):
        c = text_tower_config(config)
        self.cfg, self.device, self.tokenizer = c, torch.device(device), tokenizer
        self.tokens = tokenizer.model_max_length if tokenizer is not None else c["max_position_embeddings"]
        if not 2 <= self.tokens <= c["max_position_embeddings"]:
            raise K2Error(f"CLIP text tower: the tokenizer's model_max_length {self.tokens} does not fit the "
                          f"{c['max_position_embeddings']} positions")
        if tokenizer is not None and max(tokenizer.vocab.values()) >= c["vocab_size"]:
            raise K2Error(f"CLIP text tower: the tokenizer's ids reach {max(tokenizer.vocab.values())}, beyond the "
                          f"vocabulary of {c['vocab_size']}")
        self._take(sd, self._want())

    def _want(self):
        """{name: shape} of the state dict this tower takes."""
        c = self.cfg
        H = c["hidden_size"]
        want = {"token_embedding": (c["vocab_size"], H), "position_embedding": (c["max_position_embeddings"], H),
                "final_ln.weight": (H,), "final_ln.bias": (H,), "proj.weight": (c["projection_dim"], H)}
        want.update({f"layers.{i}.{k}": s for i in range(c["num_hidden_layers"])
                     for k, s in layer_shapes(H, c["intermediate_size"]).items()})
        return want

    @classmethod
    def from_transformers(cls, state_dict, config, device="cuda", tokenizer=None):
        """From a transformers CLIPTextModelWithProjection state dict and its config.json dict; packs the weights."""
        from ..checkpoints import transformers_clip_text_to_k2
        text_tower_config(config)
        return cls(transformers_clip_text_to_k2(state_dict), config, device, tokenizer).finalize()

    def _pack(self):
        """fp16 GEMM weights [N, K], fp32 biases / LayerNorm parameters / projection, the fp16 token and position tables."""
        c, dev, sd = self.cfg, self.device, self.sd
        return {"tok": f16(sd["token_embedding"], dev), "pos": f16(sd["position_embedding"], dev),
                "final_ln": (f32(sd["final_ln.weight"], dev), f32(sd["final_ln.bias"], dev)),
                "proj": f32(sd["proj.weight"], dev),
                "layers": pack_layers(lambda i, name: sd[f"layers.{i}.{name}"], c["num_hidden_layers"], dev)}

    def _plan(self, n, T=None):
        return super()._plan(n, self.cfg["max_position_embeddings"] if T is None else T)

    def _new_plan(self, n, T):
        return _TextPlan(self, n, T)

    @torch.no_grad()
    def forward(self, input_ids, use_graph=True):
        """input_ids integer [n, T] (T <= max_position_embeddings) -> (last_hidden_state fp16 [n, T, hidden], text_embeds fp32
        [n, projection_dim]), on the device.  One CUDA graph replay of the (n, T) launch plan (use_graph=False: the same
        launches one by one).  Ids outside [0, vocab_size) are refused before anything is copied."""
        self._check_ids(input_ids, self.cfg["max_position_embeddings"])
        plan = self._plan(*input_ids.shape)
        plan.ids.copy_(input_ids)
        plan.run(use_graph)
        return plan.hidden.clone(), plan.out.clone()

    def __call__(self, prompts):
        """The embedders' clip_text protocol: list[str] -> (text_embeds fp32 [n, projection_dim], last_hidden_state fp16
        [n, tokens, hidden], mask bool [n, tokens]), on the device.  Each distinct prompt is tokenized and encoded once and its
        rows are gathered back (diffusers encodes a prompt once and repeats its rows)."""
        if self.tokenizer is None:
            raise K2Error("CLIP text tower: calling it with prompts needs tokenizer=")
        if isinstance(prompts, str):
            prompts = [prompts]

        def encode(distinct):
            tok = self.tokenizer(distinct, max_length=self.tokens)
            hid, emb = self.forward(tok["input_ids"])
            return emb, hid, tok["attention_mask"].to(self.device).bool()
        return self._encode_distinct(prompts, encode)


class _TextPlan(LaunchPlan):
    """The tower on n sequences of T tokens as one static launch list over fixed buffers (replayed as one CUDA graph): ids ->
    embed -> L layers -> final LayerNorm (self.hidden, transformers' last_hidden_state) -> pool (fp32) -> projection (self.out).
    self.index holds the pooled positions of the last run."""

    def __init__(self, tower, n, T):
        super().__init__(tower.device, n)
        self.t, self.n, self.T = tower, n, T
        self.ids = torch.zeros(n, T, device=self.dev, dtype=torch.int32)
        self.index = torch.zeros(n, device=self.dev, dtype=torch.int32)
        self.out = torch.zeros(n, tower.cfg["projection_dim"], device=self.dev, dtype=torch.float32)
        self._build()

    def _build(self):
        c, pk, n, T, S = self.t.cfg, self.t._packed, self.n, self.T, self._add
        H, heads, eps = c["hidden_size"], c["num_attention_heads"], c["layer_norm_eps"]
        x = self._new(n, T, H)
        S(lambda: ops.clip_text_embed(self.ids, pk["tok"], pk["pos"], out=x), "embed")
        scale = c["head_dim"] ** -0.5
        h = record_layers(self, x, pk["layers"],
                          lambda qkv, out: ops.attention_small(qkv, heads, keep_mask=None, causal=True, scale=scale, out=out),
                          4 * n * heads * T * T * c["head_dim"], eps, act=self.t.act)
        self.hidden = self._new(n, T, H)
        S(lambda: ops.layernorm_f16(h, *pk["final_ln"], eps=eps, out=self.hidden), "layernorm")
        pooled = torch.empty(n, H, device=self.dev, dtype=torch.float32)
        S(lambda: ops.clip_text_pool(self.ids, self.hidden, c["pool_eos"], out=pooled, index_out=self.index), "pool")
        S(lambda: ops.linear(pooled, pk["proj"], out=self.out), "linear", 2 * n * H * c["projection_dim"])
