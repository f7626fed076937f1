"""The Kandinsky 2.1 text encoder: the reference's `TextEncoder(model_name="multiclip")` (model/text_encoders.py:108-167), a
multilingual CLIP text tower -- transformers' `XLMRobertaModel` (XLM-RoBERTa-large in `2_1/text_encoder/`) plus the
`LinearTransformation` 1024 -> 768 -- and its SentencePiece tokenizer, which `encode_text` (kandinsky2_1_model.py:116-131)
runs on [prompt x B | "" x B] for every 2.1 method:
    full_emb   [2B, 77, 1024]  last_hidden_state, every row including the padded ones (the UNet's encoder K / V);
    pooled_emb [2B, 768]       LinearTransformation(sum_t mask h / sum_t mask) (the time-embedding projection's input).

The tower is read from the folder's `config.json`; what is not implemented is refused with K2Error: any `hidden_act` but
"gelu", any head width but 64, non-absolute position embeddings, `type_vocab_size` other than 1, more than 128 tokens per
row.  XLM-R is a post-LayerNorm encoder.  Compute, per row count, one LaunchPlan replayed as one CUDA graph:
    k2_xlmr_embed (word + token-type row 0 + position, the position computed on the device from the ids, then LayerNorm,
    one fp16 rounding), the post-LN layers of model/encoder.py (q / k / v packed per head) with k2_attention_small as the
    attention (not causal, the attention mask as the key keep-mask), k2_masked_mean_f16 (fp32) and the Linear in fp32
    (ops.linear).
fp16 storage, fp32 accumulation, float64 LayerNorm statistics.  A row whose attention mask keeps no token comes out NaN
(transformers' finfo.min mask gives a uniform softmax there); the tokenizer always keeps <s>.

XLMRobertaTokenizer restates transformers 5's tokenizers-backed XLM-R tokenizer from `tokenizer.json` with the standard
library only.  Unpinned: the released `config.json` values and `tokenizer.json` layout (read from the files, refused where
not implemented), and the grapheme segmentation (_graphemes, an approximation of UAX #29; see there).

Parity: tests/test_cpu_text_encoder.py pins the tokenizer and the oracle (tests/xlmr_oracle.py) to transformers / tokenizers
(tests/golden/xlmr_tiny.pt); tests/test_gpu_zz_text_encoder.py runs the tower against the golden and, at full size on
synthetic weights, against the fp32 oracle.
"""
import base64
import re
import struct
import unicodedata

import torch

from .. import ops
from .._native import K2Error
from ..checkpoints import load_weights, read_json
from ..launch_plan import LaunchPlan
from .encoder import Tower, f16, f32, layer_shapes, pack_layers, record_layers

_REQUIRED = ("hidden_size", "intermediate_size", "num_hidden_layers", "num_attention_heads", "max_position_embeddings",
             "vocab_size")
MAX_TOKENS = 128   # k2_attention_small's sequence limit
HEAD_DIM = 64


def xlmr_config(config):
    """The transformers XLMRobertaConfig dict -> the geometry this module implements; K2Error for anything else.  A key that is
    absent takes transformers' default (hidden_act "gelu", layer_norm_eps 1e-12, pad_token_id 1, type_vocab_size 2,
    position_embedding_type "absolute")."""
    missing = [k for k in _REQUIRED if k not in config]
    if missing:
        raise K2Error(f"XLM-R config: missing {missing}")
    c = {k: int(config[k]) for k in _REQUIRED}
    c["hidden_act"] = config.get("hidden_act", "gelu")
    c["layer_norm_eps"] = float(config.get("layer_norm_eps", 1e-12))
    c["pad_token_id"] = int(config.get("pad_token_id", 1))
    c["type_vocab_size"] = int(config.get("type_vocab_size", 2))
    c["position_embedding_type"] = config.get("position_embedding_type", "absolute")
    if c["hidden_act"] != "gelu":
        raise K2Error(f"XLM-R text encoder: hidden_act {c['hidden_act']!r} is not implemented (only the exact 'gelu')")
    H, heads = c["hidden_size"], c["num_attention_heads"]
    if H % heads or H // heads != HEAD_DIM:
        raise K2Error(f"XLM-R text encoder: head width {H / heads:g} is not implemented (only {HEAD_DIM})")
    if c["position_embedding_type"] != "absolute":
        raise K2Error(f"XLM-R text encoder: position_embedding_type {c['position_embedding_type']!r} is not implemented "
                      "(only 'absolute')")
    if c["type_vocab_size"] != 1:
        raise K2Error(f"XLM-R text encoder: type_vocab_size {c['type_vocab_size']} is not implemented (only 1)")
    if not 0 <= c["pad_token_id"] < c["vocab_size"]:
        raise K2Error(f"XLM-R text encoder: pad_token_id {c['pad_token_id']} is outside the vocabulary")
    # positions pad_id + 1 .. pad_id + T must exist
    c["max_tokens"] = min(MAX_TOKENS, c["max_position_embeddings"] - c["pad_token_id"] - 1)
    if c["max_tokens"] < 1:
        raise K2Error(f"XLM-R text encoder: max_position_embeddings {c['max_position_embeddings']} leaves no position after "
                      f"pad_token_id {c['pad_token_id']}")
    c["head_dim"] = HEAD_DIM
    return c


# ---------------------------------------------------------------------------------------------------------------------------
# tokenizer
# ---------------------------------------------------------------------------------------------------------------------------
# Unicode White_Space (Rust's char::is_whitespace, which WhitespaceSplit and the added tokens' lstrip / rstrip use)
_WS = frozenset("\t\n\x0b\x0c\r \x85\xa0\u1680\u2000\u2001\u2002\u2003\u2004\u2005\u2006\u2007\u2008\u2009"
                "\u200a\u2028\u2029\u202f\u205f\u3000")

# Grapheme_Cluster_Break classes that the general category does not give
_PREPEND = frozenset([*range(0x600, 0x606), 0x6DD, 0x70F, 0x890, 0x891, 0x8E2, 0xD4E, 0x110BD, 0x110CD, 0x111C2, 0x111C3,
                      0x1193F, 0x11941, 0x11A3A, *range(0x11A84, 0x11A8A), 0x11D46, 0x11F02])
_EXTEND_EXTRA = frozenset([0x200C, 0x9BE, 0x9D7, 0xB3E, 0xB57, 0xBBE, 0xBD7, 0xCC2, 0xCD5, 0xCD6, 0xD3E, 0xD57, 0xDCF,
                           0xDDF, 0x1B35, 0x302E, 0x302F, 0xFF9E, 0xFF9F, 0x1133E, 0x11357, 0x114B0, 0x114BD, 0x115AF,
                           0x11930, 0x1D165, *range(0x1D16E, 0x1D173), *range(0x1F3FB, 0x1F400), *range(0xE0020, 0xE0080)])
_SPACING_EXTRA = frozenset([0xE33, 0xEB3])
_EXT_PICT = ((0xA9, 0xA9), (0xAE, 0xAE), (0x203C, 0x203C), (0x2049, 0x2049), (0x2122, 0x2122), (0x2139, 0x2139),
             (0x2194, 0x2199), (0x21A9, 0x21AA), (0x231A, 0x231B), (0x2328, 0x2328), (0x2388, 0x2388), (0x23CF, 0x23CF),
             (0x23E9, 0x23F3), (0x23F8, 0x23FA), (0x24C2, 0x24C2), (0x25AA, 0x25AB), (0x25B6, 0x25B6), (0x25C0, 0x25C0),
             (0x25FB, 0x25FE), (0x2600, 0x27BF), (0x2934, 0x2935), (0x2B05, 0x2B07), (0x2B1B, 0x2B1C), (0x2B50, 0x2B50),
             (0x2B55, 0x2B55), (0x3030, 0x3030), (0x303D, 0x303D), (0x3297, 0x3297), (0x3299, 0x3299),
             (0x1F000, 0x1F0FF), (0x1F10D, 0x1F10F), (0x1F12F, 0x1F12F), (0x1F16C, 0x1F171), (0x1F17E, 0x1F17F),
             (0x1F18E, 0x1F18E), (0x1F191, 0x1F19A), (0x1F1AD, 0x1F1E5), (0x1F201, 0x1F20F), (0x1F21A, 0x1F21A),
             (0x1F22F, 0x1F22F), (0x1F232, 0x1F23A), (0x1F23C, 0x1F23F), (0x1F249, 0x1F3FA), (0x1F400, 0x1F53D),
             (0x1F546, 0x1F64F), (0x1F680, 0x1F6FF), (0x1F774, 0x1F77F), (0x1F7D5, 0x1F7FF), (0x1F80C, 0x1F80F),
             (0x1F848, 0x1F84F), (0x1F85A, 0x1F85F), (0x1F888, 0x1F88F), (0x1F8AE, 0x1F8FF), (0x1F90C, 0x1F93A),
             (0x1F93C, 0x1F945), (0x1F947, 0x1FAFF), (0x1FC00, 0x1FFFD))


def _gcb(ch):
    """Grapheme_Cluster_Break of one character, from the general category plus the tables above."""
    o = ord(ch)
    if ch == "\r":
        return "CR"
    if ch == "\n":
        return "LF"
    if o == 0x200D:
        return "ZWJ"
    if o in _PREPEND:
        return "Prepend"
    if o in _EXTEND_EXTRA:
        return "Extend"
    if 0x1F1E6 <= o <= 0x1F1FF:
        return "RI"
    if 0x1100 <= o <= 0x115F or 0xA960 <= o <= 0xA97C:
        return "L"
    if 0x1160 <= o <= 0x11A7 or 0xD7B0 <= o <= 0xD7C6:
        return "V"
    if 0x11A8 <= o <= 0x11FF or 0xD7CB <= o <= 0xD7FB:
        return "T"
    if 0xAC00 <= o <= 0xD7A3:
        return "LV" if (o - 0xAC00) % 28 == 0 else "LVT"
    cat = unicodedata.category(ch)
    if cat in ("Mn", "Me"):
        return "Extend"
    if cat == "Mc" or o in _SPACING_EXTRA:
        return "SpacingMark"
    if cat in ("Cc", "Zl", "Zp", "Cf", "Cs"):
        return "Control"
    if any(a <= o <= b for a, b in _EXT_PICT):
        return "ExtPict"
    return "Other"


def _graphemes(text):
    """Extended grapheme clusters (UAX #29 rules GB3-GB13) over the classes of _gcb.  It approximates the unicode-segmentation
    crate that tokenizers uses: the class tables are abridged (Extended_Pictographic by ranges, the rarer Prepend /
    Other_Grapheme_Extend / SpacingMark exceptions left out, Python's Unicode version rather than the crate's) and the Indic
    conjunct rule GB9c is not applied.  Only clusters shorter than 6 UTF-8 bytes reach the charsmap whole, so a difference
    matters only there: a base of 1-3 bytes followed by marks, joiners or selectors of 2-3 bytes."""
    out, cur, prev, ri, pict_zwj, in_pict = [], "", None, 0, False, False
    for ch in text:
        c = _gcb(ch)
        if prev is None:
            brk = False
        elif prev == "CR" and c == "LF":
            brk = False
        elif prev in ("Control", "CR", "LF") or c in ("Control", "CR", "LF"):
            brk = True
        elif prev == "L" and c in ("L", "V", "LV", "LVT"):
            brk = False
        elif prev in ("LV", "V") and c in ("V", "T"):
            brk = False
        elif prev in ("LVT", "T") and c == "T":
            brk = False
        elif c in ("Extend", "ZWJ", "SpacingMark") or prev == "Prepend":
            brk = False
        elif prev == "ZWJ" and c == "ExtPict" and pict_zwj:
            brk = False
        elif prev == "RI" and c == "RI" and ri % 2 == 1:
            brk = False
        else:
            brk = True
        if brk and cur:
            out.append(cur)
            cur = ""
        cur += ch
        # GB11 state: an ExtPict followed by Extend* then the current ZWJ
        pict_zwj = c == "ZWJ" and in_pict
        in_pict = c == "ExtPict" or (in_pict and c == "Extend")
        ri = ri + 1 if c == "RI" else 0
        prev = c
    if cur:
        out.append(cur)
    return out


class _Precompiled:
    """tokenizers' Precompiled normalizer (the SentencePiece charsmap): a darts double-array trie over UTF-8 byte strings
    whose values index a blob of NUL-terminated replacements."""

    def __init__(self, b64):
        blob = base64.b64decode(b64)
        if len(blob) < 4:
            raise K2Error("XLM-R tokenizer: the Precompiled charsmap is truncated")
        size = struct.unpack_from("<I", blob, 0)[0]
        if size % 4 or 4 + size > len(blob):
            raise K2Error("XLM-R tokenizer: the Precompiled charsmap's trie size does not fit the blob")
        self.array = struct.unpack_from(f"<{size // 4}I", blob, 4)
        self.normalized = blob[4 + size:]
        self._cache = {}

    def _prefix_values(self, key):
        """Darts common-prefix search: the values of every key that is a prefix of `key` (bytes), shortest first."""
        a, pos, out = self.array, 0, []
        unit = a[0]
        pos ^= (unit >> 10) << ((unit & (1 << 9)) >> 6)
        for c in key:
            if c == 0:
                break
            pos ^= c
            if pos >= len(a):
                return out
            unit = a[pos]
            if (unit & ((1 << 31) | 0xFF)) != c:
                return out
            pos ^= (unit >> 10) << ((unit & (1 << 9)) >> 6)
            if (unit >> 8) & 1:
                out.append(a[pos] & ((1 << 31) - 1))
        return out

    def transform(self, chunk):
        """The replacement of the SHORTEST charsmap key that prefixes chunk, or None (spm_precompiled's transform)."""
        hit = self._cache.get(chunk)
        if hit is None:
            v = self._prefix_values(chunk.encode("utf-8"))
            if v:
                end = self.normalized.find(b"\0", v[0])
                hit = self.normalized[v[0]:end if end >= 0 else len(self.normalized)].decode("utf-8")
            else:
                hit = False
            self._cache[chunk] = hit
        return hit if hit is not False else None

    def __call__(self, text):
        """Per grapheme cluster: a cluster shorter than 6 UTF-8 bytes is replaced whole when a key prefixes it; otherwise each
        character is replaced on its own (tokenizers' normalizers/precompiled.rs)."""
        out = []
        for g in _graphemes(text):
            if len(g.encode("utf-8")) < 6:
                r = self.transform(g)
                if r is not None:
                    out.append(r)
                    continue
            for ch in g:
                r = self.transform(ch)
                out.append(ch if r is None else r)
        return "".join(out)


def _normalizer(spec):
    """tokenizer.json normalizer -> str -> str; K2Error names any kind not implemented."""
    if spec is None:
        return lambda s: s
    kind = spec.get("type")
    if kind == "Sequence":
        parts = [_normalizer(s) for s in spec["normalizers"]]

        def seq(s):
            for p in parts:
                s = p(s)
            return s
        return seq
    if kind == "Precompiled":
        if not spec.get("precompiled_charsmap"):
            return lambda s: s
        return _Precompiled(spec["precompiled_charsmap"])
    if kind == "Replace":
        pat, content = spec["pattern"], spec["content"]
        if "String" in pat:
            return lambda s: s.replace(pat["String"], content)
        if "Regex" in pat:
            rx = re.compile(pat["Regex"])
            return lambda s: rx.sub(lambda m: content, s)
        raise K2Error(f"XLM-R tokenizer: Replace pattern {pat!r} is not implemented")
    raise K2Error(f"XLM-R tokenizer: normalizer {kind!r} is not implemented (only Precompiled, Replace and Sequence)")


def _metaspace_split(word, rep):
    """Split on the replacement character with tokenizers' MergedWithNext behaviour: each occurrence starts a piece."""
    out, cur = [], ""
    for ch in word:
        if ch == rep and cur:
            out.append(cur)
            cur = ""
        cur += ch
    if cur:
        out.append(cur)
    return out


def _pre_tokenizer(spec):
    """tokenizer.json pre_tokenizer -> str -> list[str]; K2Error names any kind not implemented."""
    if spec is None:
        return lambda s: [s] if s else []
    kind = spec.get("type")
    if kind == "Sequence":
        parts = [_pre_tokenizer(s) for s in spec["pretokenizers"]]

        def seq(s):
            words = [s]
            for p in parts:
                words = [w for x in words for w in p(x)]
            return words
        return seq
    if kind == "WhitespaceSplit":
        return lambda s: "".join(" " if ch in _WS else ch for ch in s).split()
    if kind == "Metaspace":
        rep = spec.get("replacement", "▁")
        if "prepend_scheme" in spec:
            scheme = spec["prepend_scheme"]
        else:
            scheme = "always" if spec.get("add_prefix_space", True) else "never"
        if scheme not in ("always", "never"):
            raise K2Error(f"XLM-R tokenizer: Metaspace prepend_scheme {scheme!r} is not implemented (only 'always', 'never')")
        split = spec.get("split", True)

        def meta(s):
            s = s.replace(" ", rep)
            if scheme == "always" and s and not s.startswith(rep):
                s = rep + s
            if not s:
                return []
            return _metaspace_split(s, rep) if split else [s]
        return meta
    raise K2Error(f"XLM-R tokenizer: pre-tokenizer {kind!r} is not implemented (only WhitespaceSplit, Metaspace and "
                  "Sequence)")


class _Unigram:
    """tokenizers' Unigram model: the best-scoring segmentation (encode_optimized), an unknown character scored
    min_score - 10, consecutive unknowns fused into one unknown token."""

    def __init__(self, spec):
        if spec.get("byte_fallback"):
            raise K2Error("XLM-R tokenizer: Unigram byte_fallback is not implemented")
        self.vocab = [(str(p), float(s)) for p, s in spec["vocab"]]
        self.unk_id = spec.get("unk_id")
        if self.unk_id is None:
            raise K2Error("XLM-R tokenizer: a Unigram model without unk_id is not implemented")
        self.ids = {}
        self.trie = {}
        for i, (piece, _) in enumerate(self.vocab):
            self.ids.setdefault(piece, i)
            node = self.trie
            for ch in piece:
                node = node.setdefault(ch, {})
            node[None] = self.ids[piece]
        self.unk_score = min(s for _, s in self.vocab) - 10.0
        self._cache = {}

    def __call__(self, word):
        hit = self._cache.get(word)
        if hit is not None:
            return hit
        n = len(word)
        score = [0.0] * (n + 1)
        start = [None] * (n + 1)
        tid = [0] * (n + 1)
        for i in range(n):
            base, node, single = score[i], self.trie, False
            j = i
            while j < n:
                node = node.get(word[j])
                if node is None:
                    break
                j += 1
                t = node.get(None)
                if t is not None:
                    cand = self.vocab[t][1] + base
                    if start[j] is None or cand > score[j]:
                        score[j], start[j], tid[j] = cand, i, t
                    single = single or j == i + 1
            if not single:
                cand = self.unk_score + base
                if start[i + 1] is None or cand > score[i + 1]:
                    score[i + 1], start[i + 1], tid[i + 1] = cand, i, self.unk_id
        pieces, unk, end = [], [], n
        while end > 0:
            s = start[end]
            if tid[end] == self.unk_id:
                unk.append(word[s:end])
            else:
                if unk:
                    pieces.append("".join(reversed(unk)))
                    unk = []
                pieces.append(self.vocab[tid[end]][0])
            end = s
        if unk:
            pieces.append("".join(reversed(unk)))
        ids = [self.ids.get(p, self.unk_id) for p in reversed(pieces)]
        self._cache[word] = ids
        return ids


class XLMRobertaTokenizer:
    """transformers 5's XLMRobertaTokenizer (the `tokenizers` backend, reading `tokenizer.json`), restated with the standard
    library:
      1. added tokens are matched in the raw text first, leftmost-longest (lstrip / rstrip take the neighbouring white space);
      2. every other section is normalised (Precompiled charsmap per grapheme cluster, Replace, Sequence),
      3. pre-tokenised (WhitespaceSplit, Metaspace with its "▁" prefix and split, Sequence),
      4. and segmented by the Unigram model;
      5. the post-processor's specials (<s> ... </s>) around the first max_length - 2 tokens, right-padded with the pad id to
         max_length, and the attention mask.
    Kinds of normalizer, pre-tokenizer, model or post-processor outside this list are refused by name."""

    def __init__(self, spec, pad_token="<pad>", model_max_length=77):
        self.model_max_length = int(model_max_length)
        m = spec.get("model") or {}
        if m.get("type") != "Unigram":
            raise K2Error(f"XLM-R tokenizer: model {m.get('type')!r} is not implemented (only Unigram)")
        self.model = _Unigram(m)
        self.normalize = _normalizer(spec.get("normalizer"))
        self.pre_tokenize = _pre_tokenizer(spec.get("pre_tokenizer"))
        self.added = {}
        for t in spec.get("added_tokens", []):
            if t.get("single_word") or t.get("normalized"):
                raise K2Error(f"XLM-R tokenizer: added token {t['content']!r} with single_word / normalized is not "
                              "implemented")
            self.added[t["content"]] = (int(t["id"]), bool(t.get("lstrip")), bool(t.get("rstrip")))
        self._added_by_len = sorted(self.added, key=len, reverse=True)
        self.prefix, self.suffix = self._template(spec.get("post_processor"))
        if pad_token in self.added:
            self.pad_token_id = self.added[pad_token][0]
        elif pad_token in self.model.ids:
            self.pad_token_id = self.model.ids[pad_token]
        else:
            raise K2Error(f"XLM-R tokenizer: the pad token {pad_token!r} is not in the vocabulary")
        self.vocab_size = max([len(self.model.vocab)] + [i + 1 for i, _, _ in self.added.values()])

    def _token_id(self, tok):
        if tok in self.added:
            return self.added[tok][0]
        if tok in self.model.ids:
            return self.model.ids[tok]
        raise K2Error(f"XLM-R tokenizer: the post-processor's token {tok!r} is not in the vocabulary")

    def _template(self, spec):
        """(ids before, ids after) the sequence, from TemplateProcessing's single template or RobertaProcessing."""
        if spec is None:
            return [], []
        kind = spec.get("type")
        if kind == "RobertaProcessing":
            return [int(spec["cls"][1])], [int(spec["sep"][1])]
        if kind != "TemplateProcessing":
            raise K2Error(f"XLM-R tokenizer: post-processor {kind!r} is not implemented (only TemplateProcessing and "
                          "RobertaProcessing)")
        specials = spec.get("special_tokens", {})
        before, after, seen = [], [], False
        for item in spec["single"]:
            if "Sequence" in item:
                if item["Sequence"]["id"] != "A" or seen:
                    raise K2Error("XLM-R tokenizer: a single template other than specials around $A is not implemented")
                seen = True
            else:
                name = item["SpecialToken"]["id"]
                ids = specials[name]["ids"] if name in specials else [self._token_id(name)]
                (after if seen else before).extend(int(i) for i in ids)
        return before, after

    @classmethod
    def from_dir(cls, path, model_max_length=77):
        """A transformers tokenizer folder: tokenizer.json, and special_tokens_map.json / tokenizer_config.json when present
        (the pad token; default "<pad>").  model_max_length is the row length (encode_text's max_length=77)."""
        spec = read_json(path, "tokenizer.json", "XLM-R tokenizer")
        cfg = {}
        for name in ("tokenizer_config.json", "special_tokens_map.json"):
            cfg.update(read_json(path, name, "XLM-R tokenizer", False) or {})
        pad = cfg.get("pad_token", "<pad>")
        pad = pad["content"] if isinstance(pad, dict) else pad
        return cls(spec, pad_token=pad, model_max_length=model_max_length)

    def _split_added(self, text):
        """[(segment, added id or None)] with the added tokens matched leftmost-longest in the raw text."""
        out, i, start, n = [], 0, 0, len(text)
        while i < n:
            m = next((s for s in self._added_by_len if text.startswith(s, i)), None)
            if m is None:
                i += 1
                continue
            tid, lstrip, rstrip = self.added[m]
            a, b = i, i + len(m)
            if lstrip:
                while a > start and text[a - 1] in _WS:
                    a -= 1
            if rstrip:
                while b < n and text[b] in _WS:
                    b += 1
            if a > start:
                out.append((text[start:a], None))
            out.append((m, tid))
            i = start = b
        if start < n:
            out.append((text[start:], None))
        return out

    def tokenize_ids(self, text):
        """The token ids of one text, without the post-processor's specials."""
        ids = []
        for seg, tid in self._split_added(text):
            if tid is not None:
                ids.append(tid)
                continue
            for word in self.pre_tokenize(self.normalize(seg)):
                ids += self.model(word)
        return ids

    def __call__(self, texts, max_length=None):
        """texts: str or list[str] -> dict(input_ids int64 [n, L], attention_mask int64 [n, L]) on the CPU, L = max_length
        (default model_max_length): padding="max_length", truncation=True."""
        if isinstance(texts, str):
            texts = [texts]
        L = self.model_max_length if max_length is None else int(max_length)
        keep = L - len(self.prefix) - len(self.suffix)
        if keep < 0:
            raise K2Error(f"XLM-R tokenizer: max_length {L} leaves no room for the special tokens")
        ids = torch.full((len(texts), L), self.pad_token_id, dtype=torch.int64)
        mask = torch.zeros(len(texts), L, dtype=torch.int64)
        for r, t in enumerate(texts):
            row = self.prefix + self.tokenize_ids(t)[:keep] + self.suffix
            ids[r, :len(row)] = torch.tensor(row, dtype=torch.int64)
            mask[r, :len(row)] = 1
        return {"input_ids": ids, "attention_mask": mask}


# ---------------------------------------------------------------------------------------------------------------------------
# tower
# ---------------------------------------------------------------------------------------------------------------------------
class MultilingualCLIP(Tower):
    """The reference's MultilingualCLIP on this package's kernels.  sd: state dict in this module's names
    (checkpoints.mclip_to_k2); config: the transformers config.json dict; tokenizer: an XLMRobertaTokenizer (needed by
    __call__ only).  `tokens` is the row length __call__ produces: the tokenizer's model_max_length (77), or 77 without one."""

    what = "M-CLIP text encoder"

    def __init__(self, sd, config, device="cuda", tokenizer=None):
        c = xlmr_config(config)
        self.cfg, self.device, self.tokenizer = c, torch.device(device), tokenizer
        self.tokens = tokenizer.model_max_length if tokenizer is not None else 77
        if not 2 <= self.tokens <= c["max_tokens"]:
            raise K2Error(f"M-CLIP text encoder: {self.tokens} tokens per row are not implemented (at most "
                          f"{c['max_tokens']}: k2_attention_small's 128 and the position table)")
        if tokenizer is not None and tokenizer.vocab_size > c["vocab_size"]:
            raise K2Error(f"M-CLIP text encoder: the tokenizer's ids reach {tokenizer.vocab_size - 1}, beyond the vocabulary "
                          f"of {c['vocab_size']}")
        if tokenizer is not None and tokenizer.pad_token_id != c["pad_token_id"]:
            raise K2Error(f"M-CLIP text encoder: the tokenizer pads with {tokenizer.pad_token_id}, the config's pad_token_id "
                          f"is {c['pad_token_id']}")
        H = c["hidden_size"]
        proj = sd.get("proj.weight")
        # the output width is the projection's; one that is missing, not 2-D or empty is refused below as (-1, H)
        self.out_features = int(proj.shape[0]) if proj is not None and proj.dim() == 2 and proj.shape[0] > 0 else -1
        want = {"word_embedding": (c["vocab_size"], H), "position_embedding": (c["max_position_embeddings"], H),
                "token_type_embedding": (1, H), "emb_ln.weight": (H,), "emb_ln.bias": (H,),
                "proj.weight": (self.out_features, H), "proj.bias": (self.out_features,)}
        want.update({f"layers.{i}.{k}": s for i in range(c["num_hidden_layers"])
                     for k, s in layer_shapes(H, c["intermediate_size"]).items()})
        self._take(sd, want)

    @classmethod
    def from_state_dict(cls, state_dict, config, tokenizer=None, device="cuda"):
        """From the reference's MultilingualCLIP state dict (transformer.* + LinearTransformation.*) and the config.json
        dict; packs the weights."""
        from ..checkpoints import mclip_to_k2
        c = xlmr_config(config)
        return cls(mclip_to_k2(state_dict, c["num_hidden_layers"]), config, device, tokenizer).finalize()

    @classmethod
    def from_pretrained(cls, path, device="cuda"):
        """The reference's `2_1/text_encoder/` folder: config.json, pytorch_model.bin (or model.safetensors) and the
        tokenizer's tokenizer.json (+ special_tokens_map.json / tokenizer_config.json)."""
        config = read_json(path, "config.json", cls.what)
        tok = XLMRobertaTokenizer.from_dir(path)
        sd = load_weights(path, ("pytorch_model.bin", "model.safetensors"), cls.what)
        return cls.from_state_dict(sd, config, tokenizer=tok, device=device)

    def _pack(self):
        """fp16 GEMM weights [N, K] and tables, fp32 biases / LayerNorm parameters / Linear."""
        c, dev, sd = self.cfg, self.device, self.sd
        return {"word": f16(sd["word_embedding"], dev), "pos": f16(sd["position_embedding"], dev),
                "type": f16(sd["token_type_embedding"][0], dev),
                "emb_ln": (f32(sd["emb_ln.weight"], dev), f32(sd["emb_ln.bias"], dev)),
                "proj": (f32(sd["proj.weight"], dev), f32(sd["proj.bias"], dev)),
                "layers": pack_layers(lambda i, name: sd[f"layers.{i}.{name}"], c["num_hidden_layers"], dev)}

    def _plan(self, n, T=None):
        return super()._plan(n, self.tokens if T is None else T)

    def _new_plan(self, n, T):
        return _XLMRPlan(self, n, T)

    @torch.no_grad()
    def forward(self, input_ids, attention_mask, use_graph=True):
        """input_ids integer [n, T], attention_mask [n, T] (nonzero = kept), T <= max_tokens -> (last_hidden_state fp16
        [n, T, hidden], pooled fp32 [n, out_features]) on the device: MultilingualCLIP.forward's (embs, LinearTransformation
        of the masked mean).  One CUDA graph replay of the (n, T) launch plan (use_graph=False: the same launches one by
        one).  Ids outside [0, vocab_size) are refused before anything is copied."""
        self._check_ids(input_ids, self.cfg["max_tokens"])
        if tuple(attention_mask.shape) != tuple(input_ids.shape) or attention_mask.is_floating_point():
            raise K2Error(f"M-CLIP text encoder: attention_mask must be an integer or bool [n, T] like input_ids, got "
                          f"{attention_mask.dtype} {list(attention_mask.shape)}")
        plan = self._plan(*input_ids.shape)
        plan.ids.copy_(input_ids)
        plan.mask.copy_(attention_mask != 0)
        plan.run(use_graph)
        return plan.hidden.clone(), plan.out.clone()

    def __call__(self, prompt, batch_size):
        """The embedders' text_encoder protocol (encode_text, kandinsky2_1_model.py:116-131): (full_emb fp16
        [2B, tokens, hidden], pooled_emb fp32 [2B, out_features]) for [prompt x B | "" x B], on the device.  Each distinct
        prompt is tokenized and encoded once and its rows are gathered back."""
        if self.tokenizer is None:
            raise K2Error("M-CLIP text encoder: calling it with a prompt needs tokenizer=")

        def encode(distinct):
            tok = self.tokenizer(distinct, max_length=self.tokens)
            return self.forward(tok["input_ids"], tok["attention_mask"])
        return self._encode_distinct([prompt] * batch_size + [""] * batch_size, encode)


class _XLMRPlan(LaunchPlan):
    """The tower on n rows of T tokens as one static launch list over fixed buffers (replayed as one CUDA graph): ids ->
    embed -> L post-LN layers (self.hidden, last_hidden_state) -> masked mean (fp32) -> Linear (self.out)."""

    def __init__(self, tower, n, T):
        super().__init__(tower.device, n)
        self.t, self.n, self.T = tower, n, T
        self.ids = torch.zeros(n, T, device=self.dev, dtype=torch.int32)
        self.mask = torch.ones(n, T, device=self.dev, dtype=torch.uint8)
        self.out = torch.zeros(n, tower.out_features, device=self.dev, dtype=torch.float32)
        self._build()

    def _build(self):
        c, pk, n, T, S = self.t.cfg, self.t._packed, self.n, self.T, self._add
        H, heads, eps = c["hidden_size"], c["num_attention_heads"], c["layer_norm_eps"]
        x = self._new(n, T, H)
        S(lambda: ops.xlmr_embed(self.ids, c["pad_token_id"], pk["word"], pk["pos"], pk["type"], *pk["emb_ln"], eps, out=x),
          "embed")
        scale = c["head_dim"] ** -0.5
        self.hidden = record_layers(
            self, x, pk["layers"],
            lambda qkv, out: ops.attention_small(qkv, heads, keep_mask=self.mask, causal=False, scale=scale, out=out),
            4 * n * heads * T * T * c["head_dim"], eps, post_ln=True)
        pooled = self._new(n, H, dtype=torch.float32)
        S(lambda: ops.masked_mean_f16(self.hidden, self.mask, out=pooled), "masked_mean")
        S(lambda: ops.linear(pooled, *pk["proj"], out=self.out), "linear", 2 * n * H * self.t.out_features)


class TextEncoder:
    """The reference's TextEncoder (model/text_encoders.py:125-167) for model_name="multiclip", the one Kandinsky 2.1 uses:
    TextEncoder(model_path, "multiclip", in_features=1024, out_features=768) reads the text_encoder folder, and
    forward(tokens, mask) -> (full_out, pooled_out).  Other model_names are refused."""

    def __init__(self, model_path, model_name="multiclip", in_features=1024, out_features=768, device="cuda"):
        if model_name != "multiclip":
            raise K2Error(f"TextEncoder: model_name {model_name!r} is not implemented (only 'multiclip', Kandinsky 2.1's)")
        self.model_name = model_name
        self.model = MultilingualCLIP.from_pretrained(model_path, device=device)
        got = (self.model.cfg["hidden_size"], self.model.out_features)
        if got != (int(in_features), int(out_features)):
            raise K2Error(f"TextEncoder: the folder's tower maps {got[0]} -> {got[1]}, not {in_features} -> {out_features}")

    def forward(self, tokens, mask=None):
        if mask is None:
            mask = torch.ones_like(tokens)
        return self.model.forward(tokens, mask)

    __call__ = forward
