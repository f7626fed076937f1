"""The CLIP ViT-L/14 of the Kandinsky 2.1 prior pipeline: OpenAI's `clip` model (`ViT-L-14.pt`), which the reference loads
with `clip.load(..., jit=False)` (kandinsky2_1_model.py:64-67) and runs for every 2.1 prompt (the text tower in
`generate_clip_emb`, :159-166), for the image items of `mix_images` (`encode_images`, :177-181) and for the decoder negative
(`create_zero_img_emb`, :294-297).  The tokenizer is the reference's `CustomizedTokenizer` (its model/prior.py:387-416).

The towers are read from the checkpoint's tensor shapes (checkpoints.openai_clip_to_k2; ViT-L/14: text 12 layers of width
768, image 24 layers of width 1024, heads of 64, MLP 4 x width, patch 14, 257 image tokens, 77 text positions, embeddings
of 768) and reuse the Kandinsky 2.2 towers' launch plans (model/clip_text.py, model/clip_vision.py) with OpenAI's QuickGELU,
x sigmoid(1.702 x) (k2_quick_gelu_f16), as the MLP activation.  Per batch shape one LaunchPlan, replayed as one CUDA graph:
    text:   k2_clip_text_embed -> pre-LN layers with k2_attention_small (causal, no key mask: OpenAI's build_attention_mask;
            the padded positions hold token 0 and are attended causally) -> ln_final over every row -> k2_clip_text_pool
            (the first argmax of the ids, i.e. the end-of-text token) -> fp32 projection;
    image:  k2_clip_patchify -> one GEMM (patch conv, class embedding column, positional embedding as the residual) ->
            ln_pre -> pre-LN layers with k2_attention_d64 (no encoder tokens, 257 keys: a ragged last key block) -> ln_post
            of the CLS rows -> fp32 projection.
fp16 storage, fp32 accumulation, the prior's LayerNorm statistics; the projections (`x @ text_projection`, `x @ visual.proj`
in the reference) run in fp32.

Preprocessing is OpenAI's `clip` transform (Resize(224, BICUBIC), CenterCrop(224), RGB, ToTensor, Normalize) restated with
PIL and numpy; the crop offsets are int(round((h - 224) / 2)) and the scaling an fp32 division by 255, so images whose size
difference is odd are cropped one pixel apart from transformers' CLIPImageProcessor (model/clip_vision.py).

Text cleaning follows the `clip` package's SimpleTokenizer: ftfy.fix_text, html.unescape twice, runs of whitespace -> " ",
strip, lower.  ftfy is not a dependency: fix_text_restated restates the deterministic parts of its default fix_text that
prompts meet (terminal escapes, C1 controls read as Windows-1252, Latin ligatures, full-width characters, curly quotes, line
breaks, surrogates, control characters, NFC).  ftfy's mojibake repair (fix_encoding) and its own HTML step (the
html.unescape calls follow anyway) are not restated: text that ftfy would re-decode as mis-encoded UTF-8 tokenizes as it is.

Parity: tests/test_cpu_clip_vitl14.py pins the oracle (tests/openai_clip_oracle.py) and the preprocessing to transformers and
torchvision (tests/golden/openai_clip_tiny.pt); tests/test_gpu_zz_clip_vitl14.py runs both towers against the golden and, at
full size on synthetic weights, against the fp32 oracle.
"""
import gzip
import html
import os
import re
import unicodedata

import numpy as np
import torch

from .. import ops
from .._native import K2Error
from .clip_text import CLIPTextTower, CLIPTokenizer, _clip_split, bytes_to_unicode
from .clip_vision import OPENAI_CLIP_MEAN, OPENAI_CLIP_STD, CLIPVisionTower

IMAGE_SIZE = 224

# ---------------------------------------------------------------------------------------------------------------------------
# text cleaning and the tokenizer
# ---------------------------------------------------------------------------------------------------------------------------
# ftfy's fixes.LIGATURES (Latin ligatures and digraphs -> their letters)
_LIGATURES = {ord(k): v for k, v in {
    "Ĳ": "IJ", "ĳ": "ij", "ŉ": "ʼn", "Ǳ": "DZ", "ǲ": "Dz", "ǳ": "dz", "Ǆ": "DŽ", "ǅ": "Dž", "ǆ": "dž", "Ǉ": "LJ",
    "ǈ": "Lj", "ǉ": "lj", "Ǌ": "NJ", "ǋ": "Nj", "ǌ": "nj", "ﬀ": "ff", "ﬁ": "fi", "ﬂ": "fl", "ﬃ": "ffi", "ﬄ": "ffl",
    "ﬅ": "ſt", "ﬆ": "st"}.items()}
# ftfy's chardata.WIDTH_MAP: the full-width / half-width forms -> their NFKC characters, the ideographic space -> " "
_WIDTH = {i: unicodedata.normalize("NFKC", chr(i)) for i in range(0xFF01, 0xFFF0)
          if unicodedata.normalize("NFKC", chr(i)) != chr(i)}
_WIDTH[0x3000] = " "
# ftfy's chardata.CONTROL_CHARS: removed (tab, line feed, form feed and carriage return are kept)
_CONTROL = {i: None for i in (*range(0x00, 0x09), 0x0B, *range(0x0E, 0x20), 0x7F, *range(0x206A, 0x2070), 0xFEFF,
                              *range(0xFFF9, 0xFFFD))}
_TERMINAL_ESCAPE = re.compile(r"\033\[((?:\d|;)*)([a-zA-Z])")
_C1 = re.compile("[\x80-\x9f]")
_SURROGATE_PAIR = re.compile("[\ud800-\udbff][\udc00-\udfff]")
_SURROGATE = re.compile("[\ud800-\udfff]")


def _c1_as_cp1252(m):
    try:
        return bytes([ord(m.group(0))]).decode("cp1252")
    except UnicodeDecodeError:          # 0x81, 0x8d, 0x8f, 0x90, 0x9d: ftfy's sloppy-windows-1252 keeps them
        return m.group(0)


def fix_text_restated(text):
    """The deterministic part of ftfy.fix_text's defaults (see the module docstring): one pass of each fix, then NFC."""
    text = _TERMINAL_ESCAPE.sub("", text)
    text = _C1.sub(_c1_as_cp1252, text)
    text = text.translate(_LIGATURES).translate(_WIDTH)
    text = re.sub("[\u02bc\u2018-\u201b]", "'", text)
    text = re.sub("[\u201c-\u201f]", '"', text)
    for br in ("\r\n", "\r", "\u2028", "\u2029", "\x85"):
        text = text.replace(br, "\n")
    text = _SURROGATE_PAIR.sub(lambda m: (m.group(0).encode("utf-16", "surrogatepass").decode("utf-16")), text)
    text = _SURROGATE.sub("\ufffd", text)
    text = text.translate(_CONTROL)
    return unicodedata.normalize("NFC", text)


def clean_text(text):
    """SimpleTokenizer's whitespace_clean(basic_clean(text)).lower(), with fix_text_restated for ftfy.fix_text."""
    text = html.unescape(html.unescape(fix_text_restated(text))).strip()
    return re.sub(r"\s+", " ", text).strip().lower()


class OpenAICLIPTokenizer(CLIPTokenizer):
    """The reference's CustomizedTokenizer: the `clip` package's SimpleTokenizer (the BPE of OpenAI CLIP) with
    padded_tokens_and_mask.  Per text: clean_text, split by the CLIP pattern (the start / end-of-text strings are one piece
    each and map to their ids), each piece's UTF-8 bytes mapped to bytes_to_unicode characters, then BPE with "</w>" on the
    last symbol, merging every occurrence of the lowest-ranked pair left to right until none is left.  The vocabulary and
    merges are CLIPTokenizer's; its transformers-side steps (added-token matching, normalisation, padding) are not used."""

    def __init__(self, vocab, merges, **kwargs):
        kwargs.setdefault("model_max_length", 77)
        super().__init__(vocab, merges, **kwargs)
        self.sot_token, self.eot_token = self.vocab["<|startoftext|>"], self.vocab["<|endoftext|>"]

    @classmethod
    def from_bpe(cls, path):
        """clip's bpe_simple_vocab_16e6.txt.gz (or a folder holding vocab.json + merges.txt of the same vocabulary, as
        CLIPTokenizer.from_dir reads it).  The vocabulary is SimpleTokenizer's: the 256 byte characters, the same with
        "</w>", the merges of lines 1 .. 49152 - 256 - 2 (empty lines skipped), "<|startoftext|>", "<|endoftext|>"."""
        path = os.fspath(path)
        if os.path.isdir(path):
            return cls.from_dir(path)
        if not os.path.exists(path):
            raise K2Error(f"OpenAI CLIP tokenizer: {path} not found")
        with gzip.open(path) as fh:
            lines = fh.read().decode("utf-8").split("\n")
        merges = [tuple(ln.split()) for ln in lines[1:49152 - 256 - 2 + 1] if ln.strip()]
        chars = list(bytes_to_unicode().values())
        vocab = chars + [c + "</w>" for c in chars] + ["".join(m) for m in merges] + ["<|startoftext|>", "<|endoftext|>"]
        return cls({v: i for i, v in enumerate(vocab)}, merges)

    def _bpe(self, word):
        hit = self._cache.get(word)
        if hit is not None:
            return hit
        syms = list(word)
        syms[-1] += "</w>"
        while len(syms) > 1:
            pairs = {(a, b) for a, b in zip(syms, syms[1:])}
            best = min(pairs, key=lambda p: self.ranks.get(p, float("inf")))
            if best not in self.ranks:
                break
            merged, i = [], 0
            while i < len(syms):
                if i < len(syms) - 1 and (syms[i], syms[i + 1]) == best:
                    merged.append(syms[i] + syms[i + 1])
                    i += 2
                else:
                    merged.append(syms[i])
                    i += 1
            syms = merged
        ids = [self.vocab[s] for s in syms]
        self._cache[word] = ids
        return ids

    def tokenize_ids(self, text):
        """SimpleTokenizer.encode: the ids of one text, without start / end of text."""
        ids = []
        for piece in _clip_split(clean_text(text)):
            if piece in ("<|startoftext|>", "<|endoftext|>"):
                ids.append(self.vocab[piece])
            else:
                ids += self._bpe("".join(self.byte_map[b] for b in piece.encode("utf-8")))
        return ids

    def padded_tokens_and_mask(self, texts, text_ctx):
        """CustomizedTokenizer.padded_tokens_and_mask: texts list[str] -> (int32 [n, text_ctx], bool [n, text_ctx]).  Each
        row is [sot] + ids + [eot]; a longer row is cut to text_ctx with its last token set to eot; padding is 0; the mask is
        True on the first min(text_ctx, len) positions."""
        if not isinstance(texts, list) or not all(isinstance(t, str) for t in texts):
            raise K2Error("OpenAI CLIP tokenizer: texts must be a list of strings")
        rows = [[self.sot_token] + self.tokenize_ids(t) + [self.eot_token] for t in texts]
        tok = torch.zeros(len(rows), text_ctx, dtype=torch.int)
        mask = torch.zeros(len(rows), text_ctx, dtype=torch.bool)
        for i, r in enumerate(rows):
            mask[i, :min(text_ctx, len(r))] = True
            if len(r) > text_ctx:
                r = r[:text_ctx]
                r[-1] = self.eot_token
            tok[i, :len(r)] = torch.tensor(r, dtype=torch.int)
        return tok, mask


# ---------------------------------------------------------------------------------------------------------------------------
# preprocessing
# ---------------------------------------------------------------------------------------------------------------------------
def preprocess_openai(images, size=IMAGE_SIZE):
    """OpenAI clip's _transform(size), restated -> fp32 [B, 3, size, size] on the CPU.  Per image: resize (PIL BICUBIC, in the
    image's own mode) so that the shortest edge is `size` and the long edge int(size * long / short); center-crop at
    (int(round((h - size) / 2)), int(round((w - size) / 2))); convert to RGB; fp32 uint8 / 255; (x - mean) / std in fp32."""
    from PIL import Image
    if isinstance(images, Image.Image):
        images = [images]
    mean = np.array(OPENAI_CLIP_MEAN, dtype=np.float32)[:, None, None]
    std = np.array(OPENAI_CLIP_STD, dtype=np.float32)[:, None, None]
    out = []
    for img in images:
        w, h = img.size
        short, long = (w, h) if w <= h else (h, w)
        new_long = int(size * long / short)
        nw, nh = (size, new_long) if w <= h else (new_long, size)
        if (nw, nh) != (w, h):
            img = img.resize((nw, nh), resample=Image.BICUBIC)
        top, left = int(round((nh - size) / 2.0)), int(round((nw - size) / 2.0))
        img = img.crop((left, top, left + size, top + size)).convert("RGB")
        a = np.asarray(img, dtype=np.uint8).transpose(2, 0, 1).astype(np.float32) / np.float32(255)
        out.append(torch.from_numpy(np.ascontiguousarray((a - mean) / std)))
    return torch.stack(out)


# ---------------------------------------------------------------------------------------------------------------------------
# towers
# ---------------------------------------------------------------------------------------------------------------------------
class OpenAICLIPTextTower(CLIPTextTower):
    """The text side of OpenAI CLIP (`generate_clip_emb`'s tower lines) on the 2.2 text tower's launch plan with QuickGELU.
    sd: the text state dict of checkpoints.openai_clip_to_k2; geo: its geometry["text"]; tokenizer: an OpenAICLIPTokenizer
    (needed by __call__ only)."""

    what = "OpenAI CLIP text tower"
    act = "quick_gelu"

    def __init__(self, sd, geo, device="cuda", tokenizer=None):
        H, L, T = geo["width"], geo["layers"], geo["context"]
        if T > 128:
            raise K2Error(f"OpenAI CLIP text tower: {T} positions are not implemented (at most 128)")
        self.cfg = dict(hidden_size=H, intermediate_size=geo["mlp"], num_hidden_layers=L, num_attention_heads=geo["heads"],
                        head_dim=64, max_position_embeddings=T, vocab_size=geo["vocab"], projection_dim=geo["embed_dim"],
                        layer_norm_eps=1e-5, pool_eos=-1)
        self.device, self.tokenizer, self.tokens = torch.device(device), tokenizer, T
        if tokenizer is not None and max(tokenizer.vocab.values()) >= geo["vocab"]:
            raise K2Error(f"OpenAI CLIP text tower: the tokenizer's ids reach {max(tokenizer.vocab.values())}, beyond the "
                          f"vocabulary of {geo['vocab']}")
        self._take(sd, self._want())

    def __call__(self, prompts):
        """The 2.1 PriorEmbedder's clip_text protocol, with generate_clip_emb's semantics: list[str] -> (txt_feat fp32
        [n, embed_dim], txt_feat_seq fp32 [n, context, width] (the ln_final rows), mask bool [n, context] from the tokenizer),
        on the device.  Each distinct prompt is encoded once and its rows are gathered back."""
        if self.tokenizer is None:
            raise K2Error("OpenAI CLIP text tower: calling it with prompts needs tokenizer=")
        if isinstance(prompts, str):
            prompts = [prompts]

        def encode(distinct):
            tok, mask = self.tokenizer.padded_tokens_and_mask(distinct, self.tokens)
            hid, emb = self.forward(tok)
            return emb, hid.float(), mask.to(self.device)
        return self._encode_distinct(prompts, encode)


class OpenAICLIPVisionTower(CLIPVisionTower):
    """The image side of OpenAI CLIP (`clip_model.encode_image`) on the 2.2 image tower's launch plan, with QuickGELU and
    k2_attention_d64 (heads of 64).  sd: the vision state dict of checkpoints.openai_clip_to_k2; geo: its
    geometry["vision"].  zero_embed() (the 2.2 tower's: the tower on an all-zero [1, 3, S, S] tensor, not preprocessed) is
    the reference's create_zero_img_emb."""

    what = "OpenAI CLIP vision tower"
    act = "quick_gelu"

    def __init__(self, sd, geo, device="cuda"):
        P = geo["patch"]
        self.cfg = dict(hidden_size=geo["width"], intermediate_size=geo["mlp"], num_hidden_layers=geo["layers"],
                        num_attention_heads=geo["heads"], head_dim=64, image_size=geo["image_size"], patch_size=P,
                        projection_dim=geo["embed_dim"], layer_norm_eps=1e-5, tokens=geo["tokens"],
                        kp=(3 * P * P + 1 + 63) // 64 * 64)
        self.device, self.preprocessor_config = torch.device(device), None
        self._take(sd, self._want())

    def attend(self, qkv, out):
        """k2_attention_d64 over the image tokens (no encoder tokens; per-head [q | k | v], scale 1/8)."""
        return ops.attention_d64(qkv, self.cfg["num_attention_heads"], scale=0.125, out=out)

    def preprocess(self, images):
        """PIL image(s) -> fp32 [B, 3, S, S] on the CPU: OpenAI clip's transform (preprocess_openai)."""
        return preprocess_openai(images, self.cfg["image_size"])


def load_openai_clip(path_or_sd, device="cuda", bpe_path=None):
    """(text tower, image tower) of an OpenAI CLIP checkpoint (a path to a TorchScript archive or a torch.save'd state dict,
    or the state dict itself; checkpoints.load_openai_clip), packed on `device`.  bpe_path: clip's
    bpe_simple_vocab_16e6.txt.gz (or a vocab.json + merges.txt folder) for the text tower's tokenizer; None = no tokenizer."""
    from ..checkpoints import load_openai_clip as load_sd
    from ..checkpoints import openai_clip_to_k2
    text, vision, geo = openai_clip_to_k2(load_sd(path_or_sd))
    tok = OpenAICLIPTokenizer.from_bpe(bpe_path) if bpe_path is not None else None
    return (OpenAICLIPTextTower(text, geo["text"], device, tok).finalize(),
            OpenAICLIPVisionTower(vision, geo["vision"], device).finalize())
