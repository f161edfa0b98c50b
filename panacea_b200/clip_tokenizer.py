"""CLIP's byte-level BPE tokenizer, as `open_clip.tokenize` applies it for `FrozenOpenCLIPEmbedder.forward`
(reference sgm/modules/encoders/modules.py:604-607).

This restates the published CLIP tokenizer algorithm:
  * vocabulary from `bpe_simple_vocab_16e6.txt.gz`: merges are lines [1, 1 + 49152 - 256 - 2) of the file; the
    symbols are the 256 printable stand-ins of `bytes_to_unicode`, the same 256 with `</w>`, one symbol per merge,
    then `<start_of_text>` and `<end_of_text>` (ids len - 2 and len - 1: 49406 / 49407 for the released file);
  * text cleaning: ftfy.fix_text (when installed), html.unescape twice, strip, whitespace runs -> one space, lower();
  * words from the pre-tokenizer pattern below (the `regex` module, case-insensitive);
  * each word is byte-encoded, `</w>` marks its last symbol, and adjacent pairs are merged by rank until no ranked pair
    is left;
  * `tokenize` makes int64 [b, context_length] rows [sot] + ids + [eot] with zero padding; a longer row is cut to
    context_length and its last position set to eot.

The vocabulary file is not part of this repository: it comes from an explicit path, or from the copy bundled with
the `open_clip` package when that is importable."""
from __future__ import annotations

import gzip
import html
import string
from functools import lru_cache
from pathlib import Path

import regex
import torch

BPE_FILE = "bpe_simple_vocab_16e6.txt.gz"
N_MERGES = 49152 - 256 - 2
_PATTERN = regex.compile(r"""<start_of_text>|<end_of_text>|'s|'t|'re|'ve|'m|'ll|'d|[\p{L}]+|[\p{N}]|[^\s\p{L}\p{N}]+""",
                         regex.IGNORECASE)
_ASCII = set(string.printable)


def find_bpe_path(bpe_path=None) -> Path:
    """The vocabulary file: `bpe_path` when given, else the one bundled with the open_clip package."""
    if bpe_path is not None:
        p = Path(bpe_path)
        if not p.is_file():
            raise FileNotFoundError(f"CLIP BPE vocabulary {p} does not exist")
        return p
    try:
        import open_clip
        p = Path(open_clip.__file__).resolve().parent / BPE_FILE
        if p.is_file():
            return p
    except ImportError:
        pass
    raise FileNotFoundError(f"no CLIP BPE vocabulary: pass bpe_path=<path to {BPE_FILE}> (the embedder's bpe_path "
                            f"parameter), or install open_clip, whose package bundles {BPE_FILE}")


@lru_cache()
def bytes_to_unicode() -> dict:
    """byte -> printable unicode character: printable latin-1 bytes map to themselves, the other 68 to 256 + n."""
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs = bs[:]
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return dict(zip(bs, map(chr, cs)))


def _pairs(word):
    return {(a, b) for a, b in zip(word[:-1], word[1:])}


def _clean(text: str) -> str:
    try:
        import ftfy
        text = ftfy.fix_text(text)
    except ImportError:
        # ftfy leaves printable ASCII unchanged; anything else could tokenize differently without it
        bad = sorted({c for c in text if c not in _ASCII})
        if bad:
            raise NotImplementedError(f"text contains non-ASCII characters {bad[:5]!r}: tokenizing it like open_clip needs "
                                      "ftfy (ftfy.fix_text), which is not installed")
    text = html.unescape(html.unescape(text)).strip()
    return regex.sub(r"\s+", " ", text).strip().lower()


class ClipTokenizer:
    def __init__(self, bpe_path=None):
        self.path = find_bpe_path(bpe_path)
        raw = gzip.open(self.path).read() if self.path.suffix == ".gz" else self.path.read_bytes()
        lines = raw.decode("utf-8").split("\n")[1:1 + N_MERGES]
        merges = [tuple(m.split()) for m in lines if m.strip()]
        self.byte_encoder = bytes_to_unicode()
        vocab = list(self.byte_encoder.values())
        vocab = vocab + [v + "</w>" for v in vocab] + ["".join(m) for m in merges] + ["<start_of_text>", "<end_of_text>"]
        self.encoder = {v: i for i, v in enumerate(vocab)}
        self.ranks = {m: i for i, m in enumerate(merges)}
        self.vocab_size = len(vocab)
        self.sot, self.eot = self.encoder["<start_of_text>"], self.encoder["<end_of_text>"]
        self._cache = {"<start_of_text>": "<start_of_text>", "<end_of_text>": "<end_of_text>"}

    def bpe(self, token: str) -> str:
        if token in self._cache:
            return self._cache[token]
        word = tuple(token[:-1]) + (token[-1] + "</w>",)
        pairs = _pairs(word)
        while pairs:
            first, second = min(pairs, key=lambda p: self.ranks.get(p, float("inf")))
            if (first, second) not in self.ranks:
                break
            out, i = [], 0
            while i < len(word):
                if word[i] == first and i + 1 < len(word) and word[i + 1] == second:
                    out.append(first + second)
                    i += 2
                else:
                    out.append(word[i])
                    i += 1
            word = tuple(out)
            pairs = _pairs(word) if len(word) > 1 else set()
        res = " ".join(word)
        self._cache[token] = res
        return res

    def encode(self, text: str) -> list:
        ids = []
        for tok in _PATTERN.findall(_clean(text)):
            tok = "".join(self.byte_encoder[b] for b in tok.encode("utf-8"))
            ids.extend(self.encoder[s] for s in self.bpe(tok).split(" "))
        return ids

    def tokenize(self, texts, context_length: int = 77) -> torch.Tensor:
        if isinstance(texts, str):
            texts = [texts]
        out = torch.zeros(len(texts), context_length, dtype=torch.int64)
        for r, t in enumerate(texts):
            ids = [self.sot] + self.encode(t) + [self.eot]
            if len(ids) > context_length:
                ids = ids[:context_length]
                ids[-1] = self.eot
            out[r, :len(ids)] = torch.tensor(ids, dtype=torch.int64)
        return out
