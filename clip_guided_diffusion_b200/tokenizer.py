"""CLIP's byte-level BPE tokenizer, written from the published algorithm (Radford et al. 2021; GPT-2's byte-level BPE, Radford et al.
2019), with ``clip.tokenize``'s contract.

- The vocabulary is built from the merges file ``bpe_simple_vocab_16e6.txt.gz`` (a version line, then one merge "a b" per line):
  the 256 byte symbols in ``bytes_to_unicode``'s order, the same 256 with ``</w>`` (end of word; ``a</w>`` is id 320), the first 48 894 merges in rank order, ``<|startoftext|>`` and
  ``<|endoftext|>`` -- 49 408 ids, SOT = 49406 and EOT = 49407 with the published file.
- Text is cleaned like CLIP's: ``ftfy.fix_text`` when ``ftfy`` imports (it only repairs mojibake), ``html.unescape`` twice, runs of
  whitespace collapsed to one blank, stripped, lowercased.
- The pre-tokeniser splits words, single digits, punctuation runs and the contractions 's 't 're 've 'm 'll 'd; it needs the
  ``regex`` module for the Unicode classes ``\\p{L}`` / ``\\p{N}``.
- Nothing is downloaded: ``find_vocab`` looks for the file in ``bpe_path``, then ``checkpoints_dir/clip/``, then ``CACHE_PATH/clip/``.
"""
from __future__ import annotations

import functools
import gzip
import html
import os
import re

import torch as th

VOCAB_FILE = "bpe_simple_vocab_16e6.txt.gz"
N_MERGES = 49152 - 256 - 2  # merges used by CLIP: 48 894
SOT, EOT = "<|startoftext|>", "<|endoftext|>"


def bytes_to_unicode() -> dict:
    """byte -> printable unicode character: the 188 printable Latin-1 bytes map to themselves, the other 68 to chr(256 + k) in byte
    order.  The dict's order is the vocabulary's: the printable bytes first (``!`` is id 0, ``a`` id 64), then the others (chr(256)
    is id 188, the blank's ``Ġ`` id 220)."""
    keep = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    table = {b: chr(b) for b in keep}
    for k, b in enumerate(b for b in range(256) if b not in table):
        table[b] = chr(256 + k)
    return table


def _regex():
    try:
        import regex
    except ImportError as e:
        raise RuntimeError("the CLIP tokenizer needs the `regex` module (Unicode letter / number classes in its pre-tokeniser): "
                           "install `regex`, or pass target_embeds= / weights=") from e
    return regex


def clean(text: str) -> str:
    try:
        import ftfy
        text = ftfy.fix_text(text)
    except ImportError:  # only mojibake repair is lost
        pass
    text = html.unescape(html.unescape(text))
    return re.sub(r"\s+", " ", text).strip().lower()


def find_vocab(bpe_path: str = None, checkpoints_dir: str = None) -> str:
    """the merges file: ``bpe_path`` if given, else ``checkpoints_dir/clip/`` then ``CACHE_PATH/clip/``; FileNotFoundError naming them"""
    if bpe_path is not None:
        if not os.path.exists(bpe_path):
            raise FileNotFoundError(f"bpe_path={bpe_path!r} does not exist")
        return bpe_path
    from .cgd import CACHE_PATH
    places = [os.path.join(d, "clip", VOCAB_FILE) for d in (checkpoints_dir, CACHE_PATH) if d is not None]
    for p in places:
        if os.path.exists(p):
            return p
    raise FileNotFoundError(f"CLIP's BPE vocabulary {VOCAB_FILE} was not found in {' or '.join(places)}: place it there (it ships "
                            "with the `clip` package) or pass bpe_path=; nothing is downloaded")


class Tokenizer:
    def __init__(self, bpe_path: str):
        regex = _regex()
        with gzip.open(bpe_path, "rt", encoding="utf-8") as f:
            lines = f.read().split("\n")[1:]
        merges = [tuple(l.split()) for l in lines if l.strip()][:N_MERGES]
        self.byte_encoder = bytes_to_unicode()
        symbols = list(self.byte_encoder.values())
        vocab = symbols + [s + "</w>" for s in symbols] + ["".join(m) for m in merges] + [SOT, EOT]
        self.encoder = {tok: i for i, tok in enumerate(vocab)}
        self.ranks = {m: i for i, m in enumerate(merges)}
        self.sot, self.eot = self.encoder[SOT], self.encoder[EOT]
        self.pattern = regex.compile(r"""<\|startoftext\|>|<\|endoftext\|>|'s|'t|'re|'ve|'m|'ll|'d|[\p{L}]+|[\p{N}]|[^\s\p{L}\p{N}]+""",
                                     regex.IGNORECASE)
        self._cache = {}

    def __len__(self):
        return len(self.encoder)

    def bpe(self, word: str) -> "list[str]":
        """one pre-token (already byte-mapped) -> its BPE symbols; the last symbol carries </w>.  The lowest-ranked adjacent pair is
        merged everywhere it occurs, left to right, until no adjacent pair is a merge."""
        if word in (SOT, EOT):
            return [word]
        if word in self._cache:
            return self._cache[word]
        parts = list(word[:-1]) + [word[-1] + "</w>"]
        while len(parts) > 1:
            pairs = {(a, b) for a, b in zip(parts, parts[1:])}
            best = min(pairs, key=lambda p: self.ranks.get(p, float("inf")))
            if best not in self.ranks:
                break
            merged, i = [], 0
            while i < len(parts):
                if i + 1 < len(parts) and (parts[i], parts[i + 1]) == best:
                    merged.append(parts[i] + parts[i + 1])
                    i += 2
                else:
                    merged.append(parts[i])
                    i += 1
            parts = merged
        self._cache[word] = parts
        return parts

    def encode(self, text: str) -> "list[int]":
        ids = []
        for tok in self.pattern.findall(clean(text)):
            tok = "".join(self.byte_encoder[b] for b in tok.encode("utf-8"))
            ids += [self.encoder[s] for s in self.bpe(tok)]
        return ids

    def tokenize(self, texts, context_length: int = 77, truncate: bool = False) -> th.Tensor:
        """``clip.tokenize``: int32 [len(texts), context_length], SOT + tokens + EOT then zeros.  A sequence longer than
        context_length raises RuntimeError, unless ``truncate``: then it is cut and EOT goes in the last slot."""
        if isinstance(texts, str):
            texts = [texts]
        out = th.zeros(len(texts), context_length, dtype=th.int32)
        for i, text in enumerate(texts):
            ids = [self.sot] + self.encode(text) + [self.eot]
            if len(ids) > context_length:
                if not truncate:
                    raise RuntimeError(f"Input {text} is too long for context length {context_length}")
                ids = ids[:context_length]
                ids[-1] = self.eot
            out[i, :len(ids)] = th.tensor(ids, dtype=th.int32)
        return out


@functools.lru_cache(maxsize=4)
def load_tokenizer(path: str) -> Tokenizer:
    return Tokenizer(path)


def tokenize(texts, context_length: int = 77, truncate: bool = False, *, bpe_path: str = None, checkpoints_dir: str = None) -> th.Tensor:
    """``clip.tokenize(texts, context_length, truncate)`` with the vocabulary file of ``find_vocab(bpe_path, checkpoints_dir)``"""
    return load_tokenizer(find_vocab(bpe_path, checkpoints_dir)).tokenize(texts, context_length, truncate)


__all__ = ["Tokenizer", "bytes_to_unicode", "clean", "find_vocab", "load_tokenizer", "tokenize", "VOCAB_FILE"]
