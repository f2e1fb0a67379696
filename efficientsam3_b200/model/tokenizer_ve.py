"""CLIP byte-level BPE tokenizer, restated for the text encoders (the reference's `sam3/sam3/model/tokenizer_ve.py`
`SimpleTokenizer`): same constructor, same `__call__(texts, context_length)` contract, same ids.

  ids = [<start_of_text>] + bpe(clean(text)) + [<end_of_text>], zero padded to context_length; a longer sequence is
  cut to context_length and its last id replaced by <end_of_text> (tokenizer_ve.py:243-253).
  clean = "lower": ftfy.fix_text, html.unescape twice, strip, collapse whitespace, lower-case (tokenizer_ve.py:68-87).

The vocabulary is the caller's `bpe_path` (the gzip'd CLIP merge list, bpe_simple_vocab_16e6.txt.gz); this package ships
none.  `ftfy` is used when it is importable and skipped otherwise: it is an unpinned boundary (as timm is for the image
students) -- it only rewrites mojibake / unusual unicode, and plain captions tokenise identically without it.
"""
from __future__ import annotations

import gzip
import html
import os
from typing import List, Optional, Union

import torch

DEFAULT_CONTEXT_LENGTH = 77
_N_MERGES = 49152 - 256 - 2      # merges used by CLIP: vocab = 256 bytes x {plain, </w>} + merges + 2 specials = 49408


def _byte_alphabet():
    """byte value -> printable unicode character, in vocabulary order: the 188 bytes that are printable latin-1 map to
    themselves (listed first), the other 68 map to U+0100.. in byte order."""
    keep = [b for b in range(256) if 0x21 <= b <= 0x7E or 0xA1 <= b <= 0xAC or 0xAE <= b <= 0xFF]
    rest = [b for b in range(256) if b not in set(keep)]
    table = {b: chr(b) for b in keep}
    table.update({b: chr(256 + i) for i, b in enumerate(rest)})
    return table, keep + rest


def _fix_text(s: str) -> str:
    try:
        import ftfy
    except ImportError:
        return s
    return ftfy.fix_text(s)


class SimpleTokenizer:
    def __init__(self, bpe_path: Union[str, os.PathLike], additional_special_tokens: Optional[List[str]] = None,
                 context_length: Optional[int] = DEFAULT_CONTEXT_LENGTH, clean: str = "lower"):
        import regex
        if clean != "lower":
            raise NotImplementedError(f"clean={clean!r}: the text encoders tokenise with clean='lower'")
        with open(bpe_path, "rb") as fh:
            lines = gzip.decompress(fh.read()).decode("utf-8").split("\n")
        merges = [tuple(line.split()) for line in lines[1:1 + _N_MERGES]]
        self.byte_encoder, order = _byte_alphabet()
        self.byte_decoder = {v: k for k, v in self.byte_encoder.items()}
        symbols = [self.byte_encoder[b] for b in order]
        vocab = symbols + [s + "</w>" for s in symbols] + ["".join(m) for m in merges]
        self.special_tokens = ["<start_of_text>", "<end_of_text>"] + list(additional_special_tokens or [])
        vocab += self.special_tokens
        self.encoder = {tok: i for i, tok in enumerate(vocab)}
        self.decoder = {i: tok for tok, i in self.encoder.items()}
        self.bpe_ranks = {m: i for i, m in enumerate(merges)}
        self.vocab_size = len(self.encoder)
        self.all_special_ids = [self.encoder[t] for t in self.special_tokens]
        self.sot_token_id, self.eot_token_id = self.all_special_ids[0], self.all_special_ids[1]
        self.context_length = context_length
        self._ws = regex.compile(r"\s+")
        # special tokens, English contractions, letter runs, single digits, runs of other non-space characters
        self._pat = regex.compile("|".join(self.special_tokens) + r"""|'s|'t|'re|'ve|'m|'ll|'d|[\p{L}]+|[\p{N}]|[^\s\p{L}\p{N}]+""",
                                  regex.IGNORECASE)
        self._cache = {}

    def _clean(self, text: str) -> str:
        text = html.unescape(html.unescape(_fix_text(text))).strip()
        return self._ws.sub(" ", text).strip().lower()

    def bpe(self, piece: str) -> List[str]:
        """Greedy BPE of one pre-token: merge the lowest-ranked adjacent pair (all its occurrences, left to right) until no
        ranked pair is left.  The last symbol carries the end-of-word marker."""
        hit = self._cache.get(piece)
        if hit is not None:
            return hit
        syms = list(piece[:-1]) + [piece[-1] + "</w>"]
        while len(syms) > 1:
            ranked = [(self.bpe_ranks[p], p) for p in zip(syms, syms[1:]) if p in self.bpe_ranks]
            if not ranked:
                break
            a, b = min(ranked)[1]
            merged, i = [], 0
            while i < len(syms):
                if i + 1 < len(syms) and syms[i] == a and syms[i + 1] == b:
                    merged.append(a + b)
                    i += 2
                else:
                    merged.append(syms[i])
                    i += 1
            syms = merged
        self._cache[piece] = syms
        return syms

    def encode(self, text: str) -> List[int]:
        ids = []
        for piece in self._pat.findall(self._clean(text)):
            if piece in self.special_tokens:
                ids.append(self.encoder[piece])
                continue
            mapped = "".join(self.byte_encoder[b] for b in piece.encode("utf-8"))
            ids.extend(self.encoder[s] for s in self.bpe(mapped))
        return ids

    def decode(self, tokens) -> str:
        text = "".join(self.decoder[int(t)] for t in tokens)
        return bytearray(self.byte_decoder[c] for c in text).decode("utf-8", errors="replace").replace("</w>", " ")

    def __call__(self, texts: Union[str, List[str]], context_length: Optional[int] = None) -> torch.LongTensor:
        """-> int64 [len(texts), context_length] on the CPU."""
        if isinstance(texts, str):
            texts = [texts]
        n = context_length or self.context_length
        if not n:
            raise ValueError("SimpleTokenizer: no context length")
        out = torch.zeros(len(texts), n, dtype=torch.long)
        for i, t in enumerate(texts):
            ids = [self.sot_token_id] + self.encode(t) + [self.eot_token_id]
            if len(ids) > n:
                ids = ids[:n]
                ids[-1] = self.eot_token_id
            out[i, :len(ids)] = torch.tensor(ids, dtype=torch.long)
        return out
