"""open_clip's byte-level BPE tokenizer (``bpe_simple_vocab_16e6.txt.gz``), the tokenizer of CLIPScore and HPSv2.

Text is cleaned (ftfy when installed, HTML entities unescaped twice, whitespace runs collapsed), lower-cased and split
into words, numbers and punctuation runs.  Each piece is mapped byte by byte onto printable characters, and adjacent
symbol pairs are merged in the order of the merges file until no listed pair is left; the last symbol of a word carries
``</w>``.  A prompt becomes ``<start_of_text> ... <end_of_text>`` in a zero-padded row of ``context_length`` ids; a
longer prompt is cut and its last kept id replaced by ``<end_of_text>``.
"""
import gzip
import html
from functools import lru_cache

import regex
import torch

from ...prompters.wan_prompter import _fix_text

SOT, EOT = "<start_of_text>", "<end_of_text>"
N_MERGES = 49152 - 256 - 2      # merges the vocabulary uses: 49408 ids = 2 x 256 bytes + merges + 2 specials


@lru_cache()
def byte_symbols():
    """byte value -> the printable character that stands for it: printable Latin-1 bytes map to themselves, the other 68
    to U+0100 upwards in byte order."""
    keep = [*range(ord("!"), ord("~") + 1), *range(ord("¡"), ord("¬") + 1), *range(ord("®"), ord("ÿ") + 1)]
    rest = [b for b in range(256) if b not in keep]
    # insertion order is the vocabulary's order: the printable bytes first, then the remapped ones
    return {**{b: chr(b) for b in keep}, **{b: chr(256 + n) for n, b in enumerate(rest)}}


def clean(text):
    text = html.unescape(html.unescape(_fix_text(text))).strip()
    return regex.sub(r"\s+", " ", text).strip()


class SimpleTokenizer:
    def __init__(self, bpe_path):
        with gzip.open(bpe_path) as f:
            lines = f.read().decode("utf-8").split("\n")
        merges = [tuple(line.split()) for line in lines[1:N_MERGES + 1]]
        self.byte_map = byte_symbols()
        symbols = list(self.byte_map.values())
        vocab = symbols + [s + "</w>" for s in symbols] + ["".join(m) for m in merges] + [SOT, EOT]
        self.encoder = {s: i for i, s in enumerate(vocab)}
        self.ranks = {m: i for i, m in enumerate(merges)}
        self.sot, self.eot = self.encoder[SOT], self.encoder[EOT]
        self.vocab_size = len(vocab)
        self._cache = {}
        self._split = regex.compile(rf"{SOT}|{EOT}|'s|'t|'re|'ve|'m|'ll|'d|[\p{{L}}]+|[\p{{N}}]|[^\s\p{{L}}\p{{N}}]+",
                                    regex.IGNORECASE)

    def bpe(self, piece):
        """the merged symbols of one pre-split piece (already mapped to byte symbols)"""
        if piece in (SOT, EOT):
            return [piece]
        if piece in self._cache:
            return self._cache[piece]
        word = list(piece[:-1]) + [piece[-1] + "</w>"]
        while len(word) > 1:
            pairs = {(a, b) for a, b in zip(word, word[1:])}
            best = min(pairs, key=lambda p: self.ranks.get(p, float("inf")))
            if best not in self.ranks:
                break
            merged, i = [], 0
            while i < len(word):
                if i + 1 < len(word) and (word[i], word[i + 1]) == best:
                    merged.append(word[i] + word[i + 1])
                    i += 2
                else:
                    merged.append(word[i])
                    i += 1
            word = merged
        self._cache[piece] = word
        return word

    def encode(self, text):
        ids = []
        for piece in self._split.findall(clean(text).lower()):
            mapped = "".join(self.byte_map[b] for b in piece.encode("utf-8"))
            ids.extend(self.encoder[s] for s in self.bpe(mapped))
        return ids

    def __call__(self, texts, context_length=77):
        """int64 [len(texts), context_length] token ids (a single string counts as a list of one)."""
        texts = [texts] if isinstance(texts, str) else list(texts)
        out = torch.zeros(len(texts), context_length, dtype=torch.long)
        for i, text in enumerate(texts):
            ids = [self.sot] + self.encode(text) + [self.eot]
            if len(ids) > context_length:
                ids = ids[:context_length]
                ids[-1] = self.eot
            out[i, :len(ids)] = torch.tensor(ids, dtype=torch.long)
        return out
