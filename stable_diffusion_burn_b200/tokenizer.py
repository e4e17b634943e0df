"""CLIP byte-level BPE tokenizer — host-side mirror of the reference's `SimpleTokenizer`
(src/tokenizer.rs:86-203; SURVEY §8f row f1).

Same observable behaviour, including the quirks: text is trimmed, whitespace-collapsed and lower-cased; no
padding or truncation to 77 tokens; merges are lines [1, 48895) of the vocabulary file; the two special tokens
are ids 49406/49407 and pass through BPE untouched. The merge table is the OpenAI CLIP file
`bpe_simple_vocab_16e6.txt`, which the reference opens relative to the working directory (tokenizer.rs:92);
it is a data file of the reference checkout and is NOT vendored here: pass its path, set SDB_BPE_VOCAB, or run
from a directory that contains it.

The reference's only test (tokenizer.rs:205-221) is reproduced in tests/test_tokenizer_cpu.py — the one place
where parity of this repo is pinned by a golden vector of the reference itself.
"""
from __future__ import annotations

import os

import regex

VOCAB_FILE = "bpe_simple_vocab_16e6.txt"
_PATTERN = r"(?i)<\|startoftext\|>|<\|endoftext\|>|'s|'t|'re|'ve|'m|'ll|'d|\p{L}+|\p{N}|[^\s\p{L}\p{N}]+"


def find_vocab(path: str | None = None) -> str:
    cands = [path, os.environ.get("SDB_BPE_VOCAB"), VOCAB_FILE]
    for c in cands:
        if c and os.path.isfile(c):
            return c
    raise FileNotFoundError(f"{VOCAB_FILE} not found (pass a path or set SDB_BPE_VOCAB); it ships with the reference checkout")


def _byte_unicode_table():
    """bytes -> printable unicode stand-ins (tokenizer.rs:7-28): printable latin-1 bytes map to themselves,
    the remaining 68 bytes to code points 256.."""
    keep = list(range(ord("!"), ord("~") + 1)) + list(range(0xA1, 0xAC + 1)) + list(range(0xAE, 0xFF + 1))
    table = [(b, chr(b)) for b in keep]
    extra = 0
    for b in range(256):
        if b not in keep:
            table.append((b, chr(256 + extra)))
            extra += 1
    return table


class SimpleTokenizer:
    def __init__(self, vocab_path: str | None = None):
        table = _byte_unicode_table()
        self.byte_encoder = dict(table)
        self.byte_decoder = {u: b for b, u in table}
        merges = []
        with open(find_vocab(vocab_path), encoding="utf-8") as f:
            for line in f:
                parts = line.split()
                if len(parts) >= 2:
                    merges.append((parts[0], parts[1]))
        merges = merges[1:49152 - 256 - 2 + 1]  # drops the "#version: 0.2" header pair (tokenizer.rs:93)
        chars = [u for _, u in table]
        vocab = chars + [c + "</w>" for c in chars] + [a + b for a, b in merges] + ["<|startoftext|>", "<|endoftext|>"]
        self.encoder = {tok: i for i, tok in enumerate(vocab)}
        self.decoder = {i: tok for tok, i in self.encoder.items()}
        self.rank = {pair: i for i, pair in enumerate(merges)}
        self.special = {"<|startoftext|>", "<|endoftext|>"}
        self.pat = regex.compile(_PATTERN)

    def bpe(self, token: str) -> str:
        """Merged sub-words of one pre-token, space separated (tokenizer.rs:118-173)."""
        if token in self.special:
            return token
        parts = list(token[:-1]) + [token[-1] + "</w>"] if token else []
        if len(parts) < 2:
            return token + "</w>"
        while len(parts) > 1:
            best, best_rank = None, None
            for pair in zip(parts, parts[1:]):
                r = self.rank.get(pair)
                if r is not None and (best_rank is None or r < best_rank):
                    best, best_rank = pair, r
            if best is None:
                break
            first, second = best
            merged, i = [], 0
            while i < len(parts):
                if i < len(parts) - 1 and parts[i] == first and parts[i + 1] == second:
                    merged.append(first + second)
                    i += 2
                else:
                    merged.append(parts[i])
                    i += 1
            parts = merged
        return " ".join(parts)

    def encode(self, text: str) -> list[int]:
        cleaned = " ".join(text.strip().split()).lower()
        ids = []
        for m in self.pat.finditer(cleaned):
            tok = "".join(self.byte_encoder[b] for b in m.group(0).encode("utf-8"))
            ids.extend(self.encoder[t] for t in self.bpe(tok).split(" "))
        return ids

    def decode(self, tokens) -> str:
        text = "".join(self.decoder[int(t)] for t in tokens)
        raw = bytes(self.byte_decoder[c] for c in text)
        return raw.decode("utf-8", errors="replace").replace("</w>", " ")
