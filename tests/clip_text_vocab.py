"""A small openai-format BPE vocabulary for the CLIP text tests: merges trained on the given texts with the
tokenizer's own pre-tokenizer, written as ``bpe_simple_vocab_16e6.txt.gz`` is (gzip text, a version line, one
``a b`` merge per line), and the same vocabulary as HF ``CLIPTokenizer``'s ``vocab.json`` / ``merges.txt``."""
from __future__ import annotations

import collections
import gzip
import json
import os
from typing import List, Sequence

from video_features_b200 import clip_tokenizer as ct


def train_merges(texts: Sequence[str], n_merges: int) -> List[tuple]:
    """Greedy BPE over the pre-tokens of ``texts``: the most frequent adjacent pair first (ties: the smaller pair),
    skipping pairs whose concatenation is already a symbol so that every vocabulary entry is unique."""
    enc = ct.bytes_to_unicode()
    words = collections.Counter()
    for t in texts:
        for tok in ct._PAT.findall(ct.clean(t)):
            b = "".join(enc[x] for x in tok.encode("utf-8"))
            words[tuple(b[:-1]) + (b[-1] + "</w>",)] += 1
    symbols = set(enc.values()) | {v + "</w>" for v in enc.values()}
    merges = []
    while len(merges) < n_merges:
        pairs = collections.Counter()
        for w, f in words.items():
            for p in zip(w[:-1], w[1:]):
                if p[0] + p[1] not in symbols:
                    pairs[p] += f
        if not pairs:
            break
        best = min(pairs, key=lambda p: (-pairs[p], p))
        merges.append(best)
        symbols.add(best[0] + best[1])
        merged = collections.Counter()
        for w, f in words.items():
            out, i = [], 0
            while i < len(w):
                if i < len(w) - 1 and (w[i], w[i + 1]) == best:
                    out.append(w[i] + w[i + 1])
                    i += 2
                else:
                    out.append(w[i])
                    i += 1
            merged[tuple(out)] += f
        words = merged
    return merges


def write_bpe(path: str, texts: Sequence[str], n_merges: int = 400) -> str:
    merges = train_merges(texts, n_merges)
    with gzip.open(path, "wb") as f:
        f.write(("#version: 0.2\n" + "\n".join(f"{a} {b}" for a, b in merges)).encode("utf-8"))
    return path


def write_hf_files(bpe_path: str, out_dir: str):
    """vocab.json / merges.txt of the same vocabulary -> (vocab_file, merges_file)."""
    tok = ct.SimpleTokenizer(bpe_path)
    vocab_file, merges_file = os.path.join(out_dir, "vocab.json"), os.path.join(out_dir, "merges.txt")
    with open(vocab_file, "w", encoding="utf-8") as f:
        json.dump(tok.encoder, f, ensure_ascii=False)
    merges = sorted(tok.bpe_ranks, key=tok.bpe_ranks.get)
    with open(merges_file, "w", encoding="utf-8") as f:
        f.write("#version: 0.2\n" + "".join(f"{a} {b}\n" for a, b in merges))
    return vocab_file, merges_file


def standard_vocab(path: str) -> str:
    """The vocabulary the CLIP text tests share: merges trained on the 400 default prompts and a few sentences."""
    texts = ct.default_prompts() + ["a video of people dancing at a wedding", "the cat's toy isn't here",
                                    "we'll see 12 dogs running"]
    return write_bpe(path, texts, 400)
