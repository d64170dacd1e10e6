"""openai/CLIP's byte-level BPE tokenizer (``clip/simple_tokenizer.py`` ``SimpleTokenizer`` and
``clip.tokenize(texts, context_length=77)``), restated for ``--show_pred`` on the CLIP feature types.

One difference: openai runs ``ftfy.fix_text`` before the HTML unescape.  ``ftfy`` is not a dependency here, so it is
not applied; it only repairs mis-decoded Unicode (mojibake such as ``"Ã©"`` for ``"é"``), which prompts typed as text
do not carry.

The vocabulary (``bpe_simple_vocab_16e6.txt.gz``) ships with the ``clip`` package, not with the checkpoints.  It is
looked up as the checkpoints are (``find_bpe``): ``$VF_CLIP_BPE``, ``extract/checkpoints/``, ``~/.cache/clip/``.
"""
from __future__ import annotations

import gzip
import html
import os
import pathlib
from functools import lru_cache
from typing import Dict, List, Optional, Sequence, Tuple

import numpy as np
import regex as re

BPE_NAME = "bpe_simple_vocab_16e6.txt.gz"
CONTEXT_LENGTH = 77
SOT, EOT = "<|startoftext|>", "<|endoftext|>"
# openai's pre-tokenizer: special tokens, English contractions, letter runs, single digits, punctuation runs
_PAT = re.compile(r"""<\|startoftext\|>|<\|endoftext\|>|'s|'t|'re|'ve|'m|'ll|'d|[\p{L}]+|[\p{N}]|[^\s\p{L}\p{N}]+""",
                  re.IGNORECASE)


@lru_cache()
def bytes_to_unicode() -> Dict[int, str]:
    """Every byte -> a printable character: the printable Latin-1 bytes map to themselves, the rest to 256 + n."""
    bs = list(range(ord("!"), ord("~") + 1)) + list(range(ord("¡"), ord("¬") + 1)) + list(range(ord("®"), ord("ÿ") + 1))
    cs = bs[:]
    n = 0
    for b in range(256):
        if b not in bs:
            bs.append(b)
            cs.append(256 + n)
            n += 1
    return dict(zip(bs, [chr(c) for c in cs]))


def _pairs(word: Tuple[str, ...]):
    return {(a, b) for a, b in zip(word[:-1], word[1:])}


def clean(text: str) -> str:
    """HTML unescaped twice, whitespace runs collapsed to one space, stripped, lower-cased."""
    text = html.unescape(html.unescape(text)).strip()
    return re.sub(r"\s+", " ", text).strip().lower()


def bpe_candidates() -> List[str]:
    return [c for c in (os.environ.get("VF_CLIP_BPE"),
                        os.path.join(pathlib.Path(__file__).parent, "extract", "checkpoints", BPE_NAME),
                        os.path.expanduser(os.path.join("~/.cache/clip", BPE_NAME))) if c]


def find_bpe() -> str:
    """The first existing vocabulary file of ``bpe_candidates()``; FileNotFoundError naming them all otherwise."""
    cands = bpe_candidates()
    for p in cands:
        if os.path.exists(p):
            return p
    raise FileNotFoundError(f"--show_pred on CLIP needs the BPE vocabulary {BPE_NAME} (it ships with openai's clip "
                            f"package); looked at {cands} -- set VF_CLIP_BPE")


class SimpleTokenizer:
    """``bpe_path``: an openai-format merges file, gzip text: a version line, then one ``a b`` merge per line."""

    def __init__(self, bpe_path: str):
        self.byte_encoder = bytes_to_unicode()
        merges = gzip.open(bpe_path).read().decode("utf-8").split("\n")
        merges = [tuple(m.split()) for m in merges[1:49152 - 256 - 2 + 1] if m]
        vocab = list(self.byte_encoder.values())
        vocab = vocab + [v + "</w>" for v in vocab]
        vocab += ["".join(m) for m in merges]
        vocab += [SOT, EOT]
        self.encoder = {v: i for i, v in enumerate(vocab)}
        self.bpe_ranks = {m: i for i, m in enumerate(merges)}
        self.cache = {SOT: SOT, EOT: EOT}

    @property
    def vocab_size(self) -> int:
        return len(self.encoder)

    @property
    def sot(self) -> int:
        return self.encoder[SOT]

    @property
    def eot(self) -> int:
        return self.encoder[EOT]

    def bpe(self, token: str) -> str:
        """One pre-token (byte characters) -> its space-separated BPE pieces, the last one ending in ``</w>``."""
        if token in self.cache:
            return self.cache[token]
        word = tuple(token[:-1]) + (token[-1] + "</w>",)
        pairs = _pairs(word)
        if not pairs:
            return token + "</w>"
        while True:
            bigram = min(pairs, key=lambda p: self.bpe_ranks.get(p, float("inf")))
            if bigram not in self.bpe_ranks:
                break
            first, second = bigram
            merged = []
            i = 0
            while i < len(word):
                try:
                    j = word.index(first, i)
                except ValueError:
                    merged.extend(word[i:])
                    break
                merged.extend(word[i:j])
                i = j
                if i < len(word) - 1 and word[i + 1] == second:
                    merged.append(first + second)
                    i += 2
                else:
                    merged.append(word[i])
                    i += 1
            word = tuple(merged)
            if len(word) == 1:
                break
            pairs = _pairs(word)
        out = " ".join(word)
        self.cache[token] = out
        return out

    def encode(self, text: str) -> List[int]:
        ids = []
        for token in _PAT.findall(clean(text)):
            token = "".join(self.byte_encoder[b] for b in token.encode("utf-8"))
            ids.extend(self.encoder[piece] for piece in self.bpe(token).split(" "))
        return ids

    def tokenize(self, texts: Sequence[str], context_length: int = CONTEXT_LENGTH) -> np.ndarray:
        """``clip.tokenize``: (len(texts), context_length) int32 rows SOT + ids + EOT, zero-padded; a text that does
        not fit raises RuntimeError."""
        if isinstance(texts, str):
            texts = [texts]
        out = np.zeros((len(texts), context_length), np.int32)
        for i, t in enumerate(texts):
            ids = [self.sot] + self.encode(t) + [self.eot]
            if len(ids) > context_length:
                raise RuntimeError(f"Input {t} is too long for context length {context_length}")
            out[i, :len(ids)] = ids
        return out


_TOKENIZERS: Dict[str, SimpleTokenizer] = {}


def load(path: Optional[str] = None) -> SimpleTokenizer:
    """The tokenizer of ``path`` (default: ``find_bpe()``), built once per file."""
    path = path or find_bpe()
    if path not in _TOKENIZERS:
        _TOKENIZERS[path] = SimpleTokenizer(path)
    return _TOKENIZERS[path]


def default_prompts() -> List[str]:
    """``a photo of {name}`` over the 400 Kinetics-400 class names (``--pred_texts``' default)."""
    from .utils import class_names
    return [f"a photo of {name}" for name in class_names("kinetics")]
