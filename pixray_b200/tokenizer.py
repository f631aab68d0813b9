"""Byte-level BPE tokenizer of the CLIP family: the token ids `clip.tokenize` (openai-CLIP) and SLIP's
`SimpleTokenizer.__call__` (SLIP/tokenizer.py) give, for the engine's text towers.

Text is cleaned the way both do it: `ftfy.fix_text` when the `ftfy` package is importable (without it the text is used
as given, so mojibake that ftfy would repair is tokenised as it stands), `html.unescape` twice, runs of whitespace
collapsed to one space, stripped, lower-cased.  It is then split into words (contractions, letter runs, single digits,
runs of other non-space characters), each word's UTF-8 bytes are mapped to printable characters, and the vocabulary's
merges are applied in rank order with `</w>` marking the end of the word.  Every sequence is
[<|startoftext|>, tokens..., <|endoftext|>] zero-padded to the context length (77).

The two families differ only on sequences longer than the context:
- "clip" (clip.tokenize, truncate=False) raises RuntimeError naming the input;
- "slip" (SimpleTokenizer.__call__) keeps the first 77 ids, so the end-of-text token can be cut off.  The text tower
  then reads the row of the largest remaining id (encode_text's `text.argmax(dim=-1)`).

The vocabulary is the reference's `bpe_simple_vocab_16e6.txt.gz` (find_vocab says where it is looked for); only its
header line and first 49152 - 256 - 2 merges are read, so a copy cut to those lines works the same.
"""
import functools
import gzip
import html
import os

import numpy as np
import regex

SOT, EOT = 49406, 49407
CONTEXT = 77
VOCAB_NAME = "bpe_simple_vocab_16e6.txt.gz"
N_MERGES = 49152 - 256 - 2  # the merges the 49408-entry vocabulary uses (the file lists more)

_WORD = regex.compile(r"""<\|startoftext\|>|<\|endoftext\|>|'s|'t|'re|'ve|'m|'ll|'d|\p{L}+|\p{N}|[^\s\p{L}\p{N}]+""",
                      regex.IGNORECASE)
_SPACES = regex.compile(r"\s+")


def byte_alphabet():
    """One printable character per byte value: the printable Latin-1 bytes stand for themselves, the other 68 bytes take
    the code points from 256 upwards, in byte order.  Returned as a list indexed by byte; its order is also the order of
    the vocabulary's first 256 entries."""
    keep = set(range(ord("!"), ord("~") + 1)) | set(range(ord("¡"), ord("¬") + 1)) | set(range(ord("®"), ord("ÿ") + 1))
    chars, extra = {}, 0
    for b in range(256):
        if b in keep:
            chars[b] = chr(b)
        else:
            chars[b] = chr(256 + extra)
            extra += 1
    order = sorted(keep) + [b for b in range(256) if b not in keep]
    return [chars[b] for b in range(256)], [chars[b] for b in order]


def clean(text):
    try:
        import ftfy
        text = ftfy.fix_text(text)
    except ImportError:
        pass
    text = html.unescape(html.unescape(text)).strip()
    return _SPACES.sub(" ", text).strip().lower()


def find_vocab(path=None):
    """The vocabulary file: `path` (the b200_bpe_vocab setting) when given; otherwise the copy inside the installed
    `clip` package, then $PIXRAY_ROOT/SLIP/."""
    if path is not None:
        if not os.path.exists(path):
            raise FileNotFoundError(f"b200_bpe_vocab: {path} does not exist")
        return str(path)
    cands = []
    try:
        import clip
        cands.append(os.path.join(os.path.dirname(clip.__file__), VOCAB_NAME))
    except Exception:
        pass
    if os.environ.get("PIXRAY_ROOT"):
        cands.append(os.path.join(os.environ["PIXRAY_ROOT"], "SLIP", VOCAB_NAME))
    for c in cands:
        if os.path.exists(c):
            return c
    raise FileNotFoundError(f"the text towers need CLIP's BPE vocabulary {VOCAB_NAME}: set b200_bpe_vocab to its path "
                            f"(tried {cands or 'no candidate: clip is not installed and PIXRAY_ROOT is unset'})")


class Tokenizer:
    def __init__(self, vocab_path):
        with gzip.open(vocab_path, "rt", encoding="utf-8") as f:
            lines = f.read().split("\n")
        merges = [tuple(line.split()) for line in lines[1:N_MERGES + 1] if line]
        if len(merges) != N_MERGES or any(len(m) != 2 for m in merges):
            raise ValueError(f"{vocab_path}: not a CLIP BPE vocabulary (needs {N_MERGES} merge lines after the header)")
        self.byte_char, alphabet = byte_alphabet()
        vocab = alphabet + [c + "</w>" for c in alphabet] + ["".join(m) for m in merges]
        vocab += ["<|startoftext|>", "<|endoftext|>"]
        self.ids = {tok: i for i, tok in enumerate(vocab)}
        self.rank = {m: i for i, m in enumerate(merges)}

    @functools.lru_cache(maxsize=65536)
    def _bpe(self, word):
        """The symbols of one pre-tokenised word (already in the byte alphabet) after all applicable merges."""
        if word in ("<|startoftext|>", "<|endoftext|>"):
            return (word,)
        syms = list(word[:-1]) + [word[-1] + "</w>"]
        while len(syms) > 1:
            best = min(((self.rank.get(p, len(self.rank)), p) for p in zip(syms, syms[1:])))
            if best[0] == len(self.rank):
                break
            a, b = best[1]
            out, i = [], 0
            while i < len(syms):  # merge every occurrence of the pair, left to right
                if i + 1 < len(syms) and syms[i] == a and syms[i + 1] == b:
                    out.append(a + b)
                    i += 2
                else:
                    out.append(syms[i])
                    i += 1
            syms = out
        return tuple(syms)

    def encode(self, text):
        ids = []
        for word in _WORD.findall(clean(text)):
            mapped = "".join(self.byte_char[b] for b in word.encode("utf-8"))
            ids.extend(self.ids[s] for s in self._bpe(mapped))
        return ids

    def __call__(self, texts, family="clip", context_length=CONTEXT):
        """[n, context_length] int32 ids of a str or a list of str, with the family's over-length rule."""
        if family not in ("clip", "slip"):
            raise ValueError(f"tokenizer family must be 'clip' or 'slip', not {family!r}")
        if isinstance(texts, str):
            texts = [texts]
        out = np.zeros((len(texts), context_length), dtype=np.int32)
        for i, t in enumerate(texts):
            ids = [SOT] + self.encode(t) + [EOT]
            if len(ids) > context_length:
                if family == "clip":
                    raise RuntimeError(f"Input {t} is too long for context length {context_length}")
                ids = ids[:context_length]
            out[i, :len(ids)] = ids
        return out


@functools.lru_cache(maxsize=4)
def get(vocab_path):
    return Tokenizer(vocab_path)
