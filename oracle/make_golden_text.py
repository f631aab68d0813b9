"""Freeze the reference tokenizer's ids as tests/golden/text_tokens.json, and the part of its vocabulary they use next to them.

Runs the reference's own SLIP/tokenizer.py (the same SimpleTokenizer clip.tokenize wraps) with `ftfy` registered
through oracle/shim.py as the identity (ftfy is not installed in the authoring container; pixray_b200.tokenizer also
skips it when it is absent).  For each string the file keeps SimpleTokenizer.__call__'s 77 ids, i.e. SLIP's truncating
rule, and whether the sequence overflows the context, which is where clip.tokenize raises instead.

The vocabulary fixture, tests/golden/bpe_vocab_used_merges.txt.gz, is the reference's bpe_simple_vocab_16e6.txt.gz cut
to what both tokenizers read of it: the header line and the first 49152 - 256 - 2 merges (the file lists 262145; the
rest never reach the 49408-entry vocabulary).  It gives the same ids as the whole file, at a sixth of its size.

    python -m oracle.make_golden_text
"""
import gzip
import json
import os
import sys

from oracle import shim

STRINGS = [
    # pixray-style prompts, weights and stops removed
    "a cat", "A painting of a lighthouse by the sea", "Wow, that looks cool!", "an apple in the style of Cézanne",
    "pixel art of a robot", "a cyberpunk city at night #pixelart", "Beksinski dreamscape, trending on artstation",
    "a watercolor of a fox; muted colors", "a cat and a dog", "the ultimate owl",
    # punctuation, digits, contractions, apostrophes
    "it's 3:14 am, isn't it?", "we'll see what they'd do; I'm sure you've heard", "rock 'n' roll",
    "1984 vs 2001: a space odyssey", "3.14159265358979", "hello...world!!!", "(x+y)^2 = x^2 + 2xy + y^2",
    "email me @ foo_bar-baz", "don't STOP believin'", "''quoted'' \"double\" `back`",
    # HTML entities (unescaped twice)
    "fish &amp; chips", "&lt;b&gt;bold&lt;/b&gt;", "caf&eacute; au lait", "&amp;amp; twice", "&#39;single&#39;",
    # repeated whitespace
    "  lots   of\tspaces\n\nand lines  ", "a non-breaking em space",
    # non-ASCII letters ftfy leaves alone
    "Ελληνικά γράμματα", "日本語のテキスト", "naïve façade", "Straße über München", "Привет, мир",
    "emoji 🐱 cat 🚀", "ﬁne ligature", "اللغة العربية", "한국어 문장",
    "<|startoftext|> literal special tokens <|endoftext|>",
    "", "x",
    # past 77 tokens
    "a very long prompt " + " ".join(f"word{i}" for i in range(80)),
]


def main():
    shim._mod("ftfy", fix_text=lambda t: t)
    sys.path.insert(0, os.path.join(shim.REFERENCE, "SLIP"))
    import tokenizer as ref_tok  # SLIP/tokenizer.py

    tok = ref_tok.SimpleTokenizer()
    out = {"strings": STRINGS, "ids": [], "overflows": []}
    for s in STRINGS:
        out["ids"].append([int(v) for v in tok([s, s])[0].tolist()])  # a list keeps __call__'s 2-D return
        out["overflows"].append(len(tok.encode(s)) + 2 > 77)
    assert any(out["overflows"]) and not all(out["overflows"])
    here = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    with open(os.path.join(here, "tests", "golden", "text_tokens.json"), "w") as f:
        json.dump(out, f, ensure_ascii=False, indent=0)
    lines = gzip.open(ref_tok.default_bpe(), "rt", encoding="utf-8").read().split("\n")
    used = "\n".join(lines[:1 + 49152 - 256 - 2]) + "\n"
    with open(os.path.join(here, "tests", "golden", "bpe_vocab_used_merges.txt.gz"), "wb") as f:
        f.write(gzip.compress(used.encode("utf-8"), compresslevel=9, mtime=0))


if __name__ == "__main__":
    main()
