"""Regenerate tests/golden/unigram_golden.model: a small SentencePiece Unigram model (nmt_nfkc normalisation, the rule
XLM-R's sentencepiece.bpe.model was trained with) for the XLM-R tokenizer tests.

The corpus is generated here from a fixed seed: words over Latin (with accents), Cyrillic, Greek, CJK and kana letters,
digits, and lines that carry NFKC compatibility characters, so that the model has multi-character pieces in several
scripts and the charsmap has rules to apply.  Characters outside the corpus stay unknown, which the tests rely on.

    python tests/golden/make_unigram_golden.py
"""
from __future__ import annotations

import io
import random
from pathlib import Path

import sentencepiece as spm

OUT = Path(__file__).resolve().parent / "unigram_golden.model"

ALPHABETS = [
    "abcdefghijklmnopqrstuvwxyz",
    "aeiouéèêàçñüöäß",
    "абвгдежзийклмнопрстуфхцчшщыэюя",
    "αβγδεζηθικλμνξοπρστυφχψω",
    "東京大学日本語中文字学生先生水火山川",
    "あいうえおかきくけこさしすせそたちつてと",
    "アイウエオカキクケコタチツテトワン",
    "0123456789",
]
COMPAT = ["ﬁne", "Ａｂｃ", "①②③", "ｶﾀｶﾅ", "㎞", "Ⅻ", "ﬂow"]


def corpus(seed: int = 20261016, lines: int = 6000):
    g = random.Random(seed)
    for _ in range(lines):
        words = []
        for _ in range(g.randint(3, 14)):
            alpha = g.choice(ALPHABETS)
            words.append("".join(g.choice(alpha) for _ in range(g.randint(1, 7))))
        if g.random() < 0.3:
            words.append(g.choice(COMPAT))
        if g.random() < 0.3:
            words[0] = words[0].capitalize()
        yield " ".join(words)


def main() -> None:
    buf = io.BytesIO()
    spm.SentencePieceTrainer.train(sentence_iterator=corpus(), model_writer=buf, model_type="unigram",
                                   vocab_size=1200, character_coverage=1.0, normalization_rule_name="nmt_nfkc",
                                   num_threads=1, minloglevel=2)
    OUT.write_bytes(buf.getvalue())
    print(f"wrote {OUT} ({len(buf.getvalue())} bytes)")


if __name__ == "__main__":
    main()
