"""Writes tests/golden/bpe_train.json from the installed tiktoken package (0.12.0): `tiktoken._educational.bpe_train(
data, vocab_size, pat_str, visualise=None)` on small corpora cut from the tools/corpus generators, for the three
patterns, and on crafted texts (letter and whitespace runs, CRLF, contractions, digits, emoji, combining marks, empty
text, vocab_size = 256, a target past the last possible merge).  Per case: the pattern, the text, the vocab size and
either the ranks after the 256 single bytes, in dict order, as [hex bytes, rank], or the exception the reference raised.

Every text is also split by the C oracle (oracle/bpe_oracle.c), whose Unicode tables are the engine's: the generator
fails if Python's `regex` splits any fixture text differently.

    python tests/golden/make_train_golden.py"""
import json
import os
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.join(os.path.dirname(HERE), "..")]

import regex  # noqa: E402
from tiktoken._educational import bpe_train  # noqa: E402

from oracle import Oracle  # noqa: E402
from oracle.oracle import CL100K_PAT, O200K_PAT, R50K_PAT  # noqa: E402
from tools import corpus  # noqa: E402

PATS = {"r50k": R50K_PAT, "cl100k": CL100K_PAT, "o200k": O200K_PAT}


def corpus_text(kind: int, seed: int, nbytes: int) -> str:
    b = corpus.generate(kind, seed, nbytes).tobytes()
    return b.decode("utf-8", "ignore")          # a cut multi-byte character at the end goes


def cases():
    yield "english_r50k", "r50k", corpus_text(corpus.ENGLISH, 11, 12000), 256 + 300
    yield "code_r50k", "r50k", corpus_text(corpus.CODE, 12, 6000), 256 + 200
    yield "english_cl100k", "cl100k", corpus_text(corpus.ENGLISH, 13, 20000), 256 + 300
    yield "mixed_cl100k", "cl100k", corpus_text(corpus.MIXED, 14, 8000), 256 + 250
    yield "mixed_o200k", "o200k", corpus_text(corpus.MIXED, 15, 16000), 256 + 300
    yield "english_o200k", "o200k", corpus_text(corpus.ENGLISH, 16, 5000), 256 + 150
    runs = "a" * 37 + " " + "a" * 64 + " b" + "aaa" + " " + "ab" * 9 + " aaaa aaaaa " + "z" * 129 + "\n"
    for p in PATS:
        yield f"letter_runs_{p}", p, runs, 256 + 14
        yield f"whitespace_crlf_{p}", p, ("x \r\n\r\n   \t\t  y\n\n\n  z \r\n" * 5) + " " * 40 + "\r\n" * 9 + "end  ", 256 + 16
        yield f"contractions_{p}", p, ("I'm don't WE'LL they're it'S 12345 6789 0 3.14159 😀😀 🎉🎉 é Café "
                                      "naïve ΑΒΓ αβγ 日本語 日本 ÅB x€ ") * 3, 256 + 40
        yield f"empty_256_{p}", p, "", 256
        yield f"empty_{p}", p, "", 257
    yield "vocab_256", "cl100k", corpus_text(corpus.ENGLISH, 17, 3000), 256
    yield "beyond_last_merge", "cl100k", "abab ab ab", 300
    yield "beyond_last_merge_o200k", "o200k", "hello hello world", 270


def main():
    out = []
    for name, p, text, vocab in cases():
        pat = PATS[p]
        pieces = [w.encode("utf-8") for w in regex.findall(pat, text)]
        assert Oracle({}, {}, pat).split(text) == pieces, f"{name}: regex and the C oracle split differently"
        case = {"name": name, "pat": p, "text": text, "vocab_size": vocab}
        try:
            ranks = bpe_train(text, vocab, pat, visualise=None)
            items = list(ranks.items())
            assert items[:256] == [(bytes([i]), i) for i in range(256)]
            case["ranks"] = [[k.hex(), v] for k, v in items[256:]]
        except ValueError:
            case["error"] = "ValueError"
        out.append(case)
        print(name, len(text), case.get("error") or len(case["ranks"]), flush=True)
    with open(os.path.join(HERE, "bpe_train.json"), "w") as f:
        json.dump({"generator": "tiktoken._educational.bpe_train (tiktoken 0.12.0), visualise=None", "cases": out}, f,
                  ensure_ascii=False, indent=0)


if __name__ == "__main__":
    main()
