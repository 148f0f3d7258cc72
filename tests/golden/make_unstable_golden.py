"""Writes tests/golden/encode_with_unstable.json from the installed tiktoken wheel (0.12.0): `encode_with_unstable` of
edge prompts and random prompts cut from the tools/corpus generators, for the four synthetic encodings, some with an
allowed special.  Per case: the text, the allowed specials, the stable tokens, the completion count and the first 16 hex
digits of the sha256 of the sorted completions (json of the list).

    python tests/golden/make_unstable_golden.py"""
import hashlib
import json
import os
import random
import sys

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path[:0] = [os.path.dirname(HERE), os.path.join(os.path.dirname(HERE), "..")]

import tiktoken  # noqa: E402

import vocab_util as vu  # noqa: E402
from tools import corpus  # noqa: E402

ENCODINGS = ["cl100k_base", "r50k_base", "p50k_base", "o200k_base"]
KIND = {"cl100k_base": corpus.ENGLISH, "r50k_base": corpus.ENGLISH, "p50k_base": corpus.CODE, "o200k_base": corpus.MIXED}
WHITE = ["\t", "\n", "\x0b", "\x0c", "\r", " ", "\x85", "\xa0", "\u1680", "\u2000", "\u2005", "\u200a", "\u2028",
         "\u2029", "\u202f", "\u205f", "\u3000"]


def digest(comps) -> str:
    return hashlib.sha256(json.dumps(comps).encode()).hexdigest()[:16]


def edge_prompts(sp):
    return (["", sp, "hello " + sp, sp + " tail", "a" + sp + "b c", "hello fanta", "The quick brown fox jumps",
             "def f():\n    ", ".\n\n", "x.\n\n", "  \n\n", "end \n \t", "naïve é", "日本語", "emoji 😀", "café", "x €",
             "12345", "3.14159", "don't", "we'LL", "it's", "a" * 30, " " * 30, "\n" * 7, "x\r\n", "tab\t", "?!", "  !",
             "(x)", "<|", "https://ex", "Ω", "ÅB", "𝕏"]
            + ["word" + w for w in WHITE] + ["x" + w + w for w in WHITE])


def main():
    out = {}
    for enc in ENCODINGS:
        pat, ranks, special, _ = vu.load_encoding(enc, allow_real=False)
        w = tiktoken.Encoding(f"golden_{enc}", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)
        sp = sorted(special)[0]
        rnd = random.Random(20261016)
        text = corpus.generate(KIND[enc], 4, 200_000).tobytes().decode("utf-8", "ignore")
        prompts = [(t, []) for t in edge_prompts(sp)] + [(t, [sp]) for t in edge_prompts(sp)[:25]]
        for k in range(200):
            a = rnd.randrange(0, len(text) - 100)
            t = text[a:a + rnd.randrange(0, 24)]
            prompts.append((t + sp + t[:7], [sp]) if k % 10 == 0 else (t, []))
        cases = []
        for t, allowed in prompts:
            stable, comps = w.encode_with_unstable(t, allowed_special=set(allowed), disallowed_special=())
            comps = sorted(list(c) for c in comps)
            cases.append([t, allowed, stable, len(comps), digest(comps)])
        out[enc] = cases
    with open(os.path.join(HERE, "encode_with_unstable.json"), "w") as f:
        f.write("{\n")
        for i, enc in enumerate(ENCODINGS):          # one case per line
            f.write(f' "{enc}": [\n')
            f.write(",\n".join("  " + json.dumps(c, ensure_ascii=False, separators=(",", ":")) for c in out[enc]))
            f.write("\n ]" + ("," if i + 1 < len(ENCODINGS) else "") + "\n")
        f.write("}\n")


if __name__ == "__main__":
    main()
