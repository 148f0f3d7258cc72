#!/usr/bin/env python
"""Generate golden/encode_bytes.json: what the REAL reference engine's `Encoding._encode_bytes` (src/py.rs:72-115)
returns for byte strings that are mostly NOT valid UTF-8, for the four synthetic vocabularies in golden/vocab/.  Needs
the `tiktoken` wheel importable; run in the build container, the output is committed, the GPU box never runs this.
It pins tests/bytes_oracle.py (and through it the bytes mode of the CUDA engine) to the real engine."""
import json, os, random, sys

HERE = os.path.dirname(os.path.abspath(__file__))
ROOT = os.path.dirname(os.path.dirname(HERE))
sys.path.insert(0, ROOT); sys.path.insert(0, os.path.join(ROOT, "tests"))
import tiktoken                           # noqa: E402  (the installed reference engine)
import vocab_util as vu                   # noqa: E402

BYTES_EDGE = [b"", b"a", b"\xff", b"\x80", b" \xec\x8b\xa4\xed", b"hello world\xe2\x82", b"hello\xffworld",
              b"\xc0\xaf", b"ab \xe0\x80\x80", b"x\xed\xa0\x80y", b"\xf4\x90\x80\x80", b"\xf5 z", b"\xc1\xbf",
              b"caf\xc3", b"\xf0\x9f\x98", b"\xf0\x9f\x98\x80\xf0\x9f", b"a.\n\n\xff", b"end.\n\n\n\xe4\xb8",
              b"x\n\n  \n\t\xff", b"line\r\n\xff", b"line\r\n\r\n\xc3", b"hi <|endoftext|>\xff", b"<|endoftext|>\xe2\x82",
              b"   \xff", b"\t\t\n \xff tail text", b"don't\xff", b"123456\xff789", b"\xff" * 40,
              b"word \xed\xb2\x80 after", b"\xe3\x81\x82\xe3\x81" + b"x" * 20]


def bytes_fixture():
    rnd = random.Random(20261015)
    pool = [b"a", b"b", b" ", b"\n", b"\t", b"\r", b".", b"'", b"1", b"\xc3\xa9", b"\xe3\x81\x82", b"\xf0\x9f\x98\x80"]
    bad = [b"\xff", b"\x80", b"\xc3", b"\xe3\x81", b"\xf0\x9f", b"\xed\xa0\x80", b"\xc0\xaf", b"\xf4\x90\x80\x80"]
    cases = list(BYTES_EDGE)
    for _ in range(300):
        body = b"".join(rnd.choice(pool) for _ in range(rnd.randint(0, 24)))
        tail = b"".join(rnd.choice(pool + bad) for _ in range(rnd.randint(0, 6)))
        cases.append(body + rnd.choice(bad) + tail)
    for _ in range(60):
        cases.append(bytes(rnd.randrange(256) for _ in range(rnd.randint(1, 40))))
    out = {}
    for enc in ["cl100k_base", "r50k_base", "p50k_base", "o200k_base"]:
        pat, ranks, special, src = vu.load_encoding(enc, allow_real=False)
        e = tiktoken.Encoding(enc + "_synthetic", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)
        out[enc] = [[b.hex(), e._encode_bytes(b)] for b in cases]
        print("encode_bytes", enc, len(cases), file=sys.stderr)
    return out


if __name__ == "__main__":
    json.dump(bytes_fixture(), open(os.path.join(HERE, "encode_bytes.json"), "w"), indent=0)
