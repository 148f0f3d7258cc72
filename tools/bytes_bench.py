#!/usr/bin/env python
"""Bytes mode against the ordinary path on the config 2 corpus (cl100k, English-like text in ~64 KiB documents).

The variants run `Encoding.encode_bytes_packed` and, alternately, `encode_ordinary_packed` on the same pinned input, and
report the device time of the call (`last_timings()["device_total_ms"]`, summed over chunks) and the end-to-end
throughput (wall clock of the whole call, host copies included):

  valid        the corpus as it is: bytes mode pays the UTF-8 check and finds nothing
  trunc_1pct   1 % of the documents end in a truncated scalar (the common real case)
  stray_0.1pct 0.1 % of the documents have a stray 0xFF in the middle
  tail_1MiB    one document ends in 1 MiB of random bytes: one unstable piece of 1 MiB
  tail_16MiB   one document ends in 16 MiB of random bytes

The ordinary path cannot encode the damaged variants the same way; it runs on the valid corpus each time, as the
yardstick.  One JSON line per variant.  Writes nothing."""
import argparse
import json
import os
import statistics
import sys
import time

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def _variants(text, off, rng):
    docs_n = len(off) - 1
    yield "valid", text, off

    def rebuild(edits):
        """edits: {doc: (insert_at_relative or -1 for end, bytes)} -> new text, off"""
        parts, new_off, pos = [], [0], 0
        for d in range(docs_n):
            a, b = int(off[d]), int(off[d + 1])
            doc = text[a:b]
            if d in edits:
                at, ins = edits[d]
                at = len(doc) if at < 0 else at
                doc = np.concatenate([doc[:at], np.frombuffer(ins, np.uint8), doc[at:]])
            parts.append(doc)
            pos += len(doc)
            new_off.append(pos)
        return np.concatenate(parts), np.asarray(new_off, np.uint64)

    pick = rng.choice(docs_n, max(1, docs_n // 100), replace=False)
    yield "trunc_1pct", *rebuild({int(d): (-1, [b"\xe2\x82", b"\xc3", b"\xf0\x9f\x98"][i % 3]) for i, d in enumerate(pick)})
    pick = rng.choice(docs_n, max(1, docs_n // 1000), replace=False)
    yield "stray_0.1pct", *rebuild({int(d): (int(off[d + 1] - off[d]) // 2, b"\xff") for d in pick})
    for name, n in (("tail_1MiB", 1 << 20), ("tail_16MiB", 16 << 20)):
        yield name, *rebuild({docs_n // 2: (-1, b"\xff" + rng.integers(0, 256, n - 1, dtype=np.uint8).tobytes())})


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bytes", type=int, default=1 << 30, help="corpus size (config 2: 1 GiB)")
    ap.add_argument("--reps", type=int, default=3, help="timed calls of each path per variant, alternating")
    ap.add_argument("--variants", default="", help="comma-separated subset")
    args = ap.parse_args()
    import torch
    import tiktoken_b200
    import vocab_util as vu
    from tools import corpus
    pat, ranks, special, src = vu.load_encoding("cl100k_base")
    e = tiktoken_b200.Encoding("bytes_bench", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)
    text, off = corpus.config2(nbytes=args.bytes)
    want = set(args.variants.split(",")) if args.variants else None
    props = torch.cuda.get_device_properties(0)
    card = {"gpu": props.name, "vocab": src}
    try:
        import subprocess
        card["power_limit"] = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                                             capture_output=True, text=True, timeout=20).stdout.strip()
    except Exception:
        card["power_limit"] = "unknown"
    pin = lambda a: torch.from_numpy(a).pin_memory().numpy()   # noqa: E731  pinned, like bench.py's input
    base_t, base_o = pin(text), off

    def timed(fn, t, o):
        t0 = time.perf_counter()
        buf = fn(t, o)
        wall = time.perf_counter() - t0
        ms = e._core_bpe.last_timings()["device_total_ms"]
        n = buf.n_tokens
        buf.close()
        return wall, ms, n

    timed(e.encode_ordinary_packed, base_t, base_o)                # warm-up: work-spaces, pinned pool
    for name, t, o in _variants(text, off, np.random.default_rng(5)):
        if want and name not in want:
            continue
        t = pin(t)
        timed(e.encode_bytes_packed, t, o)
        rb, ro = [], []
        for _ in range(args.reps):
            rb.append(timed(e.encode_bytes_packed, t, o))
            repairs = e._core_bpe.last_bytes_repairs()
            ro.append(timed(e.encode_ordinary_packed, base_t, base_o))
        med = lambda xs, i: statistics.median(x[i] for x in xs)   # noqa: E731
        print(json.dumps({"variant": name, "bytes": int(len(t)), "repaired_docs": repairs,
                          "bytes_mode": {"device_ms": round(med(rb, 1), 3), "e2e_GBps": round(len(t) / med(rb, 0) / 1e9, 2),
                                         "runs_device_ms": [round(x[1], 3) for x in rb]},
                          "ordinary_valid": {"device_ms": round(med(ro, 1), 3),
                                             "e2e_GBps": round(len(base_t) / med(ro, 0) / 1e9, 2),
                                             "runs_device_ms": [round(x[1], 3) for x in ro]},
                          **card}), flush=True)


if __name__ == "__main__":
    main()
