"""Completion search (Encoding.encode_with_unstable_batch) on the GPU against the tiktoken wheel's per-text
encode_with_unstable over a thread pool of every core, on the same prompts: 1 k and 10 k prompts cut at random scalar
boundaries from the tools/corpus generators, for the cl100k-like and o200k-like synthetic vocabularies.  The GPU time is
a host clock around synchronous calls after a warm-up; outputs are compared (the wheel returns a set per prompt).  One
JSON line per case, with the card's name and power limit read in the same run.

    python tools/unstable_bench.py [--repeats 5]"""
import argparse
import json
import os
import random
import subprocess
import sys
import time
from concurrent.futures import ThreadPoolExecutor

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import tiktoken  # noqa: E402

import tiktoken_b200  # noqa: E402
import vocab_util as vu  # noqa: E402
from tools import corpus  # noqa: E402

KIND = {"cl100k_base": corpus.ENGLISH, "o200k_base": corpus.MIXED}


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                             text=True, timeout=30).stdout.strip().splitlines()[0]
        name, power = [x.strip() for x in out.split(",")]
        return name, power
    except Exception as e:                      # the measurement still stands; the line says what is missing
        return f"unknown ({e})", "unknown"


def prompts(enc, n, seed=1):
    rnd = random.Random(seed)
    text = corpus.generate(KIND[enc], seed, 2_000_000).tobytes().decode("utf-8", "ignore")
    out = []
    for _ in range(n):
        a = rnd.randrange(0, len(text) - 200)
        out.append(text[a:a + rnd.randrange(1, 80)])
    return out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--repeats", type=int, default=5)
    args = ap.parse_args()
    name, power = card()
    for enc in ["cl100k_base", "o200k_base"]:
        pat, ranks, special, _ = vu.load_encoding(enc, allow_real=False)
        e = tiktoken_b200.Encoding(f"ub_{enc}", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)
        w = tiktoken.Encoding(f"ubw_{enc}", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)
        for n in (1000, 10000):
            texts = prompts(enc, n)
            got = e.encode_with_unstable_batch(texts)                    # warm-up (and the lazily built tables)
            t0 = time.perf_counter()
            for _ in range(args.repeats):
                got = e.encode_with_unstable_batch(texts)
            gpu_s = (time.perf_counter() - t0) / args.repeats
            stats = e._core_bpe.last_unstable()
            cores = os.cpu_count() or 1
            t0 = time.perf_counter()
            with ThreadPoolExecutor(cores) as ex:
                ref = list(ex.map(lambda t: w.encode_with_unstable(t), texts))
            cpu_s = time.perf_counter() - t0
            equal = all(g[0] == r[0] and len(g[1]) == len(r[1]) and set(map(tuple, g[1])) == set(map(tuple, r[1]))
                        for g, r in zip(got, ref))
            print(json.dumps({"encoding": enc, "prompts": n, "gpu_ms": round(gpu_s * 1e3, 2),
                              "wheel_ms": round(cpu_s * 1e3, 1), "wheel_threads": cores, "speedup": round(cpu_s / gpu_s, 2),
                              "equal": equal, "card": name, "power_limit": power, **stats}), flush=True)


if __name__ == "__main__":
    main()
