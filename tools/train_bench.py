"""Time BPE training on the GPU (tiktoken_b200.bpe_train_packed) on a tools/corpus slice (config 2's English-like
documents, cl100k pattern) and, for reference, the C restatement tools/train_oracle.c on the same input.

    python tools/train_bench.py [--sizes-mib 64,1024] [--vocabs 32768,100000] [--ref 64:32768] [--out FILE]

Prints one JSON line per (size, vocab): wall seconds of the call, the trainer's stats (pieces, distinct words, merges,
graph batches, chunks, device ms of the split, the distinct-word stage and the merge loop) and, where --ref names the
pair, the restatement's seconds and whether the two dicts are equal.  The restatement costs O(merges x words) on one
CPU thread, so only the pairs listed in --ref run it.  Needs a CUDA device."""
from __future__ import annotations

import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path[:0] = [ROOT, os.path.join(ROOT, "tests")]

import tiktoken_b200  # noqa: E402
from oracle.oracle import CL100K_PAT  # noqa: E402
from tools import corpus  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--sizes-mib", default="64,1024")
    ap.add_argument("--vocabs", default="32768,100000")
    ap.add_argument("--ref", default="64:32768", help="comma list of size_mib:vocab pairs the C restatement runs on ('' none)")
    ap.add_argument("--seed", type=int, default=1002)
    ap.add_argument("--out", default=None, help="also append the JSON lines to this file")
    a = ap.parse_args()
    refs = {tuple(int(x) for x in r.split(":")) for r in a.ref.split(",") if r}
    import torch
    name = torch.cuda.get_device_name(0)
    lines = []
    for mib in [int(x) for x in a.sizes_mib.split(",")]:
        text, off = corpus.config2(nbytes=mib << 20, seed=a.seed)
        tiktoken_b200.bpe_train_packed(text[:1 << 16], [0, 1 << 16], 300, CL100K_PAT)     # CUDA context, module load
        for vocab in [int(x) for x in a.vocabs.split(",")]:
            t0 = time.perf_counter()
            got = tiktoken_b200.bpe_train_packed(text, off, vocab, CL100K_PAT)
            wall = time.perf_counter() - t0
            rec = {"size_mib": mib, "n_docs": len(off) - 1, "vocab": vocab, "gpu": name, "wall_s": round(wall, 3),
                   **{k: round(v, 3) for k, v in tiktoken_b200.last_train_stats().items()}}
            if (mib, vocab) in refs:
                import train_oracle
                t0 = time.perf_counter()
                want = train_oracle.bpe_train_packed(text, off, vocab, CL100K_PAT)
                rec["ref_s"] = round(time.perf_counter() - t0, 3)
                rec["equal"] = list(got.items()) == list(want.items())
            print(json.dumps(rec), flush=True)
            lines.append(rec)
    if a.out:
        with open(a.out, "a") as f:
            for r in lines:
                f.write(json.dumps(r) + "\n")


if __name__ == "__main__":
    main()
