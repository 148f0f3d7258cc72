#!/usr/bin/env python
"""Long documents through the public host API, from pinned packed input (tools/corpus.py, synthetic vocabularies):

  c2_one    config 2's English-like text (cl100k_base) as ONE document
  c2_docs   the same bytes in their usual ~64 KiB documents
  c5        config 5: one 64 MiB code-like document (p50k_base)

Arms: Encoding.encode_ordinary_packed (TokenBuffer closed right away) and Encoding.count_packed.  Per arm: wall clock of
the call (it returns after the device work and the copies), the engine's device_total_ms of the last call (summed over
chunks, the slowest device), and the device memory the engine holds after the calls: work-spaces only grow, so with
b200bpe_trim between workloads this is the peak of the workload (read with cudaMemGetInfo, over every device the
engine uses).  With --devices all the engine spreads over every visible GPU.  Prints the card and its power limit,
then one JSON line per workload and device set.  Writes nothing.

    python tools/long_doc_bench.py [--bytes N] [--reps R] [--devices 1|all|1,all] [--workloads c2_one,c2_docs,c5]
"""
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

from tools.count_bench import card  # noqa: E402


def workload(name, nbytes):
    from tools import corpus
    if name == "c2_one":
        text, _ = corpus.config2(nbytes=nbytes)
        return "cl100k_base", text, np.asarray([0, len(text)], np.uint64)
    if name == "c2_docs":
        return ("cl100k_base", *corpus.config2(nbytes=nbytes))
    if name == "c5":
        return ("p50k_base", *corpus.config5())
    raise ValueError(name)


def used_bytes(devices):
    import torch
    out = 0
    for d in devices:
        free, total = torch.cuda.mem_get_info(d)
        out += total - free
    return out


def stats(xs):
    return {"median": round(statistics.median(xs), 3), "min": round(min(xs), 3)}


def run(name, devices, args):
    import torch
    import tiktoken_b200
    import vocab_util as vu
    enc_name, text, off = workload(name, args.bytes)
    h_text = torch.from_numpy(text).pin_memory().numpy()
    pat, ranks, special, _ = vu.load_encoding(enc_name, allow_real=False)
    for d in devices:
        torch.cuda.synchronize(d)
    base = used_bytes(devices)
    enc = tiktoken_b200.Encoding(f"long_doc_{name}", pat_str=pat, mergeable_ranks=ranks, special_tokens=special,
                                 devices=devices)
    core = enc._core_bpe
    tables = used_bytes(devices) - base
    res = {"workload": name, "encoding": enc_name, "bytes": len(text), "docs": len(off) - 1, "devices": len(devices),
           "reps": args.reps}
    offs = {}
    for arm in ("encode", "count"):
        core.trim()
        wall, dev = [], []
        for rep in range(args.reps + 1):                       # the first call grows the work-spaces: not timed
            t0 = time.perf_counter()
            if arm == "encode":
                with enc.encode_ordinary_packed(h_text, off) as buf:
                    o = np.array(buf.offsets())
            else:
                o = enc.count_packed(h_text, off, disallowed_special=())
            ms = (time.perf_counter() - t0) * 1e3
            if rep:
                wall.append(ms)
                dev.append(core.last_timings()["device_total_ms"])
        offs[arm] = o
        res[f"{arm}_wall_ms"] = stats(wall)
        res[f"{arm}_device_ms"] = stats(dev)
        res[f"{arm}_workspace_gib"] = round((used_bytes(devices) - base - tables) / (1 << 30), 2)
        res[f"{arm}_gbps"] = round(len(text) / (statistics.median(wall) * 1e-3) / 1e9, 2)
        if hasattr(core, "last_doc_seams"):
            res[f"{arm}_seams"] = core.last_doc_seams()
    res["tokens"] = int(offs["encode"][-1])
    res["count_equals_encode"] = bool(np.array_equal(offs["encode"], offs["count"]))
    core.trim()
    del enc, core
    return res


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bytes", type=int, default=1 << 30, help="config 2 bytes (c2_one, c2_docs)")
    ap.add_argument("--reps", type=int, default=5)
    ap.add_argument("--devices", default="1,all", help="1: cuda:0 alone; all: every visible GPU (skipped with one)")
    ap.add_argument("--workloads", default="c2_one,c2_docs,c5")
    args = ap.parse_args()
    import torch
    if not torch.cuda.is_available():
        print(json.dumps({"error": "no CUDA device: tiktoken_b200 has no CPU fallback"}))
        sys.exit(1)
    print(json.dumps(card()), flush=True)
    n = torch.cuda.device_count()
    sets = []
    for s in args.devices.split(","):
        if s == "1":
            sets.append([0])
        elif s == "all" and n > 1:
            sets.append(list(range(n)))
    ok = True
    for devices in sets:
        for w in args.workloads.split(","):
            r = run(w, devices, args)
            ok &= r["count_equals_encode"]
            print(json.dumps(r), flush=True)
    sys.exit(0 if ok else 1)


if __name__ == "__main__":
    main()
