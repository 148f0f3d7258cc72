"""Worst case of the per-call miss memo: a corpus in which every missed piece is distinct, so the memo merges as many
pieces as before and only adds its passes.  Encodes it device-resident with the memo on and off in one process and
prints the device time per step of each; then prints misses / merged for configs 2 to 5, the repetition the memo's
gain depends on.

    python tools/miss_memo_bench.py [--bytes N] [--steps K] [--warmup W] [--configs-bytes N]
"""
import argparse
import json
import os
import subprocess
import sys

import numpy as np

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def distinct_miss_corpus(nbytes: int, seed: int = 7, doc_bytes: int = 65536):
    """Words of 9..14 random lowercase letters behind a space: every word is one piece of 10..15 bytes that no synthetic
    vocabulary holds, and 26^9 possible words make a repeat rare (the tests check small samples on the CPU)."""
    from tools import corpus
    rng = np.random.default_rng(seed)
    n_words = nbytes // 11 + 16
    lens = rng.integers(9, 15, n_words) + 1
    text = rng.integers(ord("a"), ord("z") + 1, int(lens.sum()), dtype=np.uint8)
    text[np.cumsum(lens) - lens] = ord(" ")
    text = text[:nbytes]
    return corpus.docs_fixed(text, doc_bytes, at_space=True)


def _engine(memo_slots, enc="cl100k_base"):
    import tiktoken_b200
    import vocab_util as vu
    pat, ranks, special, _ = vu.load_encoding(enc, allow_real=False)
    if memo_slots is None:
        os.environ.pop("B200BPE_MISS_MEMO_SLOTS", None)
    else:
        os.environ["B200BPE_MISS_MEMO_SLOTS"] = str(memo_slots)
    return tiktoken_b200.Encoding(f"memo_{enc}_{memo_slots}", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)


def _device_ms(e, text, off, steps, warmup):
    import torch
    d_text = torch.from_numpy(text).cuda()
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()
    d_tok = torch.empty(len(text) + 16, dtype=torch.int32, device="cuda")
    d_toff = torch.empty(len(off), dtype=torch.int64, device="cuda")
    core = e._core_bpe
    s = torch.cuda.Stream()
    ms, stages = [], []
    for i in range(warmup + steps):
        core.encode_device(d_text.data_ptr(), len(text), d_off.data_ptr(), len(off) - 1, d_tok.data_ptr(), d_toff.data_ptr(),
                           s.cuda_stream)
        if i >= warmup:
            t = core.last_timings()
            ms.append(t["device_total_ms"])
            stages.append(t["encode_ms"] - t["probe_ms"])
    return float(np.median(ms)), float(np.median(stages)), core.last_miss_memo()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--bytes", type=int, default=1 << 30)
    ap.add_argument("--steps", type=int, default=10)
    ap.add_argument("--warmup", type=int, default=3)
    ap.add_argument("--configs-bytes", type=int, default=1 << 30)
    a = ap.parse_args()
    import torch
    from tools import corpus
    gpu = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                         text=True).stdout.strip()
    print(json.dumps({"gpu": gpu}))
    text, off = distinct_miss_corpus(a.bytes)
    res = {}
    for label, slots in (("memo_on", None), ("memo_off", 0)):
        e = _engine(slots)
        res[label] = _device_ms(e, text, off, a.steps, a.warmup)
        del e
        torch.cuda.empty_cache()
    on, off_ = res["memo_on"], res["memo_off"]
    print(json.dumps({"workload": "all-distinct misses", "bytes": int(len(text)),
                      "memo_on": {"device_ms": round(on[0], 3), "miss_stage_ms": round(on[1], 3), **on[2]},
                      "memo_off": {"device_ms": round(off_[0], 3), "miss_stage_ms": round(off_[1], 3), **off_[2]},
                      "memo_cost_pct": round(100.0 * (on[0] - off_[0]) / off_[0], 2)}))
    cfgs = {"config2": ("cl100k_base", lambda: corpus.config2(nbytes=a.configs_bytes)),
            "config3": ("o200k_base", lambda: corpus.config3(nbytes=a.configs_bytes)),
            "config4": ("cl100k_base", lambda: corpus.config4()),
            "config5": ("p50k_base", lambda: corpus.config5())}
    for name, (enc, gen) in cfgs.items():
        eng = _engine(None, enc)
        t, o = gen()
        ms, stage, m = _device_ms(eng, t, o, 3, 1)
        print(json.dumps({"workload": name, "bytes": int(len(t)), "device_ms": round(ms, 3), "miss_stage_ms": round(stage, 3),
                          **m, "misses_per_merged": round(m["misses"] / max(1, m["merged"]), 2)}))
        del eng, t, o
        torch.cuda.empty_cache()


if __name__ == "__main__":
    main()
