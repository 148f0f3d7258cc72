"""Inputs that overflow one work-space of the encoder each, and the capacities they overflow.

The engine sizes four device work-spaces per pipeline call, and the host token buffer per encode call, from
experience rather than for the worst case.  When one is too small the kernels raise a flag and keep counting, and the
host grows the buffer to the exact need and runs the same work again.  The recipes below reach each of those paths on
purpose; they are generated in code, deterministic in their seed.

The capacities are written down once, here.  They restate the first-run sizes of `enqueue_pipeline` and `encode_host`
in tiktoken_b200/csrc/b200bpe.cu; test_regrow_inputs.py checks every recipe against them on the CPU, so a change to
the sizing shows up there before a GPU test silently stops reaching its path.  N is the byte count of one pipeline
call: a host-path chunk or one device call.
"""
from __future__ import annotations

import itertools

import numpy as np

MISS_CAP_MIN = 1 << 16          # b200bpe.cu MISS_CAP_MIN: floor of the miss queue, miss results and undecided positions
LONG_CAP_MIN = 1 << 20          # b200bpe.cu LONG_CAP_MIN: floor of the long-piece merge scratch
SHORT_MAX = 16                  # bpe_device.cuh: pieces up to this length are probed whole; the others are "long"
LONG_SCRATCH_MIN = 256          # dev_common.cuh: pieces longer than this merge in the global scratch


def caps(n: int) -> dict[str, int]:
    """First-run capacities of one pipeline call of n bytes (enqueue_pipeline), and of the host token buffer of an
    encode call of n bytes on an engine whose pinned pool is empty (encode_host, pass 0: n/2 + 4096 tokens asked of
    take_pinned, which allocates 1/8 + 4096 bytes more)."""
    tok_bytes = 4 * (n // 2 + 4096)
    return {
        "misses": max(n // 8 + 4096, MISS_CAP_MIN),          # miss queue entries (ERR_MISSCAP)
        "miss_bytes": max(n // 2 + 4096, MISS_CAP_MIN),      # miss result space = summed bytes of the missed pieces
        "slow": max(n // 8 + 4096, MISS_CAP_MIN),            # undecided pre-tokeniser positions (ERR_SLOWCAP)
        "long_bytes": max(n // 8 + 4096, LONG_CAP_MIN),      # bytes of pieces > 256 in the merge scratch (ERR_LONGCAP)
        "tokens": (tok_bytes + tok_bytes // 8 + 4096) // 4,  # host token buffer, pass 0 (second pass of encode_host)
    }


# which quantity of caps() each recipe is built to exceed, and the work-space that grows for it
# (the names of CoreBPE.last_reruns()["grown"]; "tokens" is the host buffer: a second token pass instead)
GROWS = {"misses": "miss", "miss_bytes": "miss", "slow": "slow", "long_bytes": "long", "tokens": None}


def miss_vocab(with_numbers: bool = False) -> dict[bytes, int]:
    """The 256 bytes, every {a, b} string of 2..3 letters with and without a leading space, " a" and " b": with the
    cl100k pattern every word of other letters, or of four and more {a, b} letters, misses the piece table.
    with_numbers adds every number of 1..3 digits, so that digit runs merge without a miss."""
    toks = [bytes([i]) for i in range(256)]
    words = ["".join(p) for k in (2, 3) for p in itertools.product("ab", repeat=k)]
    toks += [w.encode() for w in words] + [(" " + w).encode() for w in words] + [b" a", b" b"]
    if with_numbers:
        toks += [str(i).encode() for i in range(10, 1000)] + [f"{i:02d}".encode() for i in range(10)]
        toks += [f"{i:03d}".encode() for i in range(100)]
    seen, out = set(), {}
    for t in toks:
        if t not in seen:
            seen.add(t)
            out[t] = len(out)
    return out


def _pack(units: list[str], per_doc: int):
    """Units -> (uint8 text, uint64 document offsets), per_doc units per document.  Recipes cut only where a piece
    ends anyway, so the documents do not change the pre-tokeniser's split."""
    blob = "".join(units).encode()
    lens = np.fromiter((len(u) for u in units), np.int64, len(units))
    ends = np.cumsum(lens)
    off = np.concatenate([[0], ends[per_doc - 1::per_doc]])
    if off[-1] != len(blob):
        off = np.append(off, len(blob))
    return np.frombuffer(blob, np.uint8).copy(), off.astype(np.uint64)


def _letters(rng, alphabet: str, n: int) -> str:
    return "".join(rng.choice(list(alphabet), n))


def miss(seed: int = 0, n_words: int = 700_000, per_doc: int = 20_000):
    """MISS (miss_vocab, cl100k): " " + 4..6 letters of {a, b}.  Every word is one missed piece of 5..7 bytes: more
    misses than N/8 and more missed bytes than N/2."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(4, 7, n_words)
    s = _letters(rng, "ab", int(lens.sum()))
    pos = np.concatenate([[0], np.cumsum(lens)])
    return _pack([" " + s[pos[i]:pos[i + 1]] for i in range(n_words)], per_doc)


def miss_results_only(seed: int = 0, n_words: int = 150_000, per_doc: int = 10_000):
    """MISS, results only (miss_vocab, cl100k): " " + 12..15 letters of {a, b}: fewer misses than N/8, but more
    missed bytes than N/2."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(12, 16, n_words)
    s = _letters(rng, "ab", int(lens.sum()))
    pos = np.concatenate([[0], np.cumsum(lens)])
    return _pack([" " + s[pos[i]:pos[i + 1]] for i in range(n_words)], per_doc)


def miss_queue_only(seed: int = 0, n_units: int = 500_000, per_doc: int = 25_000):
    """MISS, queue only (miss_vocab, cl100k): a 2-digit number (a missed piece of 2 bytes) then " " + 3 letters of
    {a, b} (one token of 4 bytes).  One miss per 6 bytes is more than N/8; the missed bytes, N/3, stay under N/2, and
    the tokens, N/2, under the token buffer."""
    rng = np.random.default_rng(seed)
    nums = rng.integers(10, 100, n_units)
    s = _letters(rng, "ab", 3 * n_units)
    return _pack([f"{nums[i]} {s[3 * i:3 * i + 3]}" for i in range(n_units)], per_doc)


def slow(seed: int = 0, n_numbers: int = 400_000, per_doc: int = 20_000):
    """SLOW (cl100k_like, cl100k): comma-separated random integers of 9..12 digits.  The bit-parallel pre-tokeniser
    cannot decide the positions inside long digit runs alone: about 0.3 N of them go to the undecided list."""
    rng = np.random.default_rng(seed)
    lens = rng.integers(9, 13, n_numbers)
    s = "".join(rng.choice(list("0123456789"), int(lens.sum())))
    pos = np.concatenate([[0], np.cumsum(lens)])
    return _pack([s[pos[i]:pos[i + 1]] + "," for i in range(n_numbers)], per_doc)


def long_runs(seed: int = 0, nbytes: int = 3_350_000, per_doc: int = 200, lo: int = 300, hi: int = 5000):
    """LONG (cl100k_like, cl100k): the letters of the English corpus only, cut into runs of lo..hi letters joined by
    single spaces.  Every run is one piece of more than 256 bytes, so nearly all N bytes go to the merge scratch."""
    from tools import corpus
    text = corpus.generate(corpus.ENGLISH, 4000 + seed, 2 * nbytes)
    letters = text[((text >= 65) & (text <= 90)) | ((text >= 97) & (text <= 122))].tobytes().decode()
    rng = np.random.default_rng(seed)
    units, p = [], 0
    while p < nbytes:
        n = int(rng.integers(lo, hi + 1))
        units.append((" " if units else "") + letters[p:p + n])
        p += n
    return _pack(units, per_doc)


def tokens(seed: int = 0, n_lines: int = 1_500_000, per_doc: int = 50_000):
    """TOKENS (cl100k_like, cl100k): one random letter + "\\n" per line: one token per byte, twice the pass-0 token
    buffer of N/2."""
    rng = np.random.default_rng(seed)
    s = _letters(rng, "abcdefghijklmnopqrstuvwxyz", n_lines)
    return _pack([c + "\n" for c in s], per_doc)


# name -> (generator, vocabulary (see vocabulary()), the quantities of caps() it exceeds)
RECIPES = {
    "miss": (miss, "miss", {"misses", "miss_bytes"}),
    "miss_results_only": (miss_results_only, "miss", {"miss_bytes"}),
    "miss_queue_only": (miss_queue_only, "miss", {"misses"}),
    "slow": (slow, "cl100k_base", {"slow"}),
    "long": (long_runs, "cl100k_base", {"long_bytes"}),
    "tokens": (tokens, "cl100k_base", {"tokens"}),
}


def vocabulary(kind: str):
    """-> (pat_str, mergeable_ranks, special_tokens) of a recipe's vocabulary: "miss", "miss+numbers" or a synthetic
    encoding of vocab_util."""
    import vocab_util as vu
    if kind.startswith("miss"):
        return vu.CL100K_PAT, miss_vocab(with_numbers=kind == "miss+numbers"), {}
    pat, ranks, special, _ = vu.load_encoding(kind, allow_real=False)
    return pat, ranks, special


def measure(oracle, ranks: dict[bytes, int], hostcheck, text: np.ndarray, off: np.ndarray) -> dict[str, int]:
    """What one pipeline call over (text, off) needs, counted on the CPU: pieces from the oracle's split, undecided
    positions from the `slow` statistic of the span evaluator pretok_kernel runs (hc_piece_starts_fast), tokens from
    the oracle's encode."""
    n = len(text)
    raw = text.tobytes()
    misses = miss_bytes = long_bytes = 0
    for d in range(len(off) - 1):
        for p in oracle.split(raw[int(off[d]):int(off[d + 1])]):
            k = len(p)
            if 2 <= k <= SHORT_MAX and p not in ranks:
                misses += 1
                miss_bytes += k
            elif k > LONG_SCRATCH_MIN:
                long_bytes += k
    starts = np.zeros(n + 2, np.uint8)
    st = np.zeros(2, np.uint64)
    a = text if n else np.zeros(1, np.uint8)
    assert hostcheck.hc_piece_starts_fast(1, a.ctypes.data, n, off.ctypes.data, len(off) - 1, starts.ctypes.data,
                                          st.ctypes.data) == 0               # 1 = PAT_CL100K
    toks, _ = oracle.encode_ordinary_batch_np(text, off, 8)
    return {"misses": misses, "miss_bytes": miss_bytes, "slow": int(st[1]), "long_bytes": long_bytes,
            "tokens": len(toks)}


BATCH_VOCAB = "miss+numbers"     # miss_vocab(with_numbers=True): one vocabulary on which every batch document overflows


def batch(seed: int = 0, nbytes: int = 16 << 20):
    """MISS, SLOW, LONG and TOKENS documents interleaved in one batch, for 1 MiB chunks on miss_vocab(True).  MISS,
    SLOW and TOKENS documents are 0.85..1 MiB, so that every chunk is one document and a MISS or SLOW chunk overflows
    its work-space alone; LONG documents are 1.2..1.5 MiB, because a chunk of 1 MiB cannot exceed the 1 MiB scratch
    floor.  LONG and TOKENS are about one token per byte on this vocabulary, so the batch also overflows the pass-0
    token buffer.  -> (text, doc_off, kinds) with the recipe of every document."""
    rng = np.random.default_rng(seed)
    parts, kinds, total = [], [], 0
    for i in itertools.count():
        kind = ("miss", "slow", "long", "tokens")[i % 4]
        want = int(rng.integers(int(1.35 * (1 << 20)), int(1.7 * (1 << 20)))) if kind == "long" else \
            int(rng.integers(int(0.85 * (1 << 20)), 1 << 20))
        s = 1000 * seed + i
        if kind == "miss":
            t, _ = miss(s, want // 6, 1 << 30)
        elif kind == "slow":
            t, _ = slow(s, want * 2 // 25, 1 << 30)
        elif kind == "long":
            t, _ = long_runs(s, want, 1 << 30)
        else:
            t, _ = tokens(s, want // 2, 1 << 30)
        parts.append(t)
        kinds.append(kind)
        total += len(t)
        if total >= nbytes:
            break
    off = np.concatenate([[0], np.cumsum([len(p) for p in parts])]).astype(np.uint64)
    return np.concatenate(parts), off, kinds
