"""Seeded vocabularies and pieces for every length class of the long-piece merge kernels, at every rank width.

Pieces longer than 16 bytes are queued by length class (dev_common.cuh) and merged by a different kernel per class, and
by a different family of kernels when the largest rank is 2^22 or above (b200bpe.cu: the group and parallel-merge
kernels pack `rank << 10 | position` into 32 bits).  Each kernel has its own copy of the whole-piece probe (hash the
piece, look it up in the long-token table), of the missing-single-byte report and of the rank packing.  The inputs here
reach all of them on purpose:

  * a tiny-alphabet vocabulary with random distinct ranks (ties impossible, cascades frequent) and long tokens at every
    class boundary, most of them unreachable by merges, so that only the whole-piece probe can produce them;
  * per class: exact hits on those tokens, near misses of the same length (first byte, last byte, a byte of the last
    64-bit hash word changed), a token with one byte dropped or added, and adversarial merge pieces (random, periodic,
    runs) in batches of 1..70 pieces of one length;
  * rank layouts: the same vocabulary with a constant added to every rank, which keeps every merge, so that the largest
    rank sits at each limit of the engine;
  * a vocabulary without the single byte "c": pieces whose every "c" ends inside a merged token, and per class one piece
    that leaves a "c" alone.

test_merge_class_inputs.py checks all of this with the oracle on the CPU; test_gpu_merge_classes.py runs it on the GPU.
"""
from __future__ import annotations

import bisect
import random

import numpy as np

ALPHA = "abcd"                  # every token and piece letter except the top pair
TOP_PAIR = b"ee"                # the largest rank of every layout: a pair no other token contains
SHORT_LENS = (2, 2, 2, 3, 3, 4, 5, 7, 9, 12, 14, 20, 40)
N_SHORT = 90
# long tokens at every class boundary, and inside the classes; lengths that are not a multiple of 8 end the hash on a
# partial word.  The table build copies every split of every token (quadratic in its length): few tokens above 32 768.
TOKEN_LENS = (17, 23, 32, 33, 47, 64, 65, 100, 127, 128, 129, 200, 255, 256, 257, 600, 1023, 1024, 1025, 2048, 3001,
              4095, 4096, 4097, 10001, 32768, 32769, 40003)
# adversarial merge pieces: length -> the batch sizes drawn for it (one class batch holds up to 32 pieces)
ADV_LENS = (17, 18, 31, 32, 33, 34, 63, 64, 65, 66, 127, 128, 129, 130, 200, 255, 256, 257, 258, 300, 400, 511, 512,
            513, 700, 1023, 1024, 1025, 1100, 1500, 2047, 3000, 4000, 4095, 4096, 4097, 5000, 32768, 32769, 50000)
CLASS_MIN = (17, 33, 65, 129, 257, 1025, 4097, 32769)     # dev_common.cuh: first length of classes 0..7
N_CLS = len(CLASS_MIN)
GROUP_MAX_RANK = 1 << 22        # kernels_mid.cuh MIDG_MAX_RANK: from here on the lane-per-piece family runs
DEVICE_DECODE_MAX = 1 << 24     # b200bpe.cu: any id at or above this decodes on the host maps
RANK_LIMIT = 1 << 30            # bpe_tables.h: ranks must be below this
RANK_MAX = 0xFFFFFFFF           # the oracle's mark of a missing single byte
MISSING = b"c"


def length_class(n: int) -> int:
    """Length class of a piece of n > 16 bytes (find_long_kernel)."""
    assert n >= CLASS_MIN[0]
    return bisect.bisect_right(CLASS_MIN, n) - 1


def _word(rnd, n: int, alpha: str = ALPHA) -> str:
    return "".join(rnd.choice(alpha) for _ in range(n))


def base_vocab(seed: int = 0) -> dict[bytes, int]:
    """The 256 bytes at ranks 0..255; N_SHORT random {a..d} tokens of SHORT_LENS bytes and one random {a..d} token of
    each TOKEN_LENS length at random distinct ranks above them; TOP_PAIR at the largest rank."""
    rnd = random.Random(seed)
    ranks = {bytes([i]): i for i in range(256)}
    short = set()
    while len(short) < N_SHORT:
        short.add(_word(rnd, rnd.choice(SHORT_LENS)).encode())
    toks = sorted(short) + [_word(rnd, n).encode() for n in TOKEN_LENS]
    for t, r in zip(toks, rnd.sample(range(256, 256 + 4 * len(toks)), len(toks))):
        ranks[t] = r
    ranks[TOP_PAIR] = 256 + 4 * len(toks)
    return ranks


def long_tokens(ranks: dict[bytes, int]) -> list[bytes]:
    """The tokens of TOKEN_LENS bytes, shortest first."""
    by_len = {len(t): t for t in ranks if len(t) in TOKEN_LENS}
    return [by_len[n] for n in TOKEN_LENS]


def _other(rnd, ch: int) -> int:
    return ord(rnd.choice([c for c in ALPHA if ord(c) != ch]))


def _change(rnd, t: bytes, i: int) -> bytes:
    return t[:i] + bytes([_other(rnd, t[i])]) + t[i + 1:]


def _adversarial(rnd, n: int) -> str:
    style = rnd.choice(["random", "random", "periodic", "runs"])
    if style == "random":
        return _word(rnd, n)
    if style == "periodic":
        unit = _word(rnd, rnd.choice([1, 2, 3, 5, 7]))
        return (unit * (n // len(unit) + 1))[:n]
    w = ""
    while len(w) < n:
        w += rnd.choice(ALPHA) * rnd.choice([1, 2, 3, 9, 17, 40, 1000])
    return w[:n]


def pieces(ranks: dict[bytes, int], seed: int = 0) -> list[tuple[str, bytes]]:
    """(kind, piece) for the base vocabulary (or any layout of it).  Kinds: "hit"; "near_first", "near_last",
    "near_word" (a byte of the last hash word, not the last byte when the word has two or more); "drop", "add"; "adv"
    (one of a batch of 1..70 adversarial pieces of one length); "top" (1022 letters then TOP_PAIR: the largest rank
    merges at position 1022 of a 1024-byte piece)."""
    rnd = random.Random(1000 + seed)
    out = []
    for t in long_tokens(ranks):
        n = len(t)
        w0 = 8 * ((n - 1) // 8)                              # first byte of the last 64-bit word of the hash
        out += [("hit", t), ("near_first", _change(rnd, t, 0)), ("near_last", _change(rnd, t, n - 1)),
                ("near_word", _change(rnd, t, rnd.randrange(w0, n - 1) if n - 1 > w0 else w0))]
        i = rnd.randrange(n)
        out += [("drop", t[:i] + t[i + 1:]), ("add", t[:i] + rnd.choice(ALPHA).encode() + t[i:])]
    for n in ADV_LENS:
        k = rnd.choice([1, 5, 33, 70]) if n <= 300 else rnd.choice([1, 2, 7]) if n <= 4096 else 1
        out += [("adv", _adversarial(rnd, n).encode()) for _ in range(k)]
    out.append(("top", _word(rnd, 1022).encode() + TOP_PAIR))
    return out


def documents(items: list[bytes], seed: int = 0, per_doc: int = 40):
    """Pieces in shuffled order, per_doc of them per document, separated by "\\n" (a piece of its own under every
    pattern: a space would join the next letter run); one empty document.  -> (uint8 text, uint64 offsets)."""
    rnd = random.Random(2000 + seed)
    order = list(items)
    rnd.shuffle(order)
    docs = [b"\n".join(order[i:i + per_doc]) for i in range(0, len(order), per_doc)]
    docs.insert(len(docs) // 2, b"")
    off = np.zeros(len(docs) + 1, np.uint64)
    off[1:] = np.cumsum([len(d) for d in docs])
    blob = b"".join(docs)
    return np.frombuffer(blob, np.uint8).copy(), off


def class_counts(lengths) -> list[int]:
    """Pieces per length class (pieces of 16 bytes and fewer are not queued)."""
    c = [0] * N_CLS
    for n in lengths:
        if n >= CLASS_MIN[0]:
            c[length_class(n)] += 1
    return c


# name -> the largest rank of the layout (None: as built).  "all_ge_2p22" puts the SMALLEST rank at 2^22.
LAYOUTS = {
    "as_built": None,
    "top_2p22m1": GROUP_MAX_RANK - 1,
    "top_2p22": GROUP_MAX_RANK,
    "all_ge_2p22": "all",
    "top_2p24m1": DEVICE_DECODE_MAX - 1,
    "top_2p24": DEVICE_DECODE_MAX,
    "top_2p30m1": RANK_LIMIT - 1,
}


def offset(ranks: dict[bytes, int], layout: str) -> int:
    """The constant a layout adds to every rank."""
    top = LAYOUTS[layout]
    if top is None:
        return 0
    if top == "all":
        return GROUP_MAX_RANK - min(ranks.values())
    return top - max(ranks.values())


def shifted(ranks: dict[bytes, int], c: int) -> dict[bytes, int]:
    return {t: r + c for t, r in ranks.items()}


def lane_per_piece(ranks: dict[bytes, int]) -> bool:
    """Which kernel family the engine selects for these ranks."""
    return max(ranks.values()) >= GROUP_MAX_RANK


def special_tokens(ranks: dict[bytes, int]) -> dict[str, int]:
    """For vocabularies whose ids reach 2^24 (they decode on the host maps, and special ids take the same path): a
    special token at 2^25, or just below the smallest rank when the ranks reach 2^25 (special ids must stay below 2^30
    too).  None otherwise, so that the bit-packed return width follows the ranks alone."""
    top = max(ranks.values())
    if top < DEVICE_DECODE_MAX:
        return {}
    return {"<|x|>": 1 << 25 if top < 1 << 25 else min(ranks.values()) - 1}


# ---- the vocabulary without MISSING ------------------------------------------------------------------------------
MISSING_LENS = ((17, 24, 32), (33, 47, 64), (65, 100, 128), (129, 200, 256), (257, 600, 1024), (1025, 2000, 4096),
                (4097, 6000), (32769,))    # per class: lengths of the pieces that merge every "c" away


def missing_byte_vocab(seed: int = 0) -> dict[bytes, int]:
    """base_vocab without the single byte MISSING; the tokens that contain it stay."""
    ranks = base_vocab(seed)
    del ranks[MISSING]
    return ranks


def _fails(oracle, p: bytes) -> bool:
    return RANK_MAX in oracle.encode_single_piece(p)


def missing_byte_pieces(oracle, ranks: dict[bytes, int], seed: int = 0):
    """-> (ok, bad): ok = pieces of every class with one to three "c" that all end inside a merged token; bad[cls] =
    one piece of that class that leaves a "c" alone.  Drawn with the oracle of the missing-byte vocabulary (rejection
    sampling: {a, b, d} letters, "c" inserted at random places)."""
    rnd = random.Random(3000 + seed)
    ok, bad = [], {}
    for cls, lens in enumerate(MISSING_LENS):
        for n in lens:
            while True:
                w = list(_word(rnd, n - rnd.randint(1, 3), "abd"))
                for _ in range(n - len(w)):
                    w.insert(rnd.randrange(len(w) + 1), "c")
                p = "".join(w).encode()
                if p not in ranks and not _fails(oracle, p):
                    ok.append(p)
                    break
        while cls not in bad:
            w = _word(rnd, lens[0] - 1, "abd")
            i = rnd.randrange(len(w) + 1)
            p = (w[:i] + "c" + w[i:]).encode()
            if p not in ranks and _fails(oracle, p):
                bad[cls] = p
    return ok, bad
