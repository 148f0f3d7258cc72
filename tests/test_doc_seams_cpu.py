"""The seam rule and the chunk plan of the host path (tiktoken_b200/csrc/doc_seams.h, host build through hostcheck.cpp).

A seam p is a position where a document larger than a chunk may be cut: split(s) == split(s[:p]) + split(s[p:]).  The
rule is checked against the oracle's literal backtracking matcher and against the pre-tokeniser rule code the kernels
run (hc_piece_starts, hc_piece_starts_fast), on every string of a few scalars of context around each rule's bytes and on
seeded random strings with long runs.  The planner is checked for the document-boundary plan wherever no document is larger than two
chunks, for seams that satisfy the rule and cut no special token, and for its chunk bound."""
import ctypes as C
import itertools
import random

import numpy as np
import pytest

import vocab_util as vu
from oracle import Oracle

BYTES = {bytes([i]): i for i in range(256)}
PATS = {"r50k": (0, vu.R50K_PAT), "cl100k": (1, vu.CL100K_PAT), "o200k": (2, vu.O200K_PAT)}
ALPHABET = ["a", "Z", "7", " ", "\n", "\r", "\t", "'", "s", "/", ".", "é", "́", " ", "　", "中"]
# each rule's bytes, with p the offset of the seam in them
R1_CORES = [("a b", 1), ("s Z", 1), ("Z s", 1)]
R2_CORES = [(".\na", 2), ("s\n7", 2), ("/\nZ", 2), ("'\ns", 2), ("7\nZ", 2)]
PLAN_WHOLE, PLAN_DOCS, PLAN_SEAMS = 0, 1, 2


@pytest.fixture(scope="module")
def H(hostcheck):
    hostcheck.hc_is_seam.argtypes = [C.c_void_p, C.c_uint64, C.c_uint64, C.c_uint64]
    hostcheck.hc_plan_chunks.restype = C.c_int64
    hostcheck.hc_plan_chunks.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint64, C.c_int, C.c_void_p, C.c_void_p,
                                         C.c_uint64, C.c_void_p, C.c_uint64, C.c_void_p, C.c_void_p, C.c_void_p, C.c_void_p]
    return hostcheck


def rule(b: bytes, lo: int, hi: int, p: int) -> bool:
    """R1 / R2 as DESIGN §4b states them (independent of doc_seams.h)."""
    if not lo < p < hi:
        return False
    letter = lambda c: (65 <= c <= 90) or (97 <= c <= 122)
    if p + 1 < hi and b[p] == 0x20 and letter(b[p - 1]) and letter(b[p + 1]):
        return True
    return p - 2 >= lo and b[p - 1] == 0x0A and 0x21 <= b[p - 2] <= 0x7E and (letter(b[p]) or 48 <= b[p] <= 57)


def product_seam_seams(H, b: bytes) -> list[int]:
    a = np.frombuffer(b, np.uint8)
    got = [p for p in range(len(b)) if H.hc_is_seam(a.ctypes.data, 0, len(b), p)]
    assert got == [p for p in range(len(b)) if rule(b, 0, len(b), p)], b
    return got


def starts_of(pieces) -> set[int]:
    out, p = set(), 0
    for piece in pieces:
        out.add(p)
        p += len(piece)
    return out


def check_seam_oracle(o, b: bytes, p: int, cache_l: dict, cache_r: dict):
    whole = o.split(b)
    assert p in starts_of(whole), (b, p)
    left = cache_l[b[:p]] if b[:p] in cache_l else cache_l.setdefault(b[:p], o.split(b[:p]))
    right = cache_r[b[p:]] if b[p:] in cache_r else cache_r.setdefault(b[p:], o.split(b[p:]))
    assert whole == left + right, (b, p)


def check_seams_kernel_rules(H, pid: int, cases: list[tuple[bytes, int]]):
    """The piece starts of the kernels' rule code for s as one document equal those for s[:p] and s[p:] as two
    documents, and p is a piece start of s."""
    blob = b"".join(b for b, _ in cases)
    n = len(blob)
    a = np.frombuffer(blob, np.uint8)
    lens = np.asarray([len(b) for b, _ in cases], np.int64)
    one = np.zeros(len(cases) + 1, np.uint64)
    one[1:] = np.cumsum(lens)
    two = np.sort(np.concatenate([one, one[:-1] + np.asarray([p for _, p in cases], np.uint64)])).astype(np.uint64)
    for fn, extra in ((H.hc_piece_starts, ()), (H.hc_piece_starts_fast, (None,))):
        s1, s2 = np.zeros(n + 2, np.uint8), np.zeros(n + 2, np.uint8)
        assert fn(pid, a.ctypes.data, n, one.ctypes.data, len(one) - 1, s1.ctypes.data, *extra) == 0
        assert fn(pid, a.ctypes.data, n, two.ctypes.data, len(two) - 1, s2.ctypes.data, *extra) == 0
        bad = np.nonzero(s1[:n] != s2[:n])[0]
        assert len(bad) == 0, [cases[int(np.searchsorted(one, x, side="right")) - 1] for x in bad[:5]]


def contexts(k: int) -> list[str]:
    return ["".join(t) for n in range(k + 1) for t in itertools.product(ALPHABET, repeat=n)]


@pytest.mark.parametrize("name", ["r50k", "cl100k", "o200k"])
def test_rule_exhaustive_around_each_core(H, name):
    """Every left and right context of up to two scalars each, and of up to three on one side alone."""
    pid, pat = PATS[name]
    o = Oracle(BYTES, {}, pat)
    c2, c3 = contexts(2), contexts(3)
    pairs = [(l, r) for l in c2 for r in c2] + [(l, "") for l in c3 if len(l) == 3] + [("", r) for r in c3 if len(r) == 3]
    n_checked = 0
    for core, at in R1_CORES + R2_CORES:
        cache_l, cache_r, cases = {}, {}, []
        for l, r in pairs:
            b = (l + core + r).encode()
            p = len(l.encode()) + at
            assert H.hc_is_seam(np.frombuffer(b, np.uint8).ctypes.data, 0, len(b), p) == 1, (b, p)
            check_seam_oracle(o, b, p, cache_l, cache_r)
            cases.append((b, p))
        check_seams_kernel_rules(H, pid, cases)
        n_checked += len(cases)
    assert n_checked == len(pairs) * 8


RUNS = [" ", "\n", "\r\n", "\t", "a", "Z", "q", "7", "́", "é", " ", "　", "中", ".", "/", "'", "'s", "'ll",
        "s", "Ab", "x y", "z\nQ", ".\n1", "?\nw", "  \n", "\n\n"]


def random_string(rnd: random.Random) -> bytes:
    parts = []
    for _ in range(rnd.randint(2, 10)):
        parts.append(rnd.choice(RUNS) * (rnd.randint(1, 12) if rnd.random() < 0.4 else 1))
        if rnd.random() < 0.3:
            parts.append(rnd.choice([c for c, _ in R1_CORES + R2_CORES]))
    return "".join(parts).encode()


@pytest.mark.parametrize("name", ["r50k", "cl100k", "o200k"])
def test_rule_on_random_strings_with_long_runs(H, name):
    pid, pat = PATS[name]
    o = Oracle(BYTES, {}, pat)
    rnd = random.Random(1000 + pid)
    n_strings, n_seams, cases = 0, 0, []
    while n_strings < 34_000:
        b = random_string(rnd)
        n_strings += 1
        for p in product_seam_seams(H, b):
            check_seam_oracle(o, b, p, {}, {})
            cases.append((b, p))
            n_seams += 1
    check_seams_kernel_rules(H, pid, cases)
    assert n_seams > n_strings // 2


def rule_negative_cases():
    """Bytes next to each rule that must not be seams: the whitespace run before '\\n' (r50k's `\\s+(?!\\S)`), '/' after
    it (o200k's `[\\r\\n/]*`), a letter that is not ASCII, and the document edges."""
    return [(b"a  b", 2), (b"a \nb", 3), (b".\n/", 2), (b"\xc3\xa9 b", 2), (b"a \xc3\xa9", 1), (b"\n\nb", 2), (b" b", 0),
            (b"a ", 1), (b"\nb", 1)]


def test_rule_rejects_its_neighbours(H):
    for b, p in rule_negative_cases():
        assert H.hc_is_seam(np.frombuffer(b, np.uint8).ctypes.data, 0, len(b), p) == 0, (b, p)
        assert not rule(b, 0, len(b), p)


# ---- the chunk plan -----------------------------------------------------------------------------------------------
def doc_plan(off, chunk):
    """Document ranges of the host path's chunks before seams (one chunk up to 1.5 chunks; a document larger than a
    chunk is a chunk of its own)."""
    n_docs, cut = len(off) - 1, [0]
    if int(off[-1]) <= chunk + chunk // 2:
        return [0, n_docs]
    lo = 0
    while lo < n_docs:
        hi = int(np.searchsorted(off, int(off[lo]) + chunk, side="right")) - 1
        hi = min(max(hi, lo + 1), n_docs)
        cut.append(hi)
        lo = hi
    return cut


def plan(H, text: bytes, off, chunk: int, mode: int = PLAN_SEAMS, specials=(), flags=None):
    a = np.frombuffer(text, np.uint8) if text else np.zeros(1, np.uint8)
    off = np.ascontiguousarray(off, np.uint64)
    sp = [s.encode() for s in specials]
    sp_blob = np.frombuffer(b"".join(sp) or b"\0", np.uint8)
    sp_off = np.zeros(len(sp) + 1, np.uint64)
    sp_off[1:] = np.cumsum([len(s) for s in sp])
    fl = None if flags is None else np.asarray(flags, np.uint8)
    cap = len(text) + len(off) + 8
    bounds, first, head, st = np.zeros(cap + 1, np.uint64), np.zeros(cap + 1, np.uint64), np.zeros(cap, np.uint8), np.zeros(2, np.uint64)
    n = H.hc_plan_chunks(a.ctypes.data, off.ctypes.data, len(off) - 1, chunk, mode, sp_blob.ctypes.data, sp_off.ctypes.data,
                         len(sp), None if fl is None else fl.ctypes.data, cap, bounds.ctypes.data, first.ctypes.data,
                         head.ctypes.data, st.ctypes.data)
    assert n >= 0, n
    return bounds[:n + 1].tolist(), first[:n + 1].tolist(), head[:n].tolist(), {"seams": int(st[0]), "docs_cut": int(st[1])}


def check_plan_shape(text: bytes, off, bounds, first, head, stats):
    """Chunks tile the batch; a chunk starts at the start of its first document or at a seam strictly inside the
    document before it, and that seam satisfies R1 or R2."""
    off = [int(x) for x in off]
    n_docs = len(off) - 1
    assert bounds[0] == 0 and bounds[-1] == off[-1] and first[0] == 0 and first[-1] == n_docs
    assert all(a <= b for a, b in zip(bounds, bounds[1:])) and all(a <= b for a, b in zip(first, first[1:]))
    seams, docs = 0, set()
    for c, h in enumerate(head):
        d = first[c]
        if h:
            lo, hi = off[d - 1], off[d]
            assert lo < bounds[c] < hi and rule(text, lo, hi, bounds[c]), (c, bounds[c])
            assert h == (2 if (d - 1) not in docs else 1)
            seams += 1
            docs.add(d - 1)
        else:
            assert d < n_docs and bounds[c] == off[d] or (d == n_docs and bounds[c] == off[-1])
    assert stats == {"seams": seams, "docs_cut": len(docs)}


def test_plan_with_documents_of_at_most_two_chunks_is_the_document_plan(H):
    rnd = np.random.default_rng(7)
    for trial in range(300):
        chunk = int(rnd.integers(64, 4096))
        lens = rnd.integers(0, 2 * chunk + 1, size=int(rnd.integers(0, 60)))
        if trial % 3 == 0:
            lens[rnd.random(len(lens)) < 0.3] = 0                           # empty documents, at chunk bounds too
        text = bytes(rnd.choice(np.frombuffer(b"ab cd\nef. 12", np.uint8), size=int(lens.sum())))
        off = np.concatenate([[0], np.cumsum(lens)]).astype(np.uint64)
        want = doc_plan(off, chunk)
        for mode in (PLAN_SEAMS, PLAN_DOCS):
            bounds, first, head, st = plan(H, text, off, chunk, mode)
            assert first == want and bounds == [int(off[i]) for i in want] and not any(head), (trial, mode)
            assert st == {"seams": 0, "docs_cut": 0}


def english(n: int, seed: int) -> bytes:
    rnd = random.Random(seed)
    words = ["the", "of", "and", "Tokens", "x7", "don't", "it's", "naïve", "数据", "—", "http://a.b/c"]
    out, size = [], 0
    while size < n:
        w = rnd.choice(words) + (rnd.choice([" ", " ", " ", "\n", ". ", ",\n", "  "]))
        out.append(w)
        size += len(w.encode())
    return "".join(out).encode()[:n]


def test_plan_cuts_large_documents_at_seams_within_the_bound(H):
    chunk = 4096
    for seed in range(20):
        docs = [english(int(n), seed * 100 + i) for i, n in
                enumerate(np.random.default_rng(seed).choice([0, 50, 3000, 9000, 40_000], size=12))]
        text = b"".join(docs)
        off = np.concatenate([[0], np.cumsum([len(d) for d in docs])]).astype(np.uint64)
        bounds, first, head, st = plan(H, text, off, chunk)
        check_plan_shape(text, off, bounds, first, head, st)
        assert all(b - a <= chunk + chunk // 4 for a, b in zip(bounds, bounds[1:])), seed
        if max(len(d) for d in docs) > chunk * 2:
            assert st["seams"] > 0
        # the document plan for comparison: the same chunk starts wherever no document was cut
        docs_only = doc_plan(off, chunk)
        assert plan(H, text, off, chunk, PLAN_DOCS)[1] == docs_only
        assert plan(H, text, off, chunk, PLAN_WHOLE)[1] == [0, len(docs)]


def test_plan_without_seams_keeps_the_whole_document(H):
    chunk = 1024
    cjk = ("中文字符" * 2000).encode()
    run = b"a" * 10_000
    spaces = b" " * 5000 + b"\n" * 5000
    for docs in ([cjk], [run], [b"x y", cjk, b"z"], [spaces, run, cjk]):
        text = b"".join(docs)
        off = np.concatenate([[0], np.cumsum([len(d) for d in docs])]).astype(np.uint64)
        bounds, first, head, st = plan(H, text, off, chunk)
        assert st == {"seams": 0, "docs_cut": 0} and not any(head)
        assert first == doc_plan(off, chunk)


def test_plan_seam_windows_and_a_late_seam(H):
    """A document whose only seam lies two chunks in: the first target has none in its window, so the chunk runs on to
    the next target."""
    chunk = 1000
    doc = "中".encode() * 600 + b"ab cd" + "中".encode() * 600
    p = 1800 + 2
    bounds, first, head, st = plan(H, doc, [0, len(doc)], chunk)
    assert bounds == [0, p, len(doc)] and head == [0, 2] and first == [0, 1, 1]
    assert st == {"seams": 1, "docs_cut": 1}


def test_plan_never_cuts_a_special_token(H):
    specials = ["x y", "q\nZ", "<|endoftext|>"]
    rnd = random.Random(3)
    chunk = 512
    for trial in range(60):
        parts = []
        while sum(map(len, parts)) < 6000:
            parts.append(rnd.choice(["x y", "q\nZ", "ab ", "x", "y ", "q\n", "Z", "<|endoftext|>", " "]))
        text = "".join(parts).encode()
        off = [0, len(text)]
        flags = [rnd.choice([0, 1, 2]) for _ in specials]
        if not any(flags):
            flags[0] = 1
        bounds, first, head, st = plan(H, text, off, chunk, specials=specials, flags=flags)
        check_plan_shape(text, off, bounds, first, head, st)
        for s, f in zip(specials, flags):
            if not f:
                continue
            sb = s.encode()
            occ = [q for q in range(len(text)) if text.startswith(sb, q)]
            for c in range(1, len(bounds) - 1):
                assert not any(q < bounds[c] < q + len(sb) for q in occ), (trial, s, bounds[c])
    # without special handling the same texts do get seams inside "x y"
    text = b"x y" * 2000
    bounds, _, _, st = plan(H, text, [0, len(text)], chunk)
    assert st["seams"] > 0 and any(text[b - 1:b + 2] == b"x y" for b in bounds[1:-1])
    bounds, _, _, st = plan(H, text, [0, len(text)], chunk, specials=specials, flags=[1, 0, 0])
    assert st["seams"] == 0 and bounds == [0, len(text)]                 # every word gap lies inside an "x y"
