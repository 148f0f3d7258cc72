"""CPU-only check of the EXACT rule code the pre-tokeniser kernel executes
(tiktoken_b200/csrc/pretok_rules.cuh, compiled for the host by hostcheck.cpp) against the literal
backtracking matcher of the oracle."""
import itertools
import json
import os
import random

import numpy as np
import pytest

import vocab_util as vu
from oracle import Oracle

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
BYTES = {bytes([i]): i for i in range(256)}
PATS = {"r50k": (0, vu.R50K_PAT), "cl100k": (1, vu.CL100K_PAT), "o200k": (2, vu.O200K_PAT)}


def rule_starts(H, pid, docs):
    blob = b"".join(docs)
    n = len(blob)
    off = np.zeros(len(docs) + 1, np.uint64)
    off[1:] = np.cumsum([len(d) for d in docs])
    a = np.frombuffer(blob, np.uint8) if n else np.zeros(1, np.uint8)
    out = np.zeros(n + 1, np.uint8)
    assert H.hc_piece_starts(pid, a.ctypes.data, n, off.ctypes.data, len(docs), out.ctypes.data) == 0
    return out[:n], off


def fast_starts(H, pid, docs):
    """The bit-parallel span evaluator the kernel runs (pretok_fast.cuh); also returns slow-path stats."""
    blob = b"".join(docs)
    n = len(blob)
    off = np.zeros(len(docs) + 1, np.uint64)
    off[1:] = np.cumsum([len(d) for d in docs])
    a = np.frombuffer(blob, np.uint8) if n else np.zeros(1, np.uint8)
    out = np.zeros(n + 2, np.uint8)
    st = np.zeros(2, np.uint64)
    assert H.hc_piece_starts_fast(pid, a.ctypes.data, n, off.ctypes.data, len(docs), out.ctypes.data, st.ctypes.data) == 0
    assert out[n] == 1                          # end sentinel
    return out[:n], off, st


def expected_starts(o, doc):
    exp = np.zeros(len(doc), np.uint8)
    p = 0
    for piece in o.split(doc):
        exp[p] = 1
        p += len(piece)
    return exp


@pytest.mark.parametrize("name", ["r50k", "cl100k", "o200k"])
def test_rules_exhaustive(hostcheck, name):
    pid, pat = PATS[name]
    spec = json.load(open(os.path.join(G, "splits_exhaustive.json")))[name]
    o = Oracle(BYTES, {}, pat)
    L = spec["max_len"] - 1                     # one shorter than the oracle pin keeps the CPU suite quick
    for l in range(1, L + 1):
        docs = ["".join(t).encode() for t in itertools.product(spec["alphabet"], repeat=l)]
        got, off = rule_starts(hostcheck, pid, docs)
        for i, d in enumerate(docs):
            assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d)), (name, d)


@pytest.mark.parametrize("name", ["r50k", "cl100k", "o200k"])
def test_rules_random_long_strings(hostcheck, name):
    """Longer strings over the class alphabet (sampled), incl. long homogeneous runs."""
    pid, pat = PATS[name]
    alph = json.load(open(os.path.join(G, "splits_exhaustive.json")))[name]["alphabet"]
    o = Oracle(BYTES, {}, pat)
    rnd = random.Random(11)
    docs = []
    for _ in range(4000):
        n = rnd.choice([7, 8, 9, 12, 20, 40])
        chars = []
        while len(chars) < n:
            chars += [rnd.choice(alph)] * rnd.choice([1, 1, 1, 2, 3, 5, 9])
        docs.append("".join(chars[:n]).encode())
    got, off = rule_starts(hostcheck, pid, docs)
    for i, d in enumerate(docs):
        assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d)), (name, d)


@pytest.mark.parametrize("name", ["r50k", "cl100k", "o200k"])
def test_rules_on_reference_unicode_cases(hostcheck, name):
    """The random Unicode strings whose splits come straight from the reference engine; all packed
    into ONE buffer as separate documents, so document-boundary handling is exercised too."""
    pid, _ = PATS[name]
    cases = json.load(open(os.path.join(G, "splits_random.json")))[name]
    docs = [bytes.fromhex(t) for t, _ in cases]
    got, off = rule_starts(hostcheck, pid, docs)
    for i, (t, pieces) in enumerate(cases):
        exp = np.zeros(len(docs[i]), np.uint8)
        p = 0
        for ph in pieces:
            exp[p] = 1
            p += len(ph) // 2
        assert np.array_equal(got[int(off[i]):int(off[i + 1])], exp), docs[i]


def test_documents_are_separate_haystacks(hostcheck):
    # two docs "a  " + "b": the spaces end doc 0, so they stay one piece; as one doc they split
    got, _ = rule_starts(hostcheck, 1, [b"a  ", b"b"])
    assert got.tolist() == [1, 1, 0, 1]
    got, _ = rule_starts(hostcheck, 1, [b"a  b"])
    assert got.tolist() == [1, 1, 1, 0]
    got, _ = rule_starts(hostcheck, 1, [b"", b"", b"x", b""])
    assert got.tolist() == [1]


@pytest.mark.parametrize("name", ["r50k", "cl100k", "o200k"])
def test_fast_path_exhaustive(hostcheck, name):
    """pretok_fast.cuh (SWAR masks + slow-path fallback) == literal matcher, every string up to L-1."""
    pid, pat = PATS[name]
    spec = json.load(open(os.path.join(G, "splits_exhaustive.json")))[name]
    o = Oracle(BYTES, {}, pat)
    for l in range(1, spec["max_len"]):
        docs = ["".join(t).encode() for t in itertools.product(spec["alphabet"], repeat=l)]
        got, off, _ = fast_starts(hostcheck, pid, docs)
        for i, d in enumerate(docs):
            assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d)), (name, d)


@pytest.mark.parametrize("name", ["r50k", "cl100k", "o200k"])
def test_fast_path_on_reference_unicode_cases_and_corpus(hostcheck, name):
    pid, pat = PATS[name]
    cases = json.load(open(os.path.join(G, "splits_random.json")))[name]
    docs = [bytes.fromhex(t) for t, _ in cases]
    got, off, _ = fast_starts(hostcheck, pid, docs)
    for i, (t, pieces) in enumerate(cases):
        exp = np.zeros(len(docs[i]), np.uint8)
        p = 0
        for ph in pieces:
            exp[p] = 1
            p += len(ph) // 2
        assert np.array_equal(got[int(off[i]):int(off[i + 1])], exp), docs[i]
    # seeded corpus of the matching kind, cut into documents at arbitrary scalar boundaries
    from tools import corpus
    kind = {"r50k": corpus.CODE, "cl100k": corpus.ENGLISH, "o200k": corpus.MIXED}[name]
    text = corpus.generate(kind, 321, 1 << 20)
    _, doff = corpus.docs_fixed(text, 40000, at_space=False)
    cdocs = [text[int(doff[i]):int(doff[i + 1])].tobytes() for i in range(len(doff) - 1)]
    o = Oracle(BYTES, {}, pat)
    got, off, st = fast_starts(hostcheck, pid, cdocs)
    for i, d in enumerate(cdocs):
        assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d))
    assert st[1] < 0.1 * st[0]                  # the slow path stays the exception


def test_fast_path_documents_are_separate_haystacks(hostcheck):
    got, _, _ = fast_starts(hostcheck, 1, [b"a  ", b"b"])
    assert got.tolist() == [1, 1, 0, 1]
    got, _, _ = fast_starts(hostcheck, 1, [b"a  b"])
    assert got.tolist() == [1, 1, 1, 0]
    got, _, _ = fast_starts(hostcheck, 2, [b"", b"", b"x", b""])
    assert got.tolist() == [1]


@pytest.mark.parametrize("name", ["cl100k", "o200k"])
def test_fast_path_digit_run_behind_a_scalar_cut_by_the_window(hostcheck, name):
    """Regression (found by tools/fuzz_cpu.py): a non-ASCII digit whose lead byte lies before a span's
    48-byte window left 'unknown' continuation bytes that were taken for a non-digit, so an ASCII digit
    run right after it got a wrong run start.  Slide digit runs behind 2-, 3- and 4-byte digits (and
    non-digits) over every alignment."""
    pid, pat = PATS[name]
    o = Oracle(BYTES, {}, pat)
    heads = ["\u00b2", "\u0660", "\u2160", "\uff12", "\U0001d7d8", "\u4e2d", "\u00e9", "\U0001f600"]
    docs = []
    for pad in range(0, 40):
        for head in heads:
            for reps in (1, 2):
                for nd in (1, 3, 6, 7, 8, 9, 10):
                    docs.append(("a" * pad + head * reps + "2" * nd + " x").encode())
    got, off, _ = fast_starts(hostcheck, pid, docs)
    for i, d in enumerate(docs):
        assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d)), d


def test_fuzz_harness_short_run():
    """tools/fuzz_cpu.py (random multi-document batches through the kernel's pre-tokeniser code, random
    adversarial vocabularies through its merge code, both against the oracle) for a few seconds."""
    import subprocess
    import sys
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    r = subprocess.run([sys.executable, os.path.join(root, "tools", "fuzz_cpu.py"), "8", "4242"],
                       capture_output=True, text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:] + r.stderr[-2000:]
    assert "all equal" in r.stdout


@pytest.mark.timeout(120)
def test_malformed_utf8_terminates(hostcheck):
    """The packed / device entry points take raw bytes.  Malformed UTF-8 has no reference answer, but the
    rule code must still terminate and stay in bounds (a forward walk in the o200k chain automaton used to
    step over its target on such input and never end)."""
    rnd = random.Random(3)
    for it in range(400):
        mode = it % 3
        n = rnd.choice([1, 5, 33, 100, 1000])
        if mode == 0:
            blob = bytes(rnd.randrange(256) for _ in range(n))
        elif mode == 1:
            blob = bytes(rnd.choice([0x80, 0xBF, 0xE0, 0xF0, 0xC2, 0x41, 0x20, 0x0A, 0xFF, 0xF8, 0x27]) for _ in range(n))
        else:
            blob = bytes([rnd.choice([0x80, 0xE3, 0xF0])]) * n
        cuts = sorted(rnd.randrange(n + 1) for _ in range(rnd.randint(0, 3)))
        docs = [blob[a:b] for a, b in zip([0] + cuts, cuts + [n])]
        for pid in range(3):
            got, _, _ = fast_starts(hostcheck, pid, docs)
            assert len(got) == n


def test_cl100k_contraction_rule_is_exact(hostcheck):
    """The cl100k contraction rule: letters 2..3 bytes after an apostrophe decided per apostrophe (is it
    's|'t|'re|'ve|'m|'ll|'d, where does it end) instead of by the general function; with it English text has no
    undecided position left.  The whitespace-after-CR/LF cases stay with the general function (there is no bit-parallel
    rule for them) and are checked here all the same."""
    H = hostcheck
    pid, pat = PATS["cl100k"]
    o = Oracle(BYTES, {}, pat)
    spec = json.load(open(os.path.join(G, "splits_exhaustive.json")))["cl100k"]
    alphabet = spec["alphabet"] + ["v", "e", "r", "\u017f", "L"]
    for l in range(1, 5):
        docs = ["".join(t).encode() for t in itertools.product(alphabet, repeat=l)]
        got, off, _ = fast_starts(H, pid, docs)
        for i, d in enumerate(docs):
            assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d)), d
    docs = []
    for pad in range(40):
        for pre in ["x", "1", " ", "!", "\n", "", "\u00e9"]:
            for suf in ["s", "S", "t", "d", "m", "ll", "LL", "lL", "ve", "re", "rE", "l", "v", "r", "sx", "llx", "lx",
                        "\u017f", "\u212a", "\u00e9"]:
                for post in ["", "a", " ", "'s", "1"]:
                    docs.append(("z" * pad + pre + "'" + suf + post).encode())
    got, off, _ = fast_starts(H, pid, docs)
    for i, d in enumerate(docs):
        assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d)), d
    # whitespace right after CR/LF (indentation), runs shorter and longer than the window,
    # CR/LF runs behind punctuation, document ends
    docs = []
    for pad in range(0, 40, 3):
        for pre in ["x", "!", "!\n", "x\n\n", "!\r\n\n", "", "/\n"]:
            for nl in ["\n", "\r\n", "\n" * 10]:
                for ws in [" ", "    ", "\t", " " * 9, " " * 20, " " * 45, "\u3000", " \u3000"]:
                    for post in ["x", "\n", "\nx", "", "!", "\n\n  y"]:
                        docs.append(("z" * pad + pre + nl + ws + post).encode())
    got, off, _ = fast_starts(H, pid, docs)
    for i, d in enumerate(docs):
        assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d)), d
    for l in range(1, 6):
        docs = ["".join(t).encode() for t in itertools.product(["a", " ", "\t", "\n", "\r", "!", "/"], repeat=l)]
        got, off, _ = fast_starts(H, pid, docs)
        for i, d in enumerate(docs):
            assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d)), d
    cases = json.load(open(os.path.join(G, "splits_random.json")))["cl100k"]
    docs = [bytes.fromhex(t) for t, _ in cases]
    got, off, _ = fast_starts(H, pid, docs)
    for i, d in enumerate(docs):
        assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d)), d
    from tools import corpus
    text = corpus.generate(corpus.ENGLISH, 99, 1 << 20)
    _, doff = corpus.docs_fixed(text, 30000, at_space=False)
    cdocs = [text[int(doff[i]):int(doff[i + 1])].tobytes() for i in range(len(doff) - 1)]
    got, off, st = fast_starts(H, pid, cdocs)
    for i, d in enumerate(cdocs):
        assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d))
    assert st[1] * 1000 < st[0]                 # < 0.1 % undecided (0.42 % without the rule)


def test_r50k_contractions_at_every_alignment(hostcheck):
    """The case-sensitive `'(?:[sdmt]|ll|ve|re)` of the r50k / p50k pattern (decided by the general function).  Documents are packed back to back,
    so apostrophes also meet across document boundaries."""
    H = hostcheck
    pid, pat = PATS["r50k"]
    o = Oracle(BYTES, {}, pat)
    spec = json.load(open(os.path.join(G, "splits_exhaustive.json")))["r50k"]
    alphabet = spec["alphabet"] + ["v", "e", "r", "S", "\u00e9"]
    for l in range(1, 5):
        docs = ["".join(t).encode() for t in itertools.product(alphabet, repeat=l)]
        got, off, _ = fast_starts(H, pid, docs)
        for i, d in enumerate(docs):
            assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d)), d
    docs = []
    for pad in range(40):
        for pre in ["x", "1", " ", "!", "\n", "", "\u00e9", "'"]:
            for suf in ["s", "S", "t", "d", "m", "ll", "LL", "lL", "ve", "re", "rE", "l", "v", "sx", "llx", "lx", "\u017f",
                        "\u00e9a", "\u4e2da", "1", ""]:
                for post in ["", "a", " ", "'s", "1"]:
                    docs.append(("z" * pad + pre + "'" + suf + post).encode())
    got, off, _ = fast_starts(H, pid, docs)
    for i, d in enumerate(docs):
        assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d)), d
    cases = json.load(open(os.path.join(G, "splits_random.json")))["r50k"]
    docs = [bytes.fromhex(t) for t, _ in cases]
    got, off, _ = fast_starts(H, pid, docs)
    for i, d in enumerate(docs):
        assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d)), d


def test_o200k_prefix_and_apostrophe_rules_are_exact(hostcheck):
    """The two o200k rules: a letter after a punctuation scalar decided bit-parallel as
    boundary(p) = !boundary(x), and apostrophes / contraction tails decided per apostrophe.  Exhaustive strings, the
    real engine's random Unicode splits, a mixed-script corpus, and a short fuzz run."""
    import subprocess
    import sys
    from conftest import ROOT, _build_hostcheck
    H, so = hostcheck, _build_hostcheck()
    pid, pat = PATS["o200k"]
    o = Oracle(BYTES, {}, pat)
    spec = json.load(open(os.path.join(G, "splits_exhaustive.json")))["o200k"]
    for l in range(1, spec["max_len"]):
        docs = ["".join(t).encode() for t in itertools.product(spec["alphabet"], repeat=l)]
        got, off, _ = fast_starts(H, pid, docs)
        for i, d in enumerate(docs):
            assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d)), d
    # punctuation of every UTF-8 length in front of letters of every kind, at every alignment
    xs = ["(", "«", "、", "\U0001f600", "'", "/", "́"]
    befores = ["a", "1", " ", "\t", "\n", "(", "'", "、", "", "́", "/", "中"]
    letters = ["a", "A", "中", "é", "ǅ"]
    docs = []
    for pad in range(0, 34):
        for bf in befores:
            for x in xs:
                for le in letters:
                    docs.append(("z" * pad + bf + x + le + "b c").encode())
    got, off, _ = fast_starts(H, pid, docs)
    for i, d in enumerate(docs):
        assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d)), d
    # apostrophes: contraction tails of words, chains of them, apostrophes as prefixes / inside
    # punctuation runs, every alignment
    docs = []
    for pad in range(0, 34):
        for pre in ["x", "X", "1", " ", "!", "\n", "", "\u00e9", "\u4e2d", "\u0301", "/", "'", "a'", "a's", "a'll"]:
            for suf in ["s", "S", "t", "d", "m", "ll", "lL", "ve", "re", "rE", "l", "v", "sx", "sX", "llx", "lx",
                        "\u017f", "\u212a", "\u00e9", "1", " ", "!", ""]:
                for post in ["", "a", " ", "'s", "B"]:
                    docs.append(("z" * pad + pre + "'" + suf + post).encode())
    got, off, _ = fast_starts(H, pid, docs)
    for i, d in enumerate(docs):
        assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d)), d
    # whitespace right after CR/LF (general function); CR/LF runs behind punctuation / slashes / marks
    docs = []
    for pad in range(0, 40, 4):
        for pre in ["x", "!", "!\n", "x\n\n", "", "/\n", "!\n/", "a/", "x\u0301", "!\u0301"]:
            for nl in ["\n", "\r\n", "\n" * 10, "\n/\n"]:
                for ws in [" ", "    ", "\t", " " * 9, " " * 20, " " * 45, "\u3000"]:
                    for post in ["x", "\n", "\nx", "", "!", "\n\n  y"]:
                        docs.append(("z" * pad + pre + nl + ws + post).encode())
    got, off, _ = fast_starts(H, pid, docs)
    for i, d in enumerate(docs):
        assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d)), d
    alphabet = ["a", "A", "s", "l", "e", "'", "!", " ", "\n", "1", "\u0301", "\u3042"]
    for l in range(1, 5):
        docs = ["".join(t).encode() for t in itertools.product(alphabet, repeat=l)]
        got, off, _ = fast_starts(H, pid, docs)
        for i, d in enumerate(docs):
            assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d)), d
    cases = json.load(open(os.path.join(G, "splits_random.json")))["o200k"]
    docs = [bytes.fromhex(t) for t, _ in cases]
    got, off, _ = fast_starts(H, pid, docs)
    for i, d in enumerate(docs):
        assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d)), d
    from tools import corpus
    text = corpus.generate(corpus.MIXED, 99, 1 << 20)
    _, doff = corpus.docs_fixed(text, 30000, at_space=False)
    cdocs = [text[int(doff[i]):int(doff[i + 1])].tobytes() for i in range(len(doff) - 1)]
    got, off, st_new = fast_starts(H, pid, cdocs)
    for i, d in enumerate(cdocs):
        assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d))
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "fuzz_cpu.py"), "6", "777"], capture_output=True,
                       text=True, timeout=300, env=dict(os.environ, B200BPE_HOSTCHECK=so))
    assert r.returncode == 0 and "all equal" in r.stdout, r.stdout[-2000:] + r.stderr[-2000:]


@pytest.mark.parametrize("name", ["cl100k", "o200k"])
def test_long_whitespace_runs_behind_line_ends(hostcheck, name):
    """The listed positions behind CR/LF walk their whitespace run eight bytes at a time (ws_run_ahead: SWAR on an aligned
    64-bit word + the doc-start bits): runs of every length and alignment, with later line ends or none, non-ASCII
    whitespace inside, ending at a letter, at the document end or at a document boundary in the middle of a run."""
    pid, pat = PATS[name]
    o = Oracle(BYTES, {}, pat)
    rnd = random.Random(2026)
    ws_ascii = [" ", " ", " ", "\t", "\x0b", "\x0c"]
    for trial in range(400):
        parts = []
        for _ in range(rnd.randint(1, 4)):
            run = [rnd.choice(ws_ascii) for _ in range(rnd.choice([0, 1, 2, 7, 8, 9, 15, 16, 17, 40, 200]))]
            for _ in range(rnd.choice([0, 0, 1, 3])):
                run.insert(rnd.randint(0, len(run)), rnd.choice(["\n", "\r", "\r\n", " ", "　", " "]))
            parts.append(rnd.choice(["x", "", "é", "1", ".", "\n", "ab\n", "\r"]) + "".join(run) + rnd.choice(["y", "", "\n", "z9", "中"]))
        text = ("q" * rnd.randint(0, 9)) + "".join(parts)                      # every alignment of the run to the 8-byte words
        raw = text.encode()
        cuts = sorted({0, len(raw)} | {rnd.randint(0, len(raw)) for _ in range(rnd.choice([0, 1, 3]))})
        cuts = [c for c in cuts if c == len(raw) or (raw[c] & 0xC0) != 0x80]   # document boundaries on scalar starts
        docs = [raw[a:b] for a, b in zip(cuts[:-1], cuts[1:])] or [raw]
        got, off, _ = fast_starts(hostcheck, pid, docs)
        for i, d in enumerate(docs):
            assert np.array_equal(got[int(off[i]):int(off[i + 1])], expected_starts(o, d)), (name, d)
