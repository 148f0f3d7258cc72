"""Bytes mode on the CPU: the restatement of `_encode_bytes` (src/py.rs:72-115) in bytes_oracle.py against the real
engine's outputs committed in golden/encode_bytes.json (golden/make_bytes_golden.py), the device's UTF-8 classifier (utf8_check.cuh, run on the host through
hostcheck.cpp) against Python's strict decoder, and the new shim / Encoding methods on a stub of the library."""
import ctypes as C
import json
import os
import random

import numpy as np
import pytest

import vocab_util as vu
from bytes_oracle import BytesOracle, valid_up_to
from oracle import Oracle
from test_host_shim_stub import StubLib

HERE = os.path.dirname(os.path.abspath(__file__))
ENCODINGS = ["cl100k_base", "r50k_base", "p50k_base", "o200k_base"]


@pytest.fixture(scope="module")
def golden():
    with open(os.path.join(HERE, "golden", "encode_bytes.json")) as f:
        return json.load(f)


@pytest.mark.parametrize("enc", ENCODINGS)
def test_oracle_matches_the_wheel(golden, enc):
    pat, ranks, special, _ = vu.load_encoding(enc, allow_real=False)
    o = BytesOracle(Oracle(ranks, special, pat), ranks)
    cases = golden[enc]
    assert len(cases) > 300
    bad = [h for h, toks in cases if o.encode_bytes(bytes.fromhex(h)) != toks]
    assert not bad, bad[:5]
    docs = [bytes.fromhex(h) for h, _ in cases]
    text = np.frombuffer(b"".join(docs), np.uint8)
    off = np.zeros(len(docs) + 1, np.uint64)
    off[1:] = np.cumsum([len(d) for d in docs])
    t, toff = o.encode_bytes_batch_np(text, off)
    assert [t[int(toff[i]):int(toff[i + 1])].tolist() for i in range(len(docs))] == [toks for _, toks in cases]


def test_the_reference_test_case():
    """tests/test_encoding.py:86-99 of the reference, on the synthetic cl100k stand-in: " \uc2e4" is well-formed and one
    piece, so the unstable piece is the whole input."""
    pat, ranks, special, _ = vu.load_encoding("cl100k_base", allow_real=False)
    o = Oracle(ranks, special, pat)
    b = b" \xec\x8b\xa4\xed"
    assert valid_up_to(b) == 4
    assert BytesOracle(o, ranks).encode_bytes(b) == o.encode_single_piece(b)


def _valid_up_to_python(docs: list[bytes]) -> np.ndarray:
    """UnicodeDecodeError.start of the strict decoder for every document, in one decode: the documents are joined by NUL
    (a NUL never continues a sequence), decoded with surrogateescape, and the first escaped byte of each document is
    its first ill-formed byte."""
    blob = b"\x00".join(docs) + b"\x00"
    s = blob.decode("utf-8", "surrogateescape")
    cp = np.frombuffer(s.encode("utf-32-le", "surrogatepass"), np.uint32)
    esc = (cp >= 0xDC80) & (cp <= 0xDCFF)
    width = np.where(esc, 1, np.where(cp < 0x80, 1, np.where(cp < 0x800, 2, np.where(cp < 0x10000, 3, 4))))
    pos = np.concatenate([[0], np.cumsum(width)[:-1]])
    bad = np.zeros(len(blob), bool)
    bad[pos[esc]] = True
    starts = np.zeros(len(docs), np.int64)
    lens = np.fromiter((len(d) for d in docs), np.int64, len(docs))
    starts[1:] = np.cumsum(lens + 1)[:-1]
    idx = np.flatnonzero(bad)
    owner = np.searchsorted(starts, idx, side="right") - 1
    keep = idx - starts[owner] < lens[owner]
    idx, owner = idx[keep], owner[keep]
    first_pos = np.full(len(docs), np.iinfo(np.int64).max)
    np.minimum.at(first_pos, owner, idx - starts[owner])
    return np.where(first_pos == np.iinfo(np.int64).max, lens, first_pos)


def _device_valid_up_to(hostcheck, docs: list[bytes]) -> np.ndarray:
    hostcheck.hc_utf8_valid_up_to.argtypes = [C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
    blob = b"".join(docs)
    text = np.frombuffer(blob + b"\x00" * 64, np.uint8)
    off = np.zeros(len(docs) + 1, np.uint64)
    off[1:] = np.cumsum(np.fromiter((len(d) for d in docs), np.uint64, len(docs)))
    out = np.zeros(len(docs), np.uint64)
    assert hostcheck.hc_utf8_valid_up_to(text.ctypes.data, len(blob), off.ctypes.data, len(docs), out.ctypes.data) == 0
    return out.astype(np.int64)


def _check(hostcheck, docs):
    exp = _valid_up_to_python(docs)
    got = _device_valid_up_to(hostcheck, docs)
    diff = np.flatnonzero(exp != got)
    assert len(diff) == 0, [(docs[i].hex(), int(exp[i]), int(got[i])) for i in diff[:8]]


def test_python_decoder_reduction_is_the_strict_decoder():
    rnd = random.Random(3)
    docs = [bytes(rnd.randrange(256) for _ in range(rnd.randint(0, 9))) for _ in range(3000)]
    exp = []
    for d in docs:
        try:
            d.decode("utf-8")
            exp.append(len(d))
        except UnicodeDecodeError as e:
            exp.append(e.start)
    assert _valid_up_to_python(docs).tolist() == exp
    assert [valid_up_to(d) for d in docs] == exp


@pytest.mark.parametrize("n", [1, 2, 3])
def test_classifier_every_sequence_of_n_bytes(hostcheck, n):
    """Every byte string of 1, 2 and 3 bytes, each its own document, packed back to back: sequences that would continue
    across a document start must not."""
    grid = np.stack(np.meshgrid(*[np.arange(256, dtype=np.uint8)] * n, indexing="ij"), -1).reshape(-1, n)
    raw = grid.tobytes()
    docs = [raw[i * n:(i + 1) * n] for i in range(len(grid))]
    _check(hostcheck, docs)


def test_classifier_random_strings_and_positions(hostcheck):
    """Random 4..8-byte strings from lead / continuation / ASCII heavy alphabets, then long documents with the damage
    at every offset of a 32-byte span and across span seams."""
    rnd = random.Random(11)
    alph = list(range(0x80, 0xC0)) + [0xC0, 0xC1, 0xC2, 0xDF, 0xE0, 0xE1, 0xED, 0xEF, 0xF0, 0xF1, 0xF4, 0xF5, 0xFF, 0x41]
    docs = [bytes(rnd.choice(alph) for _ in range(rnd.randint(4, 8))) for _ in range(200_000)]
    _check(hostcheck, docs)
    good = "aé中😀".encode()
    long_docs = []
    for k in range(3000):
        body = (good * 20)[:rnd.randint(0, 90)]
        body = body.decode("utf-8", "ignore").encode()
        bad = bytes(rnd.choice(alph) for _ in range(rnd.randint(0, 4)))
        long_docs.append(body + bad + (good * 3)[:rnd.randint(0, 12)])
    _check(hostcheck, long_docs)
    _check(hostcheck, [b"", b"\xe2", b"", b"\x82\xac", b"a" * 63 + b"\xf0\x9f\x98\x80", b"\xf0\x9f\x98\x80" * 40 + b"\xf0"])


# ---------------------------------------------------------------- shim and Encoding on a stub of the library
class BytesStub(StubLib):
    repairs = 0

    def b200bpe_encode_bytes_batch(self, h, text, doc_off, n_docs, out):
        oracle, _, dec = self.engines[h.value]
        o = BytesOracle(oracle, {b: i for i, b in dec.items()})
        docs = self._docs(text, doc_off, n_docs)
        toks, offs = [], [0]
        for d in docs:
            t = o.encode_bytes(d)
            if 0xFFFFFFFF in t:
                return -5
            toks.extend(t)
            offs.append(len(toks))
        self.repairs = sum(valid_up_to(d) < len(d) for d in docs)
        return self._new_result(out, np.asarray(toks, np.uint32), offs)

    def b200bpe_last_bytes_repairs(self, h, n):
        n._obj.value = self.repairs
        return 0


@pytest.fixture()
def enc(monkeypatch):
    import __graft_entry__  # noqa: F401  (sys.path)
    from tiktoken_b200 import _lib, core
    stub = BytesStub()
    monkeypatch.setattr(_lib, "lib", lambda: stub)
    monkeypatch.setattr(_lib, "last_error", lambda: "stub error")
    pat, ranks, special, _ = vu.load_encoding("cl100k_base", allow_real=False)
    return (core.Encoding("stub_cl100k", pat_str=pat, mergeable_ranks=ranks, special_tokens=special),
            BytesOracle(Oracle(ranks, special, pat), ranks))


def test_encoding_bytes_methods(enc):
    e, o = enc
    docs = [b"hello world", b"", b"caf\xc3", b"a.\n\n\xff", "日本".encode() + b"\xe6", b"<|endoftext|>\xff"]
    assert e.encode_bytes_batch(docs) == [o.encode_bytes(d) for d in docs]
    assert e._core_bpe.last_bytes_repairs() == 4
    text = np.frombuffer(b"".join(docs), np.uint8)
    off = np.zeros(len(docs) + 1, np.uint64)
    off[1:] = np.cumsum([len(d) for d in docs])
    with e.encode_bytes_packed(text, off) as buf:
        t, toff = buf.tokens(), buf.offsets()
        assert [t[int(toff[i]):int(toff[i + 1])].tolist() for i in range(len(docs))] == [o.encode_bytes(d) for d in docs]
    assert e.encode_bytes_batch([]) == []
    assert e.encode_bytes_batch([b"plain text"]) == [e.encode_ordinary("plain text")]
    assert e._core_bpe.last_bytes_repairs() == 0


@pytest.mark.parametrize("enc,pat_id", [("cl100k_base", 1), ("r50k_base", 0), ("o200k_base", 2)])
def test_prefix_pieces_with_ill_formed_tails_in_a_packed_batch(hostcheck, golden, enc, pat_id):
    """Run 1 pre-tokenises the packed batch with a haystack start at every document's first ill-formed byte.  The piece
    starts of every well-formed prefix must be the oracle's split of that prefix alone, even where the ill-formed tail
    of the document before ends in a truncated lead byte (its class must not spill into the next document: the
    pre-tokeniser's bytes-mode variant stops it there)."""
    hostcheck.hc_piece_starts_fast_cut.argtypes = [C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    pat, ranks, special, _ = vu.load_encoding(enc, allow_real=False)
    o = Oracle(ranks, special, pat)
    docs = [bytes.fromhex(h) for h, _ in golden[enc]] * 2
    blob = b"".join(docs)
    bounds, exp, check, base = [0], np.zeros(len(blob) + 1, np.uint8), np.zeros(len(blob) + 1, bool), 0
    for b in docs:
        v = valid_up_to(b)
        if 0 < v < len(b):
            bounds.append(base + v)
        p = base
        for piece in o.split(b[:v]):
            exp[p] = 1
            p += len(piece)
        check[base:base + v] = True
        base += len(b)
        bounds.append(base)
    bounds = np.unique(np.asarray(bounds, np.uint64))
    text = np.frombuffer(blob + b"\x00" * 64, np.uint8)
    got = np.zeros(len(blob) + 1, np.uint8)
    assert hostcheck.hc_piece_starts_fast_cut(pat_id, text.ctypes.data, len(blob), bounds.ctypes.data, len(bounds) - 1,
                                              got.ctypes.data, None) == 0
    assert int(((got != exp) & check).sum()) == 0
