"""Bytes mode on the GPU (b200bpe_encode_bytes_batch): documents that need not be UTF-8, bit-exact against the
restatement of the reference's `_encode_bytes` (src/py.rs:72-115) in bytes_oracle.py, for all four synthetic encodings.

Every damaged case also asserts CoreBPE.last_bytes_repairs(), so that no case passes because the repair path was never
reached; every all-valid case asserts that it was not."""
import json
import os
import random

import numpy as np
import pytest

import regrow_inputs as ri
import vocab_util as vu
from bytes_oracle import BytesOracle, RANK_MAX, valid_up_to
from oracle import Oracle
from test_gpu_paths import _chunked_encoding, _same
from tools import corpus

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ENCODINGS = ["cl100k_base", "r50k_base", "p50k_base", "o200k_base"]
KIND = {"cl100k_base": corpus.ENGLISH, "r50k_base": corpus.ENGLISH, "p50k_base": corpus.CODE, "o200k_base": corpus.MIXED}
# one ill-formed sequence of every class of the contract
INVALID = [b"\xff", b"\x80", b"\xbf", b"\xc0\xaf", b"\xc1\xbf", b"\xe0\x80\x80", b"\xed\xa0\x80", b"\xed\xbf\xbf",
           b"\xf4\x90\x80\x80", b"\xf5\x80", b"\xf8", b"\xe2\x82", b"\xf0\x9f\x98", b"\xc3"]
_CACHE = {}


def _engine(enc):
    if enc not in _CACHE:
        import tiktoken_b200
        pat, ranks, special, _ = vu.load_encoding(enc, allow_real=False)
        _CACHE[enc] = (tiktoken_b200.Encoding(f"bytes_{enc}", pat_str=pat, mergeable_ranks=ranks, special_tokens=special),
                       BytesOracle(Oracle(ranks, special, pat), ranks))
    return _CACHE[enc]


def _pack(docs):
    text = np.frombuffer(b"".join(docs), np.uint8) if any(docs) else np.zeros(0, np.uint8)
    off = np.zeros(len(docs) + 1, np.uint64)
    off[1:] = np.cumsum([len(d) for d in docs])
    return text, off


def _damaged(text, off):
    return sum(valid_up_to(text[int(off[i]):int(off[i + 1])].tobytes()) < int(off[i + 1] - off[i])
               for i in range(len(off) - 1))


def _check(e, o, text, off, repairs=None):
    exp_t, exp_o = o.encode_bytes_batch_np(text, off)
    assert _same(e.encode_bytes_packed(text, off), exp_t, exp_o)
    want = _damaged(text, off) if repairs is None else repairs
    assert e._core_bpe.last_bytes_repairs() == want
    return want


def _corpus_docs(enc, seed, nbytes, doc_bytes):
    text, off = corpus.docs_fixed(corpus.generate(KIND[enc], seed, nbytes), doc_bytes, at_space=True)
    return [text[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(off) - 1)]


def _damage(docs, rng, share):
    """A share of the documents damaged in the ways the contract lists, the common one (truncated mid-scalar at the
    end) most often."""
    out = []
    for d in docs:
        if rng.random() >= share:
            out.append(d)
            continue
        k = rng.randrange(7)
        cut = rng.randrange(len(d) + 1)
        if k <= 1:                                   # truncated mid-scalar at the end
            out.append(d + rng.choice([b"\xe2\x82", b"\xc3", b"\xf0\x9f\x98", b"\xe6\x97"]))
        elif k == 2:                                 # a stray 0xFF mid-document
            out.append(d[:cut] + b"\xff" + d[cut:])
        elif k == 3:                                 # one of every invalid class, valid text after it
            out.append(d[:cut] + rng.choice(INVALID) + d[cut:])
        elif k == 4:                                 # invalid at byte 0
            out.append(rng.choice(INVALID) + d)
        elif k == 5:                                 # an all-space last piece
            out.append(d + rng.choice([b"  ", b"\n\n", b" \t\n ", b"\n \n", b"\t"]) + rng.choice(INVALID))
        else:                                        # the damage cuts a scalar of the text itself
            e = d.decode("utf-8", "ignore").encode()
            out.append(e[:cut] + b"\xe4\xb8" + e[cut:] if cut < len(e) else e + b"\xe4")
    return out


@pytest.mark.parametrize("enc", ENCODINGS)
def test_golden_cases(enc):
    """The committed outputs of the real engine, as one batch and one document per call."""
    e, o = _engine(enc)
    with open(os.path.join(HERE, "golden", "encode_bytes.json")) as f:
        cases = json.load(f)[enc]
    docs = [bytes.fromhex(h) for h, _ in cases]
    text, off = _pack(docs)
    n = _check(e, o, text, off)
    assert n > 300
    with e.encode_bytes_packed(text, off) as buf:
        t, toff = buf.tokens(), buf.offsets()
        assert [t[int(toff[i]):int(toff[i + 1])].tolist() for i in range(len(docs))] == [tk for _, tk in cases]
    assert e.encode_bytes_batch(docs[:40]) == [tk for _, tk in cases[:40]]


@pytest.mark.parametrize("enc", ENCODINGS)
def test_damaged_corpora(enc):
    e, o = _engine(enc)
    rng = random.Random(ENCODINGS.index(enc))
    docs = _damage(_corpus_docs(enc, 5, 3 << 20, 4096), rng, 0.3)
    text, off = _pack(docs)
    assert _check(e, o, text, off) > 100


@pytest.mark.parametrize("enc", ENCODINGS)
def test_traps(enc):
    """The all-space run before the last piece may end inside an earlier piece (cl100k's ".\\n\\n" is one piece, tokenised
    [".", "\\n\\n"]); "\\r" is not all-space; special-token text is ordinary text; text after the first ill-formed byte,
    valid or not, belongs to the one unstable piece."""
    e, o = _engine(enc)
    docs = [b"end.\n\n\xff", b"end.\n\n\n\xe4\xb8", b"a.\n\n  \n\t\xff", b"x .\n\n \xc3", b"line\r\n\xff", b"a\r\n\r\n\xe2\x82",
            b"\r\n \xff", b"hello <|endoftext|>\xff", b"<|endoftext|><|endoftext|>\xc3", b"<|fim_prefix|> \n\xff",
            b"\xff valid text after the damage, \xe2\x82\xac and more", b"word\xed\xa0\x80 tail", b"  \n\n\t \xff",
            b"\n\n\n\n\n\n\xff", b"\xff", b"\xc3\xa9\xc3", b"123456\xff789", b"don't\xffs"]
    text, off = _pack(docs)
    assert _check(e, o, text, off) == len(docs)


def _cls(n):
    for c, hi in enumerate([32, 64, 128, 256, 1024, 4096, 32768]):
        if n <= hi:
            return c
    return 7


@pytest.mark.parametrize("enc", ["cl100k_base", "o200k_base"])
def test_unstable_piece_in_every_length_class(enc):
    """One document per length class whose unstable piece has that length (an ill-formed first byte: the piece is the
    whole document); last_piece_classes() shows each class merged exactly once."""
    e, o = _engine(enc)
    rng = np.random.default_rng(3)
    lens = [9, 16, 30, 60, 100, 200, 700, 3000, 20000, 150_000]
    alphabet = np.frombuffer(b"abcdefghij klmn.\n\xc3\xa9\xff", np.uint8)
    docs = [b"\xff" + rng.choice(alphabet, n - 1).tobytes() for n in lens]
    text, off = _pack(docs)
    _check(e, o, text, off, len(docs))
    counts = e._core_bpe.last_piece_classes()["counts"]
    want = [0] * 8
    for n in lens:
        if n > 16:
            want[_cls(n)] += 1
    assert counts == want


def test_missing_single_byte_raises_key_error():
    import tiktoken_b200
    pat, ranks, special, _ = vu.load_encoding("cl100k_base", allow_real=False)
    ranks = {k: v for k, v in ranks.items() if k != b"\xfe"}
    e = tiktoken_b200.Encoding("no_fe", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)
    o = BytesOracle(Oracle(ranks, special, pat), ranks)
    assert o.encode_bytes(b"\xfe") == [RANK_MAX]                   # where the reference raises
    with pytest.raises(KeyError):
        e.encode_bytes_batch([b"fine", b"\xfe"])
    assert e._core_bpe.last_bytes_repairs() == 0
    text, off = _pack([b"fine", b"ok \xff"])
    _check(e, o, text, off, 1)


def test_chunk_seams():
    """1 MiB chunks: damaged documents on both sides of every seam, pinned and pageable input."""
    e, o, _ = _chunked_encoding("cl100k_base", 1)
    o = BytesOracle(o, vu.load_encoding("cl100k_base", allow_real=False)[1])
    rng = random.Random(9)
    docs = _damage(_corpus_docs("cl100k_base", 7, 6 << 20, 60_000), rng, 0.5)
    docs += [b"\xff" + bytes(rng.randrange(256) for _ in range(300_000))]        # a 300 KB unstable piece in its own chunk
    text, off = _pack(docs)
    n = _check(e, o, text, off)
    assert n > 20
    _check(e, o, text.copy(), off, n)


def test_multi_gpu():
    from tiktoken_b200 import _lib
    ndev = int(_lib.lib().b200bpe_device_count())
    if ndev < 2:
        pytest.skip("needs at least two CUDA devices")
    e, o, _ = _chunked_encoding("cl100k_base", 1, devices=list(range(min(ndev, 4))))
    o = BytesOracle(o, vu.load_encoding("cl100k_base", allow_real=False)[1])
    docs = _damage(_corpus_docs("cl100k_base", 8, 8 << 20, 50_000), random.Random(4), 0.5)
    text, off = _pack(docs)
    assert _check(e, o, text, off) > 20


@pytest.mark.parametrize("name", ["miss", "slow", "long", "tokens"])
def test_damaged_batch_that_overflows_a_capacity(name):
    """Inputs that overflow one work-space each (regrow_inputs.py), every document damaged: run 1 grows and re-runs,
    and the result is still bit-exact."""
    import tiktoken_b200
    gen, vocab, exceeds = ri.RECIPES[name]
    text, off = gen()
    pat, ranks, sp = ri.vocabulary(vocab)
    e = tiktoken_b200.Encoding(f"bytes_regrow_{name}", pat_str=pat, mergeable_ranks=ranks, special_tokens=sp)
    o = BytesOracle(Oracle(ranks, sp, pat), ranks)
    docs = [text[int(off[i]):int(off[i + 1])].tobytes() + b"\xc3" for i in range(len(off) - 1)]
    t2, o2 = _pack(docs)
    _check(e, o, t2, o2, len(docs))
    r = e._core_bpe.last_reruns()
    want = {ri.GROWS[k] for k in exceeds} - {None}
    assert want <= r["grown"], r
    if "tokens" in exceeds:
        assert r["token_passes"] == 2


@pytest.mark.parametrize("enc", ENCODINGS)
def test_all_valid_batch_is_the_ordinary_path(enc):
    e, _ = _engine(enc)
    text, off = corpus.docs_fixed(corpus.generate(KIND[enc], 11, 4 << 20), 30_000, at_space=False)
    with e.encode_ordinary_packed(text, off) as a:
        exp_t, exp_o = np.array(a.tokens()), np.array(a.offsets())
    assert _same(e.encode_bytes_packed(text, off), exp_t, exp_o)
    assert e._core_bpe.last_bytes_repairs() == 0


@pytest.mark.parametrize("enc", ENCODINGS)
def test_round_trip_of_random_bytes(enc):
    """The reference's property (tests/test_encoding.py:93-99): decode_bytes(_encode_bytes(b)) == b."""
    e, o = _engine(enc)
    rng = np.random.default_rng(21)
    docs = [rng.integers(0, 256, int(n), dtype=np.uint8).tobytes() for n in rng.integers(0, 200, 3000)]
    docs += ["héllo wörld ".encode() * 5 + rng.integers(0, 256, 7, dtype=np.uint8).tobytes() for _ in range(200)]
    text, off = _pack(docs)
    _check(e, o, text, off)
    with e.encode_bytes_packed(text, off) as buf:
        data, boff = e.decode_packed(np.array(buf.tokens()), np.array(buf.offsets()))
    assert np.array_equal(boff, off) and data.tobytes() == text.tobytes()
