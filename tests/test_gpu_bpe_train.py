"""BPE training on the GPU, bit-exact: against the reference's fixtures (tests/golden/bpe_train.json) in the str, batch
and packed forms, and against the C restatement (tools/train_oracle.c) on multi-MiB corpora that span several chunks."""
import json
import os

import numpy as np
import pytest

import tiktoken_b200
import train_oracle as T
from oracle import Oracle
from oracle.oracle import CL100K_PAT, O200K_PAT, R50K_PAT
from tools import corpus

pytestmark = pytest.mark.gpu

HERE = os.path.dirname(os.path.abspath(__file__))
PATS = {"r50k": R50K_PAT, "cl100k": CL100K_PAT, "o200k": O200K_PAT}
with open(os.path.join(HERE, "golden", "bpe_train.json"), encoding="utf-8") as f:
    GOLDEN = json.load(f)["cases"]


def expected(case) -> list:
    ranks = {bytes([i]): i for i in range(256)}
    ranks.update((bytes.fromhex(k), v) for k, v in case["ranks"])
    return list(ranks.items())


def pack(docs):
    enc = [d.encode("utf-8") if isinstance(d, str) else d for d in docs]
    blob = b"".join(enc)
    off = np.zeros(len(enc) + 1, np.uint64)
    off[1:] = np.cumsum([len(b) for b in enc])
    return (np.frombuffer(blob, np.uint8) if blob else np.zeros(0, np.uint8)), off


@pytest.mark.parametrize("form", ["str", "batch", "packed"])
@pytest.mark.parametrize("case", GOLDEN, ids=[c["name"] for c in GOLDEN])
def test_fixture(case, form):
    pat, text, vocab = PATS[case["pat"]], case["text"], case["vocab_size"]

    def run():
        if form == "str":
            return tiktoken_b200.bpe_train(text, vocab, pat)
        if form == "batch":
            return tiktoken_b200.bpe_train_batch([text], vocab, pat)
        return tiktoken_b200.bpe_train_packed(*pack([text]), vocab, pat)

    if "error" in case:
        with pytest.raises(ValueError):
            run()
    else:
        assert list(run().items()) == expected(case)


def mib_corpus(p: str, nbytes: int, seed: int):
    """Documents of a tools/corpus stream for pattern p, plus empty documents, a 48 KiB letter run and a 40 KiB
    whitespace run (each one piece) and a short tail."""
    kind = {"r50k": corpus.CODE, "cl100k": corpus.ENGLISH, "o200k": corpus.MIXED}[p]
    raw = corpus.generate(kind, seed, nbytes).tobytes().decode("utf-8", "ignore")
    rng = np.random.default_rng(seed)
    docs, i = [], 0
    while i < len(raw):
        n = int(rng.integers(1000, 200_000))
        docs.append(raw[i:i + n]); i += n
        if rng.random() < 0.2:
            docs.append("")
    mid = len(docs) // 2
    docs[mid:mid] = ["q" * (48 << 10), "", "\t" * (40 << 10), " x"]
    return docs


@pytest.mark.parametrize("p", ["r50k", "cl100k", "o200k"])
def test_multi_mib_against_restatement(p, monkeypatch):
    monkeypatch.setenv("B200BPE_CHUNK_MB", "1")
    docs = mib_corpus(p, 3 << 20, 100 + len(p))
    text, off = pack(docs)
    vocab = 256 + 1200
    merges, n_distinct = T.train_merges(PATS[p], text, off, vocab)
    want = list(T.ranks_from_merges(merges).items())
    assert list(tiktoken_b200.bpe_train_packed(text, off, vocab, PATS[p]).items()) == want
    st = tiktoken_b200.last_train_stats()
    assert st["chunks"] >= 3 and st["distinct_words"] == n_distinct and st["merges"] == len(merges)
    assert list(tiktoken_b200.bpe_train_batch(docs, vocab, PATS[p]).items()) == want


def test_thousands_of_merges_several_graph_batches():
    text, off = corpus.config2(nbytes=2 << 20, seed=77, doc_bytes=32768)
    vocab = 256 + 5000
    merges, _ = T.train_merges(CL100K_PAT, text, off, vocab)
    got = tiktoken_b200.bpe_train_packed(text, off, vocab, CL100K_PAT)
    assert list(got.items()) == list(T.ranks_from_merges(merges).items())
    st = tiktoken_b200.last_train_stats()
    assert st["merges"] == 5000 and st["graph_batches"] >= 5000 / 128


def test_no_pair_left_raises_after_the_last_merge():
    text, off = pack(["abab ab", "", "ab"])
    merges, _ = T.train_merges(CL100K_PAT, text, off, 258)
    assert list(tiktoken_b200.bpe_train_packed(text, off, 258, CL100K_PAT).items()) == list(T.ranks_from_merges(merges).items())
    with pytest.raises(ValueError):
        tiktoken_b200.bpe_train_packed(text, off, 300, CL100K_PAT)
    with pytest.raises(ValueError):
        tiktoken_b200.bpe_train_batch(["", ""], 257, CL100K_PAT)
    assert list(tiktoken_b200.bpe_train_batch(["", ""], 256, CL100K_PAT).items()) == [(bytes([i]), i) for i in range(256)]


def test_trained_vocabulary_encodes_its_corpus():
    text, off = corpus.config2(nbytes=1 << 20, seed=5, doc_bytes=16384)
    ranks = tiktoken_b200.bpe_train_packed(text, off, 256 + 2000, CL100K_PAT)
    assert sorted(ranks.values()) == list(range(len(ranks)))
    enc = tiktoken_b200.Encoding("trained", pat_str=CL100K_PAT, mergeable_ranks=ranks, special_tokens={}, device=0)
    buf = enc.encode_ordinary_packed(text, off)
    exp_t, exp_o = Oracle(ranks, {}, CL100K_PAT).encode_ordinary_batch_np(text, off, os.cpu_count() or 1)
    assert np.array_equal(buf.tokens(), exp_t) and np.array_equal(buf.offsets(), exp_o)
    assert enc.decode_bytes(buf.tokens()) == text.tobytes()
    assert len(exp_t) < len(text) / 2
    buf.close()


def test_engine_encodes_the_same_after_training():
    import vocab_util as vu
    pat, ranks, special, _ = vu.load_encoding("cl100k_base", allow_real=False)
    enc = tiktoken_b200.Encoding("before", pat_str=pat, mergeable_ranks=ranks, special_tokens=special, device=0)
    text, off = corpus.config2(nbytes=1 << 20, seed=9)
    before = enc.encode_ordinary_packed(text, off)
    t0, o0 = before.tokens().copy(), before.offsets().copy()
    before.close()
    tiktoken_b200.bpe_train_packed(text, off, 256 + 500, pat)
    after = enc.encode_ordinary_packed(text, off)
    assert np.array_equal(after.tokens(), t0) and np.array_equal(after.offsets(), o0)
    after.close()
