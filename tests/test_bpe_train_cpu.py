"""BPE training without a GPU: the C restatement (tools/train_oracle.c) against the reference's fixtures and against the
installed `tiktoken._educational.bpe_train`, the dict rebuild of tiktoken_b200.train, and the errors raised before any
device call."""
import json
import os
import random

import numpy as np
import pytest
from tiktoken._educational import bpe_train as ref_bpe_train

import tiktoken_b200
import train_oracle as T
from oracle.oracle import CL100K_PAT, O200K_PAT, R50K_PAT
from tiktoken_b200 import train as gtrain

HERE = os.path.dirname(os.path.abspath(__file__))
PATS = {"r50k": R50K_PAT, "cl100k": CL100K_PAT, "o200k": O200K_PAT}
with open(os.path.join(HERE, "golden", "bpe_train.json"), encoding="utf-8") as f:
    GOLDEN = json.load(f)["cases"]


def expected(case) -> dict:
    ranks = {bytes([i]): i for i in range(256)}
    ranks.update((bytes.fromhex(k), v) for k, v in case["ranks"])
    return ranks


@pytest.mark.parametrize("case", GOLDEN, ids=[c["name"] for c in GOLDEN])
def test_restatement_matches_fixture(case):
    pat = PATS[case["pat"]]
    if "error" in case:
        with pytest.raises(ValueError):
            T.bpe_train(case["text"], case["vocab_size"], pat)
        return
    got = T.bpe_train(case["text"], case["vocab_size"], pat)
    assert list(got.items()) == list(expected(case).items())


@pytest.mark.parametrize("seed", range(40))
def test_restatement_matches_installed_bpe_train(seed):
    rng = random.Random(seed)
    alpha = rng.choice(["ab ", "abc \n", "aab c1'", "xy z\r\n 12", "aé 😀\t", "'s 'S don't"])
    text = "".join(rng.choice(alpha) for _ in range(rng.randint(0, 400)))
    pat = rng.choice(list(PATS.values()))
    vocab = rng.randint(256, 320)
    try:
        ref = list(ref_bpe_train(text, vocab, pat, visualise=None).items())
    except ValueError:
        ref = ValueError
    if ref is ValueError:
        with pytest.raises(ValueError):
            T.bpe_train(text, vocab, pat)
    else:
        assert list(T.bpe_train(text, vocab, pat).items()) == ref


def test_restatement_batch_is_pieces_of_each_document():
    docs = ["hello wor", "ld hello", "", "world  "]
    blob = "".join(docs).encode()
    off = np.cumsum([0] + [len(d.encode()) for d in docs]).astype(np.uint64)
    b, po = T.split_packed(CL100K_PAT, np.frombuffer(blob, np.uint8), off)
    pieces = [b[int(po[i]):int(po[i + 1])].tobytes() for i in range(len(po) - 1)]
    assert pieces == [b"hello", b" wor", b"ld", b" hello", b"world", b"  "]


def test_rebuild_reproduces_overwritten_keys():
    # merges (id 256 = "ab", 257 = "abc", 258 = "bc", then a + bc = "abc" again): the reference overwrites "abc"
    merges = np.asarray([[97, 98, 256], [256, 99, 257], [98, 99, 258], [97, 258, 257]], np.uint32)
    ranks = gtrain._ranks_from_merges(merges)
    items = list(ranks.items())[256:]
    assert items == [(b"ab", 256), (b"abc", 259), (b"bc", 258)]
    assert len(ranks) == 259
    with pytest.raises(RuntimeError):
        gtrain._ranks_from_merges(np.asarray([[97, 98, 256], [97, 98, 257]], np.uint32))
    with pytest.raises(RuntimeError):
        gtrain._ranks_from_merges(np.asarray([[97, 98, 256], [98, 99, 256]], np.uint32))


@pytest.fixture
def no_device(monkeypatch):
    def boom():
        raise AssertionError("the device was touched")
    monkeypatch.setattr(gtrain._lib, "lib", boom)


@pytest.mark.parametrize("fn", ["str", "batch", "packed"])
def test_errors_before_any_device_call(no_device, fn):
    def call(text, vocab, pat):
        if fn == "str":
            return tiktoken_b200.bpe_train(text, vocab, pat)
        if fn == "batch":
            return tiktoken_b200.bpe_train_batch([text, "x"], vocab, pat)
        b = text.encode("utf-8")
        return tiktoken_b200.bpe_train_packed(np.frombuffer(b, np.uint8), np.asarray([0, len(b)], np.uint64), vocab, pat)

    with pytest.raises(ValueError, match="vocab_size must be at least 256"):
        call("hello", 255, CL100K_PAT)
    with pytest.raises(ValueError, match="pat_str"):
        call("hello", 300, r"\w+|\s+")
    if fn != "packed":
        with pytest.raises(UnicodeEncodeError):
            call("ab\ud800cd", 300, CL100K_PAT)


def test_reference_message_for_small_vocab():
    with pytest.raises(ValueError) as ref:
        ref_bpe_train("x", 100, CL100K_PAT, visualise=None)
    with pytest.raises(ValueError) as ours:
        tiktoken_b200.bpe_train("x", 100, CL100K_PAT)
    assert str(ours.value) == str(ref.value)


def test_supported_patterns_are_the_engines():
    assert set(gtrain.SUPPORTED_PATTERNS) == set(PATS.values())
