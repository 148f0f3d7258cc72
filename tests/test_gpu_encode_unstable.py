"""Completion search on the GPU (b200bpe_encode_with_unstable_batch): every case compares exactly, as lists, against the
restatement of the reference's `encode_with_unstable` in unstable_oracle.py, and asserts CoreBPE.last_unstable() so that
no case passes because the targeted path was never reached."""
import json
import os
import random

import numpy as np
import pytest

import merge_class_inputs as mci
import vocab_util as vu
from bytes_oracle import BytesOracle
from oracle import Oracle
from test_gpu_paths import _chunked_encoding
from tools import corpus
from unstable_oracle import UnstableOracle

pytestmark = pytest.mark.gpu
HERE = os.path.dirname(os.path.abspath(__file__))
ENCODINGS = ["cl100k_base", "r50k_base", "p50k_base", "o200k_base"]
KIND = {"cl100k_base": corpus.ENGLISH, "r50k_base": corpus.ENGLISH, "p50k_base": corpus.CODE, "o200k_base": corpus.MIXED}
WHITE = ["\t", "\n", "\x0b", "\x0c", "\r", " ", "\x85", "\xa0", "\u1680", "\u2000", "\u2005", "\u200a", "\u2028",
         "\u2029", "\u202f", "\u205f", "\u3000"]
_CACHE = {}


def _engine(enc):
    if enc not in _CACHE:
        import tiktoken_b200
        pat, ranks, special, _ = vu.load_encoding(enc, allow_real=False)
        o = Oracle(ranks, special, pat)
        _CACHE[enc] = (tiktoken_b200.Encoding(f"unstable_{enc}", pat_str=pat, mergeable_ranks=ranks, special_tokens=special),
                       UnstableOracle(o, ranks, special), o, ranks, special)
    return _CACHE[enc]


def _check(e, uo, texts, allowed=frozenset()):
    got = e.encode_with_unstable_batch(texts, allowed_special=set(allowed), disallowed_special=())
    st = e._core_bpe.last_unstable()
    memo = {}
    for t in texts:                                      # the restatement once per distinct text
        if t not in memo:
            memo[t] = uo.encode_with_unstable(t, allowed)
    for t, g in zip(texts, got):
        assert g[0] == memo[t][0], ("stable", t)
        assert g[1] == memo[t][1], ("completions", t)
    assert len(got) == len(texts)
    assert st["docs"] == sum(1 for t in texts if memo[t][0] != uo.o.encode(t, allowed))
    assert st["completions"] == sum(len(memo[t][1]) for t in texts)
    return st, got


def _traps(special):
    sp = sorted(special)[0]
    return ([""] + [sp, "hello " + sp, sp + " world", "a" + sp + "b c", ".\n\n", "x.\n\n", "  \n\n", "end \n \t",
                    "hello fanta", "The quick brown fox jumps", "def f():\n    ", "naïve é", "日本語のテキスト", "emoji 😀",
                    "café", "x €", "12345", "3.14159", "don't", "we'LL", "it's", "a" * 40, " " * 40, "\n" * 9]
            + ["word" + w for w in WHITE] + [w for w in WHITE] + ["x" + w + w for w in WHITE]), sp


@pytest.mark.parametrize("enc", ENCODINGS)
def test_traps_one_batch_and_one_per_call(enc):
    e, uo, _, _, special = _engine(enc)
    texts, sp = _traps(special)
    st, _ = _check(e, uo, texts, {sp})
    assert st["encoded"] > 0 and st["bpe_candidates"] > 0 and st["rounds"] >= 1
    for t in texts[:12] + texts[-6:]:
        _check(e, uo, [t], {sp})


@pytest.mark.parametrize("enc", ENCODINGS)
def test_golden_fixture(enc):
    """The wheel's cases (tests/golden/make_unstable_golden.py): the batch per allowed-special set, and one call per case."""
    import hashlib
    with open(os.path.join(HERE, "golden", "encode_with_unstable.json")) as f:
        cases = json.load(f)[enc]
    e, uo, _, _, _ = _engine(enc)
    groups = {}
    for c in cases:
        groups.setdefault(tuple(c[1]), []).append(c)
    for allowed, group in groups.items():
        _, got = _check(e, uo, [c[0] for c in group], frozenset(allowed))
        for (_, _, stable_exp, n, dig), (stable, comps) in zip(group, got):
            assert stable == stable_exp and len(comps) == n
            assert hashlib.sha256(json.dumps(sorted(comps)).encode()).hexdigest()[:16] == dig
    for c in cases[::7]:
        _check(e, uo, [c[0]], frozenset(c[1]))


def _cut_prompts(enc, seed, n):
    rnd = random.Random(seed)
    text = corpus.generate(KIND[enc], seed, 400_000).tobytes().decode("utf-8", "ignore")
    out = []
    for _ in range(n):
        a = rnd.randrange(0, len(text) - 200)
        out.append(text[a:a + rnd.randrange(0, 120)])        # str slices: cuts at scalar boundaries
    return out


@pytest.mark.parametrize("enc", ENCODINGS)
def test_corpus_prompts(enc):
    e, uo, _, _, _ = _engine(enc)
    texts = _cut_prompts(enc, 7, 2000)
    st, _ = _check(e, uo, texts)
    assert st["docs"] > 1500 and st["encoded"] > 10_000
    # core.py:229-230: decode(stable) is a prefix of the text, decode(stable + seq) starts with it
    got = e.encode_with_unstable_batch(texts[:300], disallowed_special=())
    for t, (stable, comps) in zip(texts, got):
        b = t.encode()
        assert b.startswith(e.decode_bytes(stable))
        assert all(e.decode_bytes(stable + s).startswith(b) for s in comps)


def test_disallowed_special_raises():
    e, _, _, _, special = _engine("cl100k_base")
    sp = sorted(special)[0]
    with pytest.raises(ValueError, match="disallowed special token"):
        e.encode_with_unstable_batch(["ok", "x " + sp])
    with pytest.raises(UnicodeEncodeError):
        e.encode_with_unstable_batch(["a\ud800"])


def _tiny_vocab(missing=None):
    ranks = mci.base_vocab(3)
    top = max(ranks.values()) + 1
    # tokens that their own merges do not reach: byte_pair_encode differs from probe-then-merge on them
    for i, t in enumerate([b"\x82\xac\x82", b"\xe2\x82\xac\x82", b" !!!", b"!!!\n"]):
        ranks[t] = top + i
    if missing is not None:
        del ranks[missing]
    return vu.CL100K_PAT, ranks, {"<|endoftext|>": 1 << 20}


def test_unreachable_tokens_take_byte_pair_encode():
    import tiktoken_b200
    pat, ranks, special = _tiny_vocab()
    e = tiktoken_b200.Encoding("unreach", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)
    uo = UnstableOracle(Oracle(ranks, special, pat), ranks, special)
    texts = ["€", "x €", "x !!!\n", "abcd !!!\n", "dcba !!!\t", "ab€", " !!!"]
    st, _ = _check(e, uo, texts)
    assert st["bpe_candidates"] > 0
    exp = uo.encode_with_unstable("x !!!\n")[1]
    assert [ranks[b" "], ranks[b"!"], ranks[b"!"], ranks[b"!"], ranks[b"\n"]] in exp


def test_missing_single_byte_raises_key_error():
    import tiktoken_b200
    pat, ranks, special = _tiny_vocab(missing=b"!")
    e = tiktoken_b200.Encoding("nobyte", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)
    with pytest.raises(KeyError):
        e.encode_with_unstable_batch(["ok !!\n"])


def test_rounds_and_chunk_seams():
    """1 MiB chunks: rounds of at most 1 MiB of candidate text and 32 Ki candidates; one prompt's candidates span rounds."""
    e = _chunked_encoding("cl100k_base", 1)[0]
    _, uo, _, _, _ = _engine("cl100k_base")
    st, _ = _check(e, uo, ["def f():\n    ", "x" + " " * 300, "word " + "abc" * 100, "tail \n\n"])
    assert st["rounds"] > 1
    many = _cut_prompts("cl100k_base", 11, 2000) + ["word " * 60 + "end"] * 6000   # > 1.5 MiB: several chunks
    st, _ = _check(e, uo, many)
    assert st["rounds"] >= 3


def test_multi_gpu():
    import torch
    if torch.cuda.device_count() < 2:
        pytest.skip("needs two GPUs")
    e = _chunked_encoding("o200k_base", 1, devices=[0, 1])[0]
    _, uo, _, _, _ = _engine("o200k_base")
    _check(e, uo, _cut_prompts("o200k_base", 5, 1000) + ["word " * 60 + "end"] * 6000)


def test_other_paths_after_unstable_call():
    e, uo, o, ranks, special = _engine("p50k_base")
    texts = _cut_prompts("p50k_base", 3, 500)
    _check(e, uo, texts)
    assert e.encode_ordinary_batch(texts) == [o.encode_ordinary(t) for t in texts]
    bo = BytesOracle(o, ranks)
    docs = [t.encode()[:-1] for t in texts if len(t.encode()) > 1]
    assert e.encode_bytes_batch(docs) == [bo.encode_bytes(d) for d in docs]
    assert e._core_bpe.last_unstable()["docs"] == 0


def test_packed_matches_lists():
    e, uo, _, _, _ = _engine("o200k_base")
    texts = _cut_prompts("o200k_base", 9, 200) + [""]
    blob = "".join(texts).encode()
    off = np.zeros(len(texts) + 1, np.uint64)
    off[1:] = np.cumsum([len(t.encode()) for t in texts])
    st, so, ct, co, grp = e.encode_with_unstable_packed(np.frombuffer(blob, np.uint8), off, disallowed_special=())
    got = e.encode_with_unstable_batch(texts, disallowed_special=())
    for d, (stable, comps) in enumerate(got):
        assert st[so[d]:so[d + 1]].tolist() == stable
        assert [ct[co[q]:co[q + 1]].tolist() for q in range(int(grp[d]), int(grp[d + 1]))] == comps
    assert e.encode_with_unstable_batch([], disallowed_special=()) == []
