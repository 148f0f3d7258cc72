"""Parity tests proper: the CUDA engine, called through the C ABI (ctypes shim), against
(1) the committed golden vectors generated from the reference engine, (2) the oracle on seeded
inputs, (3) size-independent properties at larger sizes.  Bit-exact: integer/byte work."""
import json
import os
import pickle

import numpy as np
import pytest

import vocab_util as vu
from conftest import have_gpu
from tools import corpus

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden")
ENCS = [("cl100k_base", corpus.ENGLISH), ("r50k_base", corpus.ENGLISH), ("p50k_base", corpus.CODE),
        ("o200k_base", corpus.MIXED)]
_cache = {}


def get(enc):
    if enc not in _cache:
        import tiktoken_b200
        from oracle import Oracle
        pat, ranks, special, src = vu.load_encoding(enc, allow_real=False)
        e = tiktoken_b200.Encoding(enc + "_syn", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)
        _cache[enc] = (e, Oracle(ranks, special, pat), special)
    return _cache[enc]


@pytest.mark.parametrize("enc,kind", ENCS)
def test_golden_vectors_from_reference_engine(enc, kind):
    e, _, special = get(enc)
    gold = np.load(os.path.join(G, f"tokens_{enc}.npz"))
    text = corpus.generate(kind, 31337, 96 << 10).tobytes().decode("utf-8")
    assert e.encode_ordinary(text) == gold["corpus"].tolist()
    edge = json.load(open(os.path.join(G, "edge_texts.json")))["edge"]
    assert e.encode_ordinary_batch(edge) == [gold[f"edge_{i}"].tolist() for i in range(len(edge))]
    got = e.encode_batch(edge, allowed_special="all")
    assert got == [gold[f"edge_special_{i}"].tolist() for i in range(len(edge))]


def test_reference_adversarial_bpe_vectors_through_single_piece():
    import tiktoken_b200
    vocs = json.load(open(os.path.join(G, "bpe_adversarial.json")))[:40]
    for voc in vocs:
        ranks = {bytes([i]): i for i in range(256)}
        ranks.update({k.encode(): v for k, v in voc["extra"].items()})
        e = tiktoken_b200.Encoding("adv", pat_str=vu.R50K_PAT, mergeable_ranks=ranks, special_tokens={})
        for piece, expected in voc["cases"]:
            assert e._encode_single_piece(piece) == expected, (piece, voc["extra"])


@pytest.mark.parametrize("enc,kind", ENCS)
def test_against_oracle_on_seeded_corpus(enc, kind):
    e, o, _ = get(enc)
    text = corpus.generate(kind, 4242, 3 << 20)
    for off in (corpus.docs_fixed(text, 65536, at_space=(kind == corpus.ENGLISH))[1],
                np.asarray([0, len(text)], np.uint64)):
        buf = e.encode_ordinary_packed(text, off)
        exp_t, exp_o = o.encode_ordinary_batch_np(text, off, os.cpu_count() or 1)
        assert np.array_equal(buf.tokens(), exp_t) and np.array_equal(buf.offsets(), exp_o)
        buf.close()


def test_many_short_and_empty_documents():
    e, o, _ = get("cl100k_base")
    text, off = corpus.config4(n_docs=200_000, seed=1004)
    assert (np.diff(off.astype(np.int64)) == 0).any()
    buf = e.encode_ordinary_packed(text, off)
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, os.cpu_count() or 1)
    assert np.array_equal(buf.tokens(), exp_t) and np.array_equal(buf.offsets(), exp_o)
    buf.close()


def test_edge_shapes():
    e, o, _ = get("cl100k_base")
    assert e.encode_ordinary("") == []
    assert e.encode_ordinary_batch([]) == []
    assert e.encode_ordinary_batch(["", "", ""]) == [[], [], []]
    docs = ["x" * n for n in (1, 15, 16, 17, 31, 32, 33, 99, 100, 101, 4095, 4096, 4097, 8193, 70000)]
    docs += [" " * n for n in (1, 2, 16, 17, 64, 5000)] + ["\n" * 3000, "a\n" * 2000, "0" * 10000, "'s" * 5000]
    docs += ["^" * 10000, " " + "a" * 10000 + "\n", "日本語" * 3000, "\U0001F600‍\U0001F3FB" * 500]
    got = e.encode_ordinary_batch(docs)
    for d, g in zip(docs, got):
        assert g == o.encode_ordinary(d), d[:20]


def test_catastrophically_repetitive_roundtrip():
    # tests/test_encoding.py:113-124
    e, _, _ = get("o200k_base")
    for c in ["^", "0", "a", "'s", " ", "\n"]:
        big = c * 10_000
        for s in (big, " " + big, big + "\n"):
            assert e.decode(e.encode_ordinary(s)) == s


def test_million_x_does_not_blow_up():
    # tests/test_encoding.py:52-57 (o200k, 1_000_000 x 'x'), checked against the oracle's heap path
    e, o, _ = get("o200k_base")
    s = "x" * 1_000_000
    assert e.encode_ordinary(s) == o.encode_ordinary(s)


@pytest.mark.parametrize("enc,kind", ENCS)
def test_roundtrip_and_batch_properties_at_size(enc, kind):
    # decode(encode(t)) == t  (tests/test_encoding.py:149-155);  batch == per-document (:239-264)
    e, _, _ = get(enc)
    text = corpus.generate(kind, 777, 24 << 20)
    _, off = corpus.docs_fixed(text, 1 << 20, at_space=False)
    buf = e.encode_ordinary_packed(text, off)
    toks, toff = np.array(buf.tokens()), np.array(buf.offsets()); buf.close()
    assert e.decode_bytes(toks) == text.tobytes()
    one = e.encode_ordinary_packed(text, np.asarray([off[3], off[4]], np.uint64) - off[3]) if False else None
    d = 5
    s, t = int(off[d]), int(off[d + 1])
    single = e.encode_ordinary(text[s:t].tobytes().decode("utf-8"))
    assert toks[int(toff[d]):int(toff[d + 1])].tolist() == single
    assert int(toff[-1]) == len(toks)


def test_special_token_policy_and_slicing():
    e, o, special = get("cl100k_base")
    s = "hello <|endoftext|> a  <|fim_prefix|>b"
    with pytest.raises(ValueError):
        e.encode(s)                                              # disallowed by default (core.py:120-124)
    assert e.encode(s, disallowed_special=()) == e.encode_ordinary(s)
    assert e.encode(s, allowed_special="all") == o.encode(s, set(special))
    only = {"<|endoftext|>"}
    assert e.encode(s, allowed_special=only, disallowed_special=()) == o.encode(s, only)
    assert e.encode("<|endoftext|>", allowed_special="all") == [special["<|endoftext|>"]]
    assert e.encode_ordinary(s) == e.encode(s, disallowed_special=())      # tests/test_encoding.py:226-231
    assert e.encode_to_numpy(s, allowed_special="all").tolist() == o.encode(s, set(special))


def test_many_special_occurrences_in_a_batch():
    """Documents with thousands of allowed specials (adjacent, at both ends, overlapping look-alikes)
    while other allowed specials never occur: every haystack boundary and every spliced id must match."""
    import random
    e, o, special = get("cl100k_base")
    rnd = random.Random(9)
    names = sorted(special)
    words = ["alpha", " beta", "\n", " 42", "<|", "|>", "<|endoftext", " <|endoftext|", "x" * 40]
    docs = []
    for d in range(6):
        parts = []
        use = names if d % 2 else names[:1]
        for _ in range(3000 if d < 2 else 200):
            parts.append(rnd.choice(words) if rnd.random() < 0.7 else rnd.choice(use))
        docs.append(rnd.choice(use) + "".join(parts) + rnd.choice(use) * 2)
    docs += ["", names[0], names[0] * 3]
    got = e.encode_batch(docs, allowed_special="all")
    assert got == [o.encode(d, set(special)) for d in docs]
    only = {names[0]}
    got = e.encode_batch(docs, allowed_special=only, disallowed_special=())
    assert got == [o.encode(d, only) for d in docs]


def test_errors_and_misc_api():
    e, o, special = get("cl100k_base")
    with pytest.raises(KeyError):
        e.decode_bytes([10 ** 7])
    with pytest.raises(KeyError):
        e.encode_single_token(b"\xff\xfe not a token")
    assert e.decode_single_token_bytes(special["<|endoftext|>"]) == b"<|endoftext|>"
    for t in (0, 255, 256, 1000, 100255):
        assert e.encode_single_token(e.decode_single_token_bytes(t)) == t
    assert e.decode_with_offsets(e.encode_ordinary("hello world"))[0] == "hello world"
    assert e.encode_ordinary("\ud83d") == e.encode_ordinary("�")   # lone surrogate fix-up (core.py:77-80)
    assert e._encode_single_piece("helloqqqq") == o.encode_single_piece(b"helloqqqq")
    e2 = pickle.loads(pickle.dumps(e))
    assert e2.encode_ordinary("pickled hello") == e.encode_ordinary("pickled hello")
    assert e.n_vocab == max(special.values()) + 1 and e.is_special_token(special["<|endoftext|>"])


def test_missing_single_byte_is_an_error_not_garbage():
    import tiktoken_b200
    ranks = {bytes([i]): i for i in range(256) if i != ord("q")}
    ranks[b"qu"] = 300
    e = tiktoken_b200.Encoding("nobyte", pat_str=vu.R50K_PAT, mergeable_ranks=ranks, special_tokens={})
    assert e.encode_ordinary("quu") == [300, ord("u")]          # merging THROUGH the missing byte works
    with pytest.raises(KeyError):
        e.encode_ordinary("q")                                   # reference: index panic (lib.rs:202)


def test_device_resident_entry_point():
    import torch
    e, o, _ = get("cl100k_base")
    text, off = corpus.config2(nbytes=8 << 20, seed=1002)
    d_text = torch.from_numpy(text).cuda()
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()
    d_tok = torch.empty(len(text), dtype=torch.int32, device="cuda")
    d_toff = torch.empty(len(off), dtype=torch.int64, device="cuda")
    n = e._core_bpe.encode_device(d_text.data_ptr(), len(text), d_off.data_ptr(), len(off) - 1, d_tok.data_ptr(),
                                  d_toff.data_ptr())
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, os.cpu_count() or 1)
    assert n == len(exp_t)
    assert np.array_equal(d_tok[:n].cpu().numpy().view(np.uint32), exp_t)
    assert np.array_equal(d_toff.cpu().numpy().astype(np.uint64), exp_o)


def test_device_decode_batch_roundtrip_and_errors():
    """"next" row: CoreBPE::decode_bytes (src/lib.rs:345-358) as one device gather per batch."""
    e, o, special = get("o200k_base")
    text, off = corpus.config3(nbytes=6 << 20, seed=5)
    buf = e.encode_ordinary_packed(text, off)
    toks, toff = np.array(buf.tokens()), np.array(buf.offsets()); buf.close()
    data, boff = e.decode_packed(toks, toff)
    assert np.array_equal(data, text) and np.array_equal(boff, off)           # decode(encode(x)) == x, per document
    docs = ["hello world", "", "x" * 5000, "日本語 <|endoftext|>", "\n\n  a"]
    enc = e.encode_batch(docs, allowed_special="all")
    assert e.decode_batch(enc) == docs
    assert e.decode_bytes_batch(enc) == [e.decode_bytes(t) for t in enc]    # same as the per-call table read
    assert e.decode_bytes_batch([]) == [] and e.decode_bytes_batch([[], []]) == [b"", b""]
    with pytest.raises(KeyError):
        e.decode_bytes_batch([[1, 2, 10 ** 7]])
