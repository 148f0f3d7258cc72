"""Documents larger than a chunk: the host path cuts them at seams (doc_seams.h) so that they chunk, pipeline and shard
like a batch, and the tokens stay those of the whole document.  Every comparison is bit-exact against the oracle in
full, and each test asserts CoreBPE.last_doc_seams() so that no case passes because nothing was cut."""
import os

import numpy as np
import pytest

import vocab_util as vu
from test_doc_seams_cpu import rule
from test_gpu_paths import _chunked_encoding
from tools import corpus

pytestmark = pytest.mark.gpu
CORES = os.cpu_count() or 1
MiB = 1 << 20


def _lead(text, p):
    """p moved back onto a UTF-8 lead byte."""
    while 0 < p < len(text) and (text[p] & 0xC0) == 0x80:
        p -= 1
    return p


def _check(e, o, text, off, want_seams=True):
    off = np.ascontiguousarray(off, np.uint64)
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, CORES)
    with e.encode_ordinary_packed(text, off) as buf:
        assert np.array_equal(buf.tokens(), exp_t) and np.array_equal(buf.offsets(), exp_o)
    s = e._core_bpe.last_doc_seams()
    assert (s["seams"] > 0) == want_seams, s
    assert np.array_equal(e.count_packed(text, off), exp_o)
    assert e._core_bpe.last_doc_seams() == s
    return s


@pytest.mark.parametrize("enc,kind,mib", [("cl100k_base", corpus.ENGLISH, 8), ("o200k_base", corpus.MIXED, 12),
                                          ("p50k_base", corpus.CODE, 16), ("r50k_base", corpus.ENGLISH, 24)])
def test_one_long_document_1mib_chunks(enc, kind, mib):
    e, o, _ = _chunked_encoding(enc, 1)
    text = corpus.generate(kind, 31, mib * MiB)
    s = _check(e, o, text, [0, len(text)])
    assert s["docs_cut"] == 1 and s["seams"] >= mib // 2


@pytest.mark.parametrize("enc,kind", [("cl100k_base", corpus.ENGLISH), ("o200k_base", corpus.MIXED)])
def test_mixed_batch_of_short_and_long_documents(enc, kind):
    e, o, _ = _chunked_encoding(enc, 1)
    text = corpus.generate(kind, 32, 12 * MiB)
    n = len(text)
    marks = [0, 10, 10, 700, 3000, 3 * MiB + 7, 3 * MiB + 9, 3 * MiB + 9, 5 * MiB, 5 * MiB + 40_000, 9 * MiB, n - 100, n, n]
    off = np.asarray([_lead(text, m) for m in marks], np.uint64)
    s = _check(e, o, text, off)
    assert s["docs_cut"] >= 3
    # small documents around the long ones, many per chunk
    off2 = np.concatenate([np.arange(0, 2 * MiB, 5000), [6 * MiB], np.arange(6 * MiB + 1, 8 * MiB, 70_000), [n]])
    off2 = np.asarray([_lead(text, int(m)) for m in off2], np.uint64)
    assert _check(e, o, text, off2)["docs_cut"] >= 2


def test_allowed_specials_next_to_seams_and_the_leftmost_disallowed():
    e, o, special = _chunked_encoding("cl100k_base", 1)
    words = corpus.generate(corpus.ENGLISH, 33, 3 * MiB).tobytes().decode()
    pieces, step = [], 40_000
    for i, lo in enumerate(range(0, len(words), step)):
        chunk = words[lo:lo + step]
        sp = "<|endoftext|>" if i % 2 else "<|endofprompt|>"
        pieces.append(chunk + (sp + "\nNext " if i % 3 else " " + sp + " and"))
    doc = "".join(pieces)
    allowed = {"<|endoftext|>", "<|endofprompt|>"}
    b = np.frombuffer(doc.encode(), np.uint8)
    off = np.asarray([0, len(b)], np.uint64)
    exp = np.asarray(o.encode(doc, allowed_special=allowed), np.uint32)
    with e.encode_packed(b, off, allowed_special=allowed) as buf:
        assert np.array_equal(buf.tokens(), exp)
    assert e._core_bpe.last_doc_seams()["seams"] > 0
    assert e.count_packed(b, off, allowed_special=allowed)[-1] == len(exp)
    # two disallowed specials behind the first seam: the leftmost one is reported, by encode and count alike
    at1, at2 = _lead(b, int(1.6 * MiB)), _lead(b, int(2.4 * MiB))
    bad = (b[:at1].tobytes() + b"<|fim_suffix|>" + b[at1:at2].tobytes() + b"<|fim_prefix|>" + b[at2:].tobytes())
    bb = np.frombuffer(bad, np.uint8)
    off = np.asarray([0, len(bb)], np.uint64)
    for call in (e.encode_packed, e.count_packed):
        with pytest.raises(ValueError, match=r"disallowed special token '<\|fim_suffix\|>'"):
            call(bb, off, allowed_special=allowed)


def test_document_without_seams_is_one_chunk():
    e, o, _ = _chunked_encoding("o200k_base", 1)
    text = np.frombuffer(("中文字符。数据、" * 150_000).encode(), np.uint8)
    assert _check(e, o, text, [0, len(text)], want_seams=False) == {"seams": 0, "docs_cut": 0}


def test_bytes_mode_and_completion_search_keep_documents_whole():
    e, o, _ = _chunked_encoding("cl100k_base", 1)
    text = corpus.generate(corpus.ENGLISH, 34, 3 * MiB)
    off = np.asarray([0, 100, len(text)], np.uint64)
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, CORES)
    with e.encode_bytes_packed(text, off) as buf:
        assert np.array_equal(buf.tokens(), exp_t) and np.array_equal(buf.offsets(), exp_o)
    assert e._core_bpe.last_doc_seams() == {"seams": 0, "docs_cut": 0}
    got = e.encode_with_unstable_packed(text, off)
    assert e._core_bpe.last_doc_seams() == {"seams": 0, "docs_cut": 0}
    # the same call with every document inside one chunk
    e64, _, _ = _chunked_encoding("cl100k_base", 64)
    want = e64.encode_with_unstable_packed(text, off)
    assert all(np.array_equal(a, b) for a, b in zip(got, want))
    st_t, st_o = got[0], got[1]
    for d in range(2):
        assert np.array_equal(st_t[int(st_o[d]):int(st_o[d + 1])], exp_t[int(exp_o[d]):int(exp_o[d]) + int(st_o[d + 1] - st_o[d])])


def test_one_long_document_on_two_devices():
    from tiktoken_b200 import _lib
    if _lib.lib().b200bpe_device_count() < 2:
        pytest.skip("needs two visible GPUs")
    e, o, _ = _chunked_encoding("cl100k_base", 1, devices=[0, 1])
    text = corpus.generate(corpus.ENGLISH, 35, 16 * MiB)
    assert _check(e, o, text, [0, len(text)])["docs_cut"] == 1


def _available_host_bytes():
    with open("/proc/meminfo") as f:
        for line in f:
            if line.startswith("MemAvailable:"):
                return int(line.split()[1]) * 1024
    return 0


def test_document_over_4gib():
    if _available_host_bytes() < (48 << 30):
        pytest.skip("needs 48 GiB of free host memory")
    import tiktoken_b200
    pat, ranks, special, _ = vu.load_encoding("cl100k_base", allow_real=False)
    e = tiktoken_b200.Encoding("over_4gib", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)
    n = 17 << 28                                                   # 4.25 GiB
    text = corpus.generate(corpus.ENGLISH, 36, n)
    one = np.asarray([0, n], np.uint64)
    with e.encode_ordinary_packed(text, one) as buf:
        toks = np.array(buf.tokens())
        assert buf.offsets().tolist() == [0, len(toks)]
    assert e._core_bpe.last_doc_seams()["seams"] > 0
    assert e.count_packed(text, one).tolist() == [0, len(toks)]
    # the same text as a batch cut where the rule allows, about every 512 MiB: the same tokens
    cuts = [0]
    for t in range(512 * MiB, n, 512 * MiB):
        p = t
        while not rule(text[p - 2:p + 2].tobytes(), 0, 4, 2):
            p += 1
        cuts.append(p)
    cuts.append(n)
    cuts = np.asarray(cuts, np.uint64)
    with e.encode_ordinary_packed(text, cuts) as buf:
        assert np.array_equal(buf.tokens(), toks)
        toff = np.array(buf.offsets())
    # decode(encode(x)) == x, a part at a time
    for d in range(len(cuts) - 1):
        lo, hi = int(toff[d]), int(toff[d + 1])
        data, _ = e._core_bpe.decode_batch_buffer(toks[lo:hi], np.asarray([0, hi - lo], np.uint64))
        assert np.array_equal(data, text[int(cuts[d]):int(cuts[d + 1])])
