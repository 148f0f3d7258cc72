"""The per-call miss memo: every distinct missed piece is merged once and its other occurrences copy the result.

Every case is bit-exact against the oracle and asserts CoreBPE.last_miss_memo() against counts taken on the CPU from
the oracle's split: `misses` = pieces of up to 16 bytes that are not tokens (a single byte only when the vocabulary
lacks it), and `merged` = one per distinct piece of up
to 15 bytes plus every 16-byte piece, give or take the pieces the memo could not place
(distinct + n16 <= merged <= distinct + n16 + unplaced, with equality when nothing was unplaced)."""
import os
import random

import numpy as np
import pytest

import vocab_util as vu
from test_gpu_paths import _chunked_encoding, _same
from tools import corpus
from tools.miss_memo_bench import distinct_miss_corpus

pytestmark = pytest.mark.gpu
CORES = os.cpu_count() or 1
BIG_MEMO = 1 << 22          # over ten times more slots than distinct misses: (almost) nothing is unplaced


def _missed(o, ranks, docs):
    """The missed pieces of a batch, one entry per occurrence (documents are separate haystacks)."""
    return [pc for d in docs for pc in o.split(d) if len(pc) <= 16 and pc not in ranks]


def _docs(text, off):
    return [text[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(off) - 1)]


def _check_memo(e, missed, exact):
    m = e._core_bpe.last_miss_memo()
    n16 = sum(len(pc) == 16 for pc in missed)
    distinct = len({pc for pc in missed if len(pc) < 16})
    assert m["misses"] == len(missed), m
    assert distinct + n16 <= m["merged"] <= distinct + n16 + m["unplaced"], (m, distinct, n16)
    if exact:
        assert m["unplaced"] == 0 and m["merged"] == distinct + n16, (m, distinct, n16)
    return m


def test_config2_like_text_merges_each_distinct_piece_once():
    text, off = corpus.config2(nbytes=32 << 20, seed=1002)
    e, o, _ = _chunked_encoding("cl100k_base", 64, B200BPE_MISS_MEMO_SLOTS=BIG_MEMO)
    ranks = vu.load_encoding("cl100k_base", allow_real=False)[1]
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, CORES)
    missed = _missed(o, ranks, _docs(text, off))
    assert _same(e.encode_ordinary_packed(text, off), exp_t, exp_o)
    m = _check_memo(e, missed, exact=True)
    assert m["merged"] * 3 < m["misses"], m
    # the default size (one slot per 128 bytes) and the memo off give the same tokens
    d, _, _ = _chunked_encoding("cl100k_base", 64)
    assert _same(d.encode_ordinary_packed(text, off), exp_t, exp_o)
    m = _check_memo(d, missed, exact=False)
    assert m["merged"] < m["misses"], m
    f, _, _ = _chunked_encoding("cl100k_base", 64, B200BPE_MISS_MEMO_SLOTS=0)
    assert _same(f.encode_ordinary_packed(text, off), exp_t, exp_o)
    assert f._core_bpe.last_miss_memo() == {"misses": len(missed), "merged": len(missed), "unplaced": 0}
    # trim() releases the memo with the other work-spaces; the next call allocates it again
    e._core_bpe.trim()
    assert _same(e.encode_ordinary_packed(text, off), exp_t, exp_o)
    _check_memo(e, missed, exact=True)


def test_every_missed_piece_distinct():
    text, off = distinct_miss_corpus(4 << 20, seed=11)
    e, o, _ = _chunked_encoding("cl100k_base", 64, B200BPE_MISS_MEMO_SLOTS=BIG_MEMO)
    ranks = vu.load_encoding("cl100k_base", allow_real=False)[1]
    missed = _missed(o, ranks, _docs(text, off))
    assert len(set(missed)) == len(missed) > 300_000
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, CORES)
    assert _same(e.encode_ordinary_packed(text, off), exp_t, exp_o)
    m = _check_memo(e, missed, exact=False)     # 335 k keys at load 0.08: a few may find 4 full slots
    assert m["merged"] == m["misses"]


def test_more_distinct_misses_than_slots_are_unplaced():
    text, off = distinct_miss_corpus(1 << 20, seed=12)
    e, o, _ = _chunked_encoding("cl100k_base", 64, B200BPE_MISS_MEMO_SLOTS=64)
    ranks = vu.load_encoding("cl100k_base", allow_real=False)[1]
    missed = _missed(o, ranks, _docs(text, off))
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, CORES)
    assert _same(e.encode_ordinary_packed(text, off), exp_t, exp_o)
    m = _check_memo(e, missed, exact=False)
    assert m["unplaced"] >= len(missed) - 64 and m["merged"] == m["misses"], m


def _edge_docs(rnd):
    """Repeated pieces across sub-tiles and documents, NUL-padded look-alikes, 15- and 16-byte misses, and merges that
    end as 2, 3 and more than 3 tokens."""
    letters = "qzxjvkwy"
    words = [" " + "".join(rnd.choice(letters) for _ in range(n)) for n in (1, 2, 3, 5, 8, 11, 13, 14, 15)]
    nul = ["!" + "\0" * k for k in range(1, 15)] + [" \0" * k for k in range(1, 8)] + ["\0" + "qz" * k for k in range(1, 8)]
    docs = []
    for d in range(60):
        parts = [rnd.choice(words + nul) for _ in range(rnd.randrange(1, 900))]
        docs.append("".join(parts))
    return docs + ["", "!\0", "!\0\0", " \0", "\0qz"]


def test_edge_keys_host_and_device_paths():
    import torch
    rnd = random.Random(21)
    docs = _edge_docs(rnd)
    e, o, _ = _chunked_encoding("cl100k_base", 64, B200BPE_MISS_MEMO_SLOTS=BIG_MEMO)
    ranks = vu.load_encoding("cl100k_base", allow_real=False)[1]
    missed = _missed(o, ranks, docs)
    lens = {len(pc) for pc in missed}
    assert {15, 16} <= lens and any(b"\0" in pc for pc in missed)
    ntok = {len(o.encode_single_piece(pc)) for pc in set(missed)}
    assert 2 in ntok and 3 in ntok and max(ntok) > 3, ntok
    exp = [o.encode_ordinary(d) for d in docs]
    assert e.encode_ordinary_batch(docs) == exp
    _check_memo(e, missed, exact=True)
    # device-resident, one call and a queued series (the counters describe the last call)
    blob = "".join(docs).encode()
    off = np.cumsum([0] + [len(d.encode()) for d in docs]).astype(np.uint64)
    text = np.frombuffer(blob, np.uint8).copy()
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, CORES)
    core = e._core_bpe
    d_text = torch.from_numpy(text).cuda(); d_off = torch.from_numpy(off.astype(np.int64)).cuda()
    d_tok = torch.empty(len(text) + 16, dtype=torch.int32, device="cuda"); d_toff = torch.empty(len(off), dtype=torch.int64, device="cuda")
    s = torch.cuda.Stream()
    n = core.encode_device(d_text.data_ptr(), len(text), d_off.data_ptr(), len(off) - 1, d_tok.data_ptr(), d_toff.data_ptr(), s.cuda_stream)
    s.synchronize()
    assert n == len(exp_t) and np.array_equal(d_tok[:n].cpu().numpy().view(np.uint32), exp_t)
    assert np.array_equal(d_toff.cpu().numpy().astype(np.uint64), exp_o)
    _check_memo(e, missed, exact=True)
    half = len(docs) // 2
    sets, counts = [], torch.zeros((2, 2), dtype=torch.int64, device="cuda")
    for k, part in enumerate((docs[:half], docs[half:])):
        b = "".join(part).encode()
        po = np.cumsum([0] + [len(x.encode()) for x in part]).astype(np.uint64)
        pt = np.frombuffer(b, np.uint8).copy()
        sets.append((pt, po, torch.from_numpy(pt).cuda(), torch.from_numpy(po.astype(np.int64)).cuda(),
                     torch.empty(len(pt) + 16, dtype=torch.int32, device="cuda"), torch.empty(len(po), dtype=torch.int64, device="cuda")))
    s.synchronize()
    for k, (pt, po, dt, do, dk, dko) in enumerate(sets):
        core.encode_device_async(dt.data_ptr(), len(pt), do.data_ptr(), len(po) - 1, dk.data_ptr(), dko.data_ptr(),
                                 counts[k].data_ptr(), s.cuda_stream)
    core.device_wait()
    s.synchronize()
    for k, (pt, po, dt, do, dk, dko) in enumerate(sets):
        et, eo = o.encode_ordinary_batch_np(pt, po, CORES)
        assert int(counts[k, 0]) == len(et) and np.array_equal(dk[:len(et)].cpu().numpy().view(np.uint32), et)
        assert np.array_equal(dko.cpu().numpy().astype(np.uint64), eo)
    _check_memo(e, _missed(o, ranks, docs[half:]), exact=True)


def test_1mib_chunks():
    """Misses and merges summed over chunks; one memo per chunk, so a piece is merged once per chunk it occurs in."""
    e, o, _ = _chunked_encoding("cl100k_base", 1, B200BPE_MISS_MEMO_SLOTS=BIG_MEMO)
    ranks = vu.load_encoding("cl100k_base", allow_real=False)[1]
    text, off = corpus.config2(nbytes=6 << 20, seed=31, doc_bytes=100_000)
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, CORES)
    assert _same(e.encode_ordinary_packed(text, off), exp_t, exp_o)
    docs = _docs(text, off)
    m = e._core_bpe.last_miss_memo()
    missed = _missed(o, ranks, docs)
    assert m["misses"] == len(missed) and m["unplaced"] == 0
    # per chunk: the documents of each ~1 MiB chunk (b200bpe.cu cuts at the last document boundary within a chunk)
    chunk, lo, merged = 1 << 20, 0, 0
    while lo < len(docs):
        hi = int(np.searchsorted(off, off[lo] + chunk, side="right")) - 1
        hi = min(max(hi, lo + 1), len(docs))
        part = _missed(o, ranks, docs[lo:hi])
        merged += len({pc for pc in part if len(pc) < 16}) + sum(len(pc) == 16 for pc in part)
        lo = hi
    assert m["merged"] == merged < m["misses"], (m, merged)


def test_bytes_mode_and_allowed_specials():
    e, o, special = _chunked_encoding("cl100k_base", 64, B200BPE_MISS_MEMO_SLOTS=BIG_MEMO)
    ranks = vu.load_encoding("cl100k_base", allow_real=False)[1]
    text, off = corpus.config2(nbytes=2 << 20, seed=41, doc_bytes=20_000)
    docs = _docs(text, off)
    damaged = [d[:len(d) // 2] + b"\xff" + d[len(d) // 2:] if i % 7 == 3 else d for i, d in enumerate(docs)]
    from bytes_oracle import BytesOracle
    bo = BytesOracle(o, ranks)
    assert e.encode_bytes_batch(damaged) == [bo.encode_bytes(d) for d in damaged]
    m = e._core_bpe.last_miss_memo()
    assert 0 < m["merged"] < m["misses"] and m["unplaced"] == 0, m
    names = sorted(special)
    rnd = random.Random(5)
    sdocs = []
    for d in docs[:60]:
        s = d.decode()
        cut = sorted(rnd.sample(range(len(s)), 10))
        sdocs.append("".join(s[a:b] + rnd.choice(names) for a, b in zip([0] + cut, cut)) + s[cut[-1]:])
    assert e.encode_batch(sdocs, allowed_special="all") == [o.encode(d, set(special)) for d in sdocs]
    m = e._core_bpe.last_miss_memo()
    assert 0 < m["merged"] < m["misses"] and m["unplaced"] == 0, m


def test_missing_single_byte_raises_with_the_memo():
    pat, ranks, special = vu.load_encoding("cl100k_base", allow_real=False)[:3]
    ranks = {k: v for k, v in ranks.items() if b"\x01" not in k}
    e, o, _ = _chunked_encoding("cl100k_base", 64, vocab=(pat, ranks, special), B200BPE_MISS_MEMO_SLOTS=BIG_MEMO)
    docs = ["hello world! \x01\x01 again"] * 200 + ["plain text"]
    with pytest.raises(KeyError):
        e.encode_ordinary_batch(docs)
    assert e.encode_ordinary_batch(docs[-1:]) == [o.encode_ordinary(docs[-1])]


def test_multi_gpu_engine():
    from tiktoken_b200 import _lib
    ndev = int(_lib.lib().b200bpe_device_count())
    if ndev < 2:
        pytest.skip("needs at least two CUDA devices")
    e, o, _ = _chunked_encoding("cl100k_base", 8, devices=list(range(min(ndev, 4))), B200BPE_MISS_MEMO_SLOTS=BIG_MEMO)
    ranks = vu.load_encoding("cl100k_base", allow_real=False)[1]
    text, off = corpus.config2(nbytes=32 << 20, seed=51)
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, CORES)
    assert _same(e.encode_ordinary_packed(text, off), exp_t, exp_o)
    m = e._core_bpe.last_miss_memo()
    assert m["misses"] == len(_missed(o, ranks, _docs(text, off))) and 0 < m["merged"] < m["misses"], m
