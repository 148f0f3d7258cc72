"""What the b200bpe_last_* getters report after each kind of call, in one fixed sequence on one engine.

Every encode entry point zeroes the re-run counters, piece classes, miss memo, bytes repairs and completion figures
before it starts, and keeps the timings and launches of the call before until it has something to report.  A host
call reports the timings and launches of the runs whose output it returns; bytes mode adds the tail runs of a damaged
chunk to them, the completion search does not add its candidate runs.  A device wait reports no copies and counts the
special-token record kernel.  A failing host call keeps the call before's timings and launches.  A batch decode
overwrites the timings and launches (six launches) and nothing else.  Launches are a pure function of the input, and a
batch cut into chunks launches what its chunks launch as calls of their own."""
import numpy as np
import pytest

import vocab_util as vu
from test_gpu_paths import _chunked_encoding
from tools import corpus

pytestmark = pytest.mark.gpu
COPIES = ("h2d_ms", "d2h_ms")
PIPELINE = ("mark_docs_ms", "pretok_ms", "long_ms", "encode_ms", "gather_ms", "probe_ms")
ZERO_UNSTABLE = {"docs": 0, "encoded": 0, "bpe_candidates": 0, "rounds": 0, "completions": 0}


def _stats(e):
    c = e._core_bpe
    return {"timings": c.last_timings(), "reruns": c.last_reruns(), "classes": c.last_piece_classes(),
            "memo": c.last_miss_memo(), "repairs": c.last_bytes_repairs(), "unstable": c.last_unstable()}


def _pack(docs):
    off = np.zeros(len(docs) + 1, np.uint64)
    np.cumsum([len(d) for d in docs], out=off[1:])
    return np.frombuffer(b"".join(docs), np.uint8).copy(), off


def _host_call(s):
    """A host call that returned its output."""
    assert s["reruns"]["token_passes"] == 1
    assert s["timings"]["launches"] > 0 and s["timings"]["device_total_ms"] > 0
    assert s["memo"]["misses"] >= s["memo"]["unplaced"]


def test_call_sequence():
    import tiktoken_b200
    import torch
    pat, ranks, special, _ = vu.load_encoding("cl100k_base", allow_real=False)
    e = tiktoken_b200.Encoding("call_stats", pat_str=pat, mergeable_ranks=ranks, special_tokens=special, device=0)
    c = e._core_bpe
    sp = sorted(special)[0]
    text, off = corpus.config2(nbytes=2 << 20, seed=5)
    docs = [text[int(off[i]):int(off[i + 1])].tobytes() for i in range(len(off) - 1)]
    toks = np.asarray(c.encode_ordinary("hello world, a decode"), np.uint32)
    tok_off = np.asarray([0, len(toks)], np.uint64)

    # ordinary, twice: launches depend on the input alone
    c.encode_ordinary_batch_buffer(text, off).close()
    s_ord = _stats(e)
    _host_call(s_ord)
    assert s_ord["repairs"] == 0 and s_ord["unstable"] == ZERO_UNSTABLE and s_ord["memo"]["misses"] > 0
    c.encode_ordinary_batch_buffer(text, off).close()
    s = _stats(e)
    assert s["timings"]["launches"] == s_ord["timings"]["launches"]
    assert s["classes"] == s_ord["classes"] and s["memo"]["misses"] == s_ord["memo"]["misses"]
    assert s["reruns"] == {"grown": set(), "reruns": 0, "token_passes": 1}

    # special: the same documents with an allowed special in each; the scan adds two launches
    sp_text, sp_off = _pack([d + sp.encode() for d in docs])
    c.encode_batch_buffer(sp_text, sp_off, allowed_special={sp}).close()
    s = _stats(e)
    _host_call(s)
    assert s["repairs"] == 0 and s["unstable"] == ZERO_UNSTABLE
    assert s["timings"]["launches"] == s_ord["timings"]["launches"] + 2

    # count only: the same classes and memo as the encode of the same text, fewer launches
    c.count_batch_offsets(text, off, allowed_special=set())
    s = _stats(e)
    _host_call(s)
    assert s["classes"] == s_ord["classes"] and s["memo"]["misses"] == s_ord["memo"]["misses"]
    assert s["timings"]["launches"] < s_ord["timings"]["launches"]

    # bytes mode: clean, then the same documents with every fourth one damaged (same length, same run 1 shape)
    c.encode_bytes_batch_buffer(text, off).close()
    s_clean = _stats(e)
    _host_call(s_clean)
    assert s_clean["repairs"] == 0
    bad = [d[:len(d) // 2] + b"\xff" + d[len(d) // 2 + 1:] if i % 4 == 0 else d for i, d in enumerate(docs)]
    b_text, b_off = _pack(bad)
    assert np.array_equal(b_off, off)
    c.encode_bytes_batch_buffer(b_text, b_off).close()
    s = _stats(e)
    _host_call(s)
    assert s["repairs"] == (len(docs) + 3) // 4 and s["unstable"] == ZERO_UNSTABLE
    assert s["timings"]["launches"] > s_clean["timings"]["launches"] + 9        # run 1 + run 2 + the splice's nine
    assert s["timings"]["device_total_ms"] > 0

    # completion search: the timings and launches of run 1 (the pipeline and the walk kernel) only
    prompts = [b"hello wor", b"The quick bro", b"def f():\n    ", b"it's a ", b"x = 3.14", b"caf\xc3\xa9 "] * 50
    u_text, u_off = _pack(prompts)
    c.encode_ordinary_batch_buffer(u_text, u_off).close()
    s_run1 = _stats(e)
    stable, comp = c.encode_with_unstable_batch_buffer(u_text, u_off, allowed_special=set())
    stable.close()
    comp.close()
    s_unst = _stats(e)
    _host_call(s_unst)
    assert s_unst["repairs"] == 0
    assert s_unst["unstable"]["docs"] > 0 and s_unst["unstable"]["completions"] > 0 and s_unst["unstable"]["rounds"] > 0
    assert s_unst["timings"]["launches"] == s_run1["timings"]["launches"] + 1

    # a decode keeps everything but the timings and launches
    c.decode_batch_buffer(toks, tok_off)
    s = _stats(e)
    assert s["timings"]["launches"] == 6 and all(s["timings"][k] == 0 for k in PIPELINE)
    assert {k: v for k, v in s.items() if k != "timings"} == {k: v for k, v in s_unst.items() if k != "timings"}

    # single piece: the figures of the completion search are gone
    c.encode_single_piece(b"x" * 3000)
    s = _stats(e)
    _host_call(s)
    assert s["unstable"] == ZERO_UNSTABLE and s["repairs"] == 0

    # device calls: no copies, one pass; with a special-token policy the record kernel is one more launch
    d_text = torch.from_numpy(sp_text).cuda()
    d_off = torch.from_numpy(sp_off.astype(np.int64)).cuda()
    d_tok = torch.empty(len(sp_text), dtype=torch.int32, device="cuda")
    d_toff = torch.empty(len(sp_off), dtype=torch.int64, device="cuda")
    c.encode_batch_buffer(sp_text, sp_off, allowed_special={sp}).close()
    s_host = _stats(e)
    c.encode_device_special_async(d_text.data_ptr(), len(sp_text), d_off.data_ptr(), len(sp_off) - 1, d_tok.data_ptr(),
                                  d_toff.data_ptr(), allowed_special={sp})
    s = _stats(e)
    assert s["reruns"] == {"grown": set(), "reruns": 0, "token_passes": 0} and s["timings"] == s_host["timings"]
    c.device_wait()
    s_dev = _stats(e)
    assert s_dev["reruns"] == {"grown": set(), "reruns": 0, "token_passes": 1}
    assert all(s_dev["timings"][k] == 0 for k in COPIES) and s_dev["timings"]["device_total_ms"] > 0
    assert s_dev["timings"]["launches"] == s_host["timings"]["launches"] + 1
    assert s_dev["classes"] == s_host["classes"] and s_dev["memo"]["misses"] == s_host["memo"]["misses"]
    d_text2 = torch.from_numpy(text).cuda()
    d_off2 = torch.from_numpy(off.astype(np.int64)).cuda()
    assert c.encode_device(d_text2.data_ptr(), len(text), d_off2.data_ptr(), len(off) - 1, d_tok.data_ptr(),
                           d_toff.data_ptr()) > 0
    s_dev = _stats(e)
    assert s_dev["timings"]["launches"] == s_ord["timings"]["launches"]
    assert s_dev["classes"] == s_ord["classes"] and s_dev["memo"]["misses"] == s_ord["memo"]["misses"]

    # a failing call: the timings and launches of the call before, zeros for what it would have returned
    with pytest.raises(ValueError):
        c.encode_batch_buffer(sp_text, sp_off, allowed_special=set(), disallowed_special={sp})
    s_fail = _stats(e)
    assert s_fail["timings"] == s_dev["timings"]
    assert s_fail["reruns"] == {"grown": set(), "reruns": 0, "token_passes": 1}
    assert s_fail["classes"]["counts"] == [0] * 8 and s_fail["memo"] == {"misses": 0, "merged": 0, "unplaced": 0}
    assert s_fail["repairs"] == 0 and s_fail["unstable"] == ZERO_UNSTABLE

    # decode last: its own timings, the failing call's zeros kept
    c.decode_batch_buffer(toks, tok_off)
    s = _stats(e)
    assert s["timings"]["launches"] == 6 and all(s["timings"][k] == 0 for k in PIPELINE)
    assert {k: v for k, v in s.items() if k != "timings"} == {k: v for k, v in s_fail.items() if k != "timings"}


def _chunk_plan(off, chunk):
    """Document ranges of the host path's chunks (b200bpe.cu chunk_plan)."""
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


def test_chunked_launches_are_the_sum_of_their_chunks():
    e, _, _ = _chunked_encoding("cl100k_base", 1)
    text, off = corpus.config2(nbytes=(7 << 20) // 2, seed=9, doc_bytes=200_000)
    cut = _chunk_plan(off, 1 << 20)
    assert len(cut) > 3
    e._core_bpe.encode_ordinary_batch_buffer(text, off).close()
    whole = e._core_bpe.last_timings()["launches"]
    parts = 0
    for lo, hi in zip(cut[:-1], cut[1:]):
        t = text[int(off[lo]):int(off[hi])]
        o = (off[lo:hi + 1] - off[lo]).astype(np.uint64)
        e._core_bpe.encode_ordinary_batch_buffer(t, o).close()
        parts += e._core_bpe.last_timings()["launches"]
    assert whole == parts
