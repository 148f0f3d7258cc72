"""Every grow-and-re-run path of the encoder, bit-exact against the oracle.

The miss queue, the miss result space, the list of undecided pre-tokeniser positions and the long-piece merge scratch
are sized from experience; when one is too small the kernels flag it, the host grows it to the exact need and runs the
same chunk again.  The host token buffer is sized per call and gets a second pass when it is too small.  The inputs
of regrow_inputs.py overflow one of them each (test_regrow_inputs.py checks that on the CPU).  Every case here:
  1. a fresh engine, so the work-spaces are at their first-run sizes;
  2. all tokens and per-document offsets against the oracle;
  3. CoreBPE.last_reruns() names exactly the work-spaces that grew (or the second token pass), so that no case passes
     merely because nothing overflowed;
  4. the same call again: the same output and no re-run; after trim() the capacities are back at their first-run
     sizes and the call re-runs again.
The token buffer comes from the engine's pool of pinned blocks, which trim() empties; whether a repeated call gets a
block large enough to skip the second token pass is the pool's business, so only the first call and the call after
trim() pin the pass count of an input that overflows the token buffer."""
import os
import random

import numpy as np
import pytest

import regrow_inputs as ri
from test_gpu_paths import _chunked_encoding, _same

pytestmark = pytest.mark.gpu
CORES = os.cpu_count() or 1
NONE = {"grown": set(), "reruns": 0, "token_passes": 1}


def _fresh(vocab, special=None):
    import tiktoken_b200
    from oracle import Oracle
    pat, ranks, sp = ri.vocabulary(vocab)
    sp = sp if special is None else special
    return (tiktoken_b200.Encoding(f"regrow_{vocab}", pat_str=pat, mergeable_ranks=ranks, special_tokens=sp),
            Oracle(ranks, sp, pat))


RERUNS_PER_CHUNK = 4        # b200bpe.cu: a chunk that still overflows after 4 re-runs fails ("sizing did not converge")


def _expect(e, grown, passes, what, chunks=1):
    """passes: the exact token pass count, or a set of allowed ones.  A chunk re-runs at most RERUNS_PER_CHUNK times in
    each token pass."""
    r = e._core_bpe.last_reruns()
    assert r["grown"] == grown and r["token_passes"] in (passes if isinstance(passes, set) else {passes}), (what, r)
    if grown:
        assert 1 <= r["reruns"] <= RERUNS_PER_CHUNK * chunks * r["token_passes"], (what, r)
    else:
        assert r["reruns"] == 0, (what, r)


def _intended(exceeds):
    return {ri.GROWS[k] for k in exceeds} - {None}, 2 if "tokens" in exceeds else 1


def _three_calls(e, call, grown, passes, chunks=1):
    """call() encodes and checks the output; first call, repeated call, call after trim().  The first call and the call
    after trim() find the engine's pinned pool empty, so their pass-0 token buffer is the first-run size.  A repeated
    call may be given a larger pooled block, so an input that needs a second pass on its first call may or may not need
    it again; an input that fits the first-run size always fits."""
    call()
    _expect(e, grown, passes, "first call", chunks)
    call()
    _expect(e, set(), {1, 2} if passes == 2 else 1, "repeated call", chunks)
    e._core_bpe.trim()
    call()
    _expect(e, grown, passes, "after trim", chunks)


@pytest.mark.parametrize("name", sorted(ri.RECIPES))
def test_host_path_regrows(name):
    """encode_ordinary_packed on pageable memory, one chunk."""
    gen, vocab, exceeds = ri.RECIPES[name]
    text, off = gen()
    e, o = _fresh(vocab)
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, CORES)
    grown, passes = _intended(exceeds)
    _three_calls(e, lambda: _check_host(e, text, off, exp_t, exp_o), grown, passes)


def _check_host(e, text, off, exp_t, exp_o):
    assert _same(e.encode_ordinary_packed(text, off), exp_t, exp_o)


@pytest.mark.parametrize("name", sorted(n for n in ri.RECIPES if n != "tokens"))
def test_device_path_regrows(name):
    """The device-resident encode_device (the caller sizes d_tokens, so the token buffer does not apply)."""
    import torch
    gen, vocab, exceeds = ri.RECIPES[name]
    text, off = gen()
    e, o = _fresh(vocab)
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, CORES)
    d_text = torch.from_numpy(text).cuda()
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()
    d_tok = torch.empty(len(text), dtype=torch.int32, device="cuda")
    d_toff = torch.empty(len(off), dtype=torch.int64, device="cuda")

    def call():
        d_tok.fill_(-1)                                   # nothing of an earlier call can pass for this one's output
        d_toff.fill_(-1)
        torch.cuda.synchronize()
        n = e._core_bpe.encode_device(d_text.data_ptr(), len(text), d_off.data_ptr(), len(off) - 1, d_tok.data_ptr(),
                                      d_toff.data_ptr())
        assert n == len(exp_t)
        assert np.array_equal(d_tok[:n].cpu().numpy().view(np.uint32), exp_t)
        assert np.array_equal(d_toff.cpu().numpy().astype(np.uint64), exp_o)

    grown, passes = _intended(exceeds)
    assert passes == 1
    _three_calls(e, call, grown, passes)


@pytest.mark.parametrize("variant", ["plain", "multi_gpu"])
def test_batch_of_all_recipes_in_1mib_chunks(variant):
    """MISS, SLOW, LONG and TOKENS documents interleaved, 1 MiB chunks: every pipeline slot overflows on its first
    chunk while the other slots have uploads and kernels in flight, slots re-run with other causes later, and the
    whole batch overflows the pass-0 token buffer, so the second pass runs across all chunks (and devices).
    Variants: as is; the one-process multi-GPU engine."""
    devices = None
    if variant == "multi_gpu":
        from tiktoken_b200 import _lib
        ndev = int(_lib.lib().b200bpe_device_count())
        if ndev < 2:
            pytest.skip("needs at least two CUDA devices")
        devices = list(range(min(ndev, 8)))
    text, off, kinds = ri.batch()
    e, o, _ = _chunked_encoding("regrow_batch", 1, vocab=ri.vocabulary(ri.BATCH_VOCAB), devices=devices)
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, CORES)
    assert len(exp_t) > ri.caps(len(text))["tokens"]
    # every document is one chunk (test_regrow_inputs.py checks that)
    _three_calls(e, lambda: _check_host(e, text, off, exp_t, exp_o), {"miss", "slow", "long"}, 2, chunks=len(kinds))


def test_single_piece_over_1mib():
    """encode_single_piece of 1.5 MiB of {a..h} on miss_vocab: the piece overflows the 1 MiB scratch floor and, with
    few merges, leaves more tokens than the pass-0 buffer holds."""
    rnd = random.Random(7)
    piece = "".join(rnd.choice("abcdefgh") for _ in range(3 << 19)).encode()
    e, o = _fresh("miss")
    exp = o.encode_single_piece(piece)
    assert len(exp) > ri.caps(len(piece))["tokens"]

    def call():
        assert e._encode_single_piece(piece) == exp

    _three_calls(e, call, {"long"}, 2)


def _special_docs(special_name, disallowed=None):
    """MISS and SLOW text on miss_vocab (digit runs miss there too), allowed specials every few thousand bytes; the
    disallowed special, if any, near the end of the last document, after everything that overflows."""
    rnd = random.Random(11)
    texts = [ri.miss(5, 200_000)[0].tobytes().decode(), ri.slow(5, 320_000)[0].tobytes().decode()]
    docs = []
    for t in texts:
        for k in range(3):
            s = t[k * len(t) // 3:(k + 1) * len(t) // 3]
            cuts = sorted(rnd.sample(range(len(s)), len(s) // 3000))
            parts, prev = [], 0
            for c in cuts:
                parts += [s[prev:c], special_name]
                prev = c
            docs.append("".join(parts) + s[prev:])
    if disallowed:
        docs[-1] = docs[-1][:-100] + disallowed + docs[-1][-100:]
    return docs


def test_special_tokens_in_overflowing_text():
    base = len(ri.miss_vocab())
    special = {"<|endoftext|>": base, "<|fim_prefix|>": base + 1}
    e, o = _fresh("miss", special)
    docs = _special_docs("<|endoftext|>")
    exp = [o.encode(d, {"<|endoftext|>"}) for d in docs]
    n_bytes = sum(len(d) for d in docs)
    assert sum(map(len, exp)) > ri.caps(n_bytes)["tokens"]

    def call():
        assert e.encode_batch(docs, allowed_special="all") == exp

    _three_calls(e, call, {"miss", "slow"}, 2)
    # a disallowed special after the overflowing text: ERR_SPECIAL is checked before the capacity flags, so the call
    # fails with the reference's ValueError and re-runs nothing
    e2, _ = _fresh("miss", special)
    bad = _special_docs("<|endoftext|>", disallowed="<|fim_prefix|>")
    with pytest.raises(ValueError, match="disallowed special token '<\\|fim_prefix\\|>'"):
        e2.encode_batch(bad, allowed_special={"<|endoftext|>"})
    assert e2._core_bpe.last_reruns() == NONE


@pytest.mark.parametrize("overflowing", ["first", "last"])
def test_queued_device_calls_with_an_overflowing_one(overflowing):
    """Three encode_device_async calls on one stream, one of them overflowing the miss queue of a fresh engine: the
    wait fails with the "work-space had to grow" error.  One synchronous call of the overflowing input settles the
    sizes, and the same series queued again succeeds, every call's tokens, offsets and counts row exact."""
    import torch
    from tools import corpus
    e, o = _fresh("miss")
    core = e._core_bpe
    inputs = [ri.miss(3, 400_000, 20_000)]
    for k in range(2):                                     # small English: inside every first-run capacity
        t = corpus.generate(corpus.ENGLISH, 60 + k, 48 << 10)
        inputs.append((t, corpus.docs_fixed(t, 4096, at_space=True)[1]))
    if overflowing == "last":
        inputs = inputs[1:] + inputs[:1]
    big = 0 if overflowing == "first" else 2
    expected = [o.encode_ordinary_batch_np(t, off, CORES) for t, off in inputs]
    stream = torch.cuda.Stream()
    sets = []
    for t, off in inputs:
        sets.append((torch.from_numpy(t).cuda(), torch.from_numpy(off.astype(np.int64)).cuda(),
                     torch.empty(len(t), dtype=torch.int32, device="cuda"),
                     torch.empty(len(off), dtype=torch.int64, device="cuda")))
    counts = torch.zeros((3, 2), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()

    def queue():
        for k, (t, off) in enumerate(inputs):
            d_text, d_off, d_tok, d_toff = sets[k]
            core.encode_device_async(d_text.data_ptr(), len(t), d_off.data_ptr(), len(off) - 1, d_tok.data_ptr(),
                                     d_toff.data_ptr(), counts[k].data_ptr(), stream.cuda_stream)
        return core.device_wait()

    with pytest.raises(RuntimeError, match="work-space had to grow"):
        queue()
    # the wait re-runs the last call when that one overflowed; an earlier one is only reported
    _expect(e, {"miss"} if overflowing == "last" else set(), 1, "failed series")
    t, off = inputs[big]
    d_text, d_off, d_tok, d_toff = sets[big]
    n = core.encode_device(d_text.data_ptr(), len(t), d_off.data_ptr(), len(off) - 1, d_tok.data_ptr(),
                           d_toff.data_ptr(), stream.cuda_stream)
    assert n == len(expected[big][0])
    _expect(e, {"miss"} if overflowing == "first" else set(), 1, "synchronous call")
    for s in sets:
        s[2].fill_(-1)
        s[3].fill_(-1)
    counts.fill_(-1)
    torch.cuda.synchronize()
    n_last = queue()
    assert core.last_reruns() == NONE
    stream.synchronize()
    for k, (t, off) in enumerate(inputs):
        exp_t, exp_o = expected[k]
        assert counts[k].tolist() == [len(exp_t), len(off) - 1]
        assert np.array_equal(sets[k][2][:len(exp_t)].cpu().numpy().view(np.uint32), exp_t)
        assert np.array_equal(sets[k][3].cpu().numpy().astype(np.uint64), exp_o)
    assert n_last == len(expected[2][0])


def test_every_call_resets_the_counters():
    """last_reruns() describes the most recent call only: a call that fails before it runs, and a device call that has
    been enqueued but not yet waited for, report zeros rather than what the call before them redid."""
    import torch
    e, o = _fresh("miss")
    core = e._core_bpe
    zeros = {"grown": set(), "reruns": 0, "token_passes": 0}
    text, off = ri.miss(2, 150_000, 10_000)
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, CORES)
    _check_host(e, text, off, exp_t, exp_o)
    _expect(e, {"miss"}, 1, "host call")
    bad = off.copy()
    bad[0] = 1
    with pytest.raises(ValueError):
        e.encode_ordinary_packed(text, bad)
    assert core.last_reruns() == zeros
    e._core_bpe.trim()
    d_text = torch.from_numpy(text).cuda()
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()
    d_tok = torch.empty(len(text), dtype=torch.int32, device="cuda")
    d_toff = torch.empty(len(off), dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    args = (d_text.data_ptr(), len(text), d_off.data_ptr(), len(off) - 1, d_tok.data_ptr(), d_toff.data_ptr())
    assert core.encode_device(*args) == len(exp_t)
    _expect(e, {"miss"}, 1, "device call")
    core.encode_device_async(*args)
    assert core.last_reruns() == zeros
    assert core.device_wait() == len(exp_t)
    assert core.last_reruns() == NONE
    assert np.array_equal(d_tok[:len(exp_t)].cpu().numpy().view(np.uint32), exp_t)
    assert np.array_equal(d_toff.cpu().numpy().astype(np.uint64), exp_o)
    with pytest.raises(ValueError):
        core.encode_device_async(d_text.data_ptr(), len(text), 0, len(off) - 1, d_tok.data_ptr(), d_toff.data_ptr())
    assert core.last_reruns() == zeros
