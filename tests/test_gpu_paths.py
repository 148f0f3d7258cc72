"""Parity of the paths the plain parity suite does not reach (VERDICT round 1, "parity holes"):
  * the chunked host pipeline (3-slot H2D / kernels / D2H) with chunk seams, forced by B200BPE_CHUNK_MB=1
    and, at the default chunk size, by an input of > 200 MiB -- every token compared with the oracle;
  * one device-resident call of > 256 MiB (the large-batch workspace path) compared in full;
  * pieces of 4 097 ... 100 000 bytes on adversarial tiny-alphabet vocabularies (rank ties, cascades,
    non-monotone ranks) through the block / cluster round-synchronous merge (ref src/lib.rs:47-138);
  * result lifetime (TokenBuffer / arrays outliving the Encoding);
  * the reference's OWN host class (`tiktoken.core.Encoding`, unmodified, from the installed wheel) running on
    top of `tiktoken_b200._tiktoken` -- the true drop-in.
All through the C ABI, bit-exact."""
import gc
import os
import pickle
import random

import numpy as np
import pytest

import vocab_util as vu
from tools import corpus

pytestmark = pytest.mark.gpu
CORES = os.cpu_count() or 1


def _oracle(ranks, special, pat):
    from oracle import Oracle
    return Oracle(ranks, special, pat)


def _chunked_encoding(enc_name, chunk_mb, vocab=None, devices=None, **env):
    """An Encoding whose host pipeline cuts batches into chunk_mb-MiB chunks (knobs are read at construction).
    vocab = (pat_str, mergeable_ranks, special_tokens) replaces the named synthetic encoding; devices as Encoding's."""
    import tiktoken_b200
    pat, ranks, special = vocab or vu.load_encoding(enc_name, allow_real=False)[:3]
    env = dict(env, B200BPE_CHUNK_MB=chunk_mb)
    old = {k: os.environ.get(k) for k in env}
    os.environ.update({k: str(v) for k, v in env.items()})
    try:
        e = tiktoken_b200.Encoding(f"{enc_name}_chunk", pat_str=pat, mergeable_ranks=ranks, special_tokens=special,
                                   devices=devices)
    finally:
        for k, v in old.items():
            if v is None:
                os.environ.pop(k, None)
            else:
                os.environ[k] = v
    return e, _oracle(ranks, special, pat), special


def _same(buf, exp_t, exp_o):
    ok = np.array_equal(buf.tokens(), exp_t) and np.array_equal(buf.offsets(), exp_o)
    buf.close()
    return ok


@pytest.mark.parametrize("enc,kind", [("cl100k_base", corpus.ENGLISH), ("o200k_base", corpus.MIXED),
                                      ("p50k_base", corpus.CODE), ("r50k_base", corpus.ENGLISH)])
def test_chunk_seams_1mib_chunks(enc, kind):
    e, o, special = _chunked_encoding(enc, 1)
    text = corpus.generate(kind, 99, 7 << 20)
    layouts = [corpus.docs_fixed(text, 65536, at_space=False)[1],                       # ~16 docs per chunk
               corpus.docs_fixed(text, 300_000, at_space=False)[1],                     # docs that do not divide a chunk
               np.asarray([0, 10, 10, 3 << 20, (3 << 20) + 5, len(text)], np.uint64)]   # docs larger than a chunk, empty doc
    lens = np.clip(np.rint(np.random.default_rng(3).lognormal(np.log(90), 0.5, size=200_000)), 0, 2000).astype(np.int64)
    layouts.append(corpus.docs_from_lengths(text, lens[:int(np.searchsorted(np.cumsum(lens), len(text)))], False)[1])
    for off in layouts:
        off = np.ascontiguousarray(off, np.uint64)
        # cut points must not split a UTF-8 scalar: move them back onto lead bytes
        for i in range(1, len(off) - 1):
            while 0 < off[i] < len(text) and (text[int(off[i])] & 0xC0) == 0x80:
                off[i] -= 1
        off = np.maximum.accumulate(off)
        exp_t, exp_o = o.encode_ordinary_batch_np(text, off, CORES)
        assert _same(e.encode_ordinary_packed(text, off), exp_t, exp_o)
    # allowed specials across chunk seams (CoreBPE::encode, lib.rs:375-442)
    names = sorted(special)
    rnd = random.Random(5)
    docs = []
    for d in range(40):
        s = text[d * 150_000:(d + 1) * 150_000].tobytes().decode("utf-8", "ignore")
        cut = sorted(rnd.sample(range(len(s)), 20))
        parts, prev = [], 0
        for c in cut:
            parts += [s[prev:c], rnd.choice(names)]
            prev = c
        docs.append("".join(parts) + s[prev:])
    got = e.encode_batch(docs, allowed_special="all")
    assert got == [o.encode(d, set(special)) for d in docs]


def test_default_chunks_over_200mib_full_compare():
    import tiktoken_b200
    pat, ranks, special, _ = vu.load_encoding("cl100k_base", allow_real=False)
    e = tiktoken_b200.Encoding("big_host", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)
    o = _oracle(ranks, special, pat)
    text, off = corpus.config2(nbytes=208 << 20, seed=4321)
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, CORES)
    assert _same(e.encode_ordinary_packed(text, off), exp_t, exp_o)
    # the same bytes as ONE document (chunking cannot cut it, one pipeline pass takes it whole): checked through
    # the round trip decode(encode(x)) == x on the device decoder (the oracle is single-threaded on one document)
    one = np.asarray([0, len(text)], np.uint64)
    buf = e.encode_ordinary_packed(text, one)
    toks, toff = np.array(buf.tokens()), np.array(buf.offsets())
    buf.close()
    assert int(toff[-1]) == len(toks) and len(toff) == 2
    data, boff = e.decode_packed(toks, toff)
    assert np.array_equal(data, text) and np.array_equal(boff, one)


def test_device_resident_call_over_256mib_full_compare():
    import torch
    import tiktoken_b200
    pat, ranks, special, _ = vu.load_encoding("o200k_base", allow_real=False)
    e = tiktoken_b200.Encoding("big_dev", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)
    o = _oracle(ranks, special, pat)
    text, off = corpus.config3(nbytes=288 << 20, seed=77)
    d_text = torch.from_numpy(text).cuda()
    d_off = torch.from_numpy(off.astype(np.int64)).cuda()
    d_tok = torch.empty(len(text), dtype=torch.int32, device="cuda")
    d_toff = torch.empty(len(off), dtype=torch.int64, device="cuda")
    n = e._core_bpe.encode_device(d_text.data_ptr(), len(text), d_off.data_ptr(), len(off) - 1, d_tok.data_ptr(),
                                  d_toff.data_ptr())
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, CORES)
    assert n == len(exp_t)
    assert np.array_equal(d_toff.cpu().numpy().astype(np.uint64), exp_o)
    assert np.array_equal(d_tok[:n].cpu().numpy().view(np.uint32), exp_t)
    # and the host path on the same input agrees with it (three pipeline slots, default chunks)
    assert _same(e.encode_ordinary_packed(text, off), exp_t, exp_o)


def _adversarial_vocab(rnd, alpha, n_tokens, lens):
    ranks = {bytes([i]): i for i in range(256)}
    toks = set()
    while len(toks) < n_tokens:
        toks.add("".join(rnd.choice(alpha) for _ in range(rnd.choice(lens))).encode())
    for t, r in zip(sorted(toks), rnd.sample(range(256, 256 + 4 * n_tokens), len(toks))):
        ranks[t] = r                                          # random ranks: ties impossible, order adversarial
    return ranks


@pytest.mark.parametrize("trial", range(4))
def test_giant_pieces_with_adversarial_vocabulary(trial):
    """Pieces beyond 4 096 bytes (block per piece) and beyond 32 768 bytes (thread-block cluster per piece) on
    vocabularies where a merge often creates a LOWER-ranked pair next to it (the "violation" of the
    round-synchronous merge) and long chains of equal-rank candidates overlap."""
    import tiktoken_b200
    rnd = random.Random(1000 + trial)
    alpha = ["ab", "abc", "ab", "abcd"][trial]
    ranks = _adversarial_vocab(rnd, alpha, [12, 40, 25, 80][trial], [2, 2, 2, 3, 3, 4, 5, 6, 9, 14])
    if trial == 2:                                            # powers of one letter: the x*1_000_000 shape, with gaps
        for k, r in ((2, 300), (4, 290), (8, 310), (16, 280), (3, 305)):
            ranks[b"a" * k] = 5000 + r
    e = tiktoken_b200.Encoding("adv_giant", pat_str=vu.CL100K_PAT, mergeable_ranks=ranks, special_tokens={})
    o = _oracle(ranks, {}, vu.CL100K_PAT)
    pieces = []
    for n in (4097, 5000, 10_000, 32_768, 32_769, 50_000, 100_000):
        style = rnd.choice(["random", "periodic", "runs"])
        if style == "random":
            p = "".join(rnd.choice(alpha) for _ in range(n))
        elif style == "periodic":
            unit = "".join(rnd.choice(alpha) for _ in range(rnd.choice([1, 2, 3, 5, 7])))
            p = (unit * (n // len(unit) + 1))[:n]
        else:
            p, out = "", []
            while len(p) < n:
                p += rnd.choice(alpha) * rnd.choice([1, 2, 3, 17, 64, 1000])
            p = p[:n]
        pieces.append(p)
    for p in pieces:                                         # single-piece entry point (py.rs:145-150)
        assert e._encode_single_piece(p) == o.encode_single_piece(p.encode()), len(p)
    docs = [" ".join(pieces), pieces[3], "\n".join(pieces[::2]) + "\n", ""]     # letter runs split at the separators
    assert e.encode_ordinary_batch(docs) == [o.encode_ordinary(d) for d in docs]


def test_results_outlive_their_encoding():
    import tiktoken_b200
    pat, ranks, special, _ = vu.load_encoding("r50k_base", allow_real=False)
    o = _oracle(ranks, special, pat)
    text, off = corpus.config2(nbytes=1 << 20, seed=8)
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, CORES)

    def make():
        return tiktoken_b200.Encoding("short_lived", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)

    toks = make().encode_ordinary_packed(text, off).tokens()     # Encoding and TokenBuffer both unreferenced now
    gc.collect()
    other = make()
    junk = other.encode_ordinary_packed(text[::-1].copy() & 0x7F, np.asarray([0, len(text)], np.uint64))   # would reuse a pooled block
    assert np.array_equal(toks, exp_t)
    junk.close()
    buf = make().encode_ordinary_packed(text, off)               # buffer alive, engine object gone
    gc.collect()
    assert np.array_equal(buf.offsets(), exp_o) and np.array_equal(buf.tokens(), exp_t)
    buf.close()
    buf.close()                                                  # idempotent


def test_reference_host_class_runs_on_the_b200_core(monkeypatch):
    """The drop-in itself: the reference's unmodified `tiktoken.core.Encoding` (installed wheel == the
    reference's host code, SURVEY 8(c)) with `tiktoken.core._tiktoken` swapped for `tiktoken_b200._tiktoken`
    (core.py:7 import, :57 constructor, :161 encode_to_tiktoken_buffer -> np.frombuffer, :409-428 pickling)."""
    tiktoken = pytest.importorskip("tiktoken")
    import tiktoken.core as ref_core
    from tiktoken_b200 import _tiktoken as shim
    monkeypatch.setattr(ref_core, "_tiktoken", shim)
    pat, ranks, special, _ = vu.load_encoding("cl100k_base", allow_real=False)
    enc = tiktoken.Encoding("dropin", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)
    assert isinstance(enc._core_bpe, shim.CoreBPE)
    o = _oracle(ranks, special, pat)
    docs = ["hello world", "", "don't  stop\n\n  x", "日本語 text <|endoftext|> tail", "x" * 300, " " * 40 + "\n" * 3]
    docs += [corpus.generate(corpus.ENGLISH, 5, 20_000).tobytes().decode()]
    for d in docs:
        assert enc.encode_ordinary(d) == o.encode_ordinary(d)
        assert enc.encode(d, allowed_special="all") == o.encode(d, set(special))
        assert enc.encode_to_numpy(d, allowed_special="all").tolist() == o.encode(d, set(special))
        assert enc.decode(enc.encode(d, allowed_special="all")) == d
    with pytest.raises(ValueError):
        enc.encode("a <|endoftext|> b")                              # disallowed by default (core.py:120-124)
    assert enc.encode_ordinary_batch(docs) == [o.encode_ordinary(d) for d in docs]          # thread pool over per-doc calls
    assert enc.encode_batch(docs, allowed_special="all") == [o.encode(d, set(special)) for d in docs]
    assert enc.decode_batch(enc.encode_ordinary_batch(docs)) == docs
    assert enc.encode_single_token(b"a") == ranks[b"a"] and enc.decode_single_token_bytes(ranks[b"a"]) == b"a"
    assert enc.decode_bytes(enc.encode_ordinary("héllo")) == "héllo".encode()
    assert enc._encode_single_piece(b"helloqqqq") == o.encode_single_piece(b"helloqqqq")
    assert sorted(enc.token_byte_values()) == sorted(ranks)
    assert enc.encode_ordinary("\ud83d") == enc.encode_ordinary("�")                   # surrogate fix-up, core.py:77-80
    enc2 = pickle.loads(pickle.dumps(enc))                                                 # by value (not in the registry)
    assert isinstance(enc2._core_bpe, shim.CoreBPE)
    assert enc2.encode_ordinary("pickled hello") == o.encode_ordinary("pickled hello")


def test_device_special_scan_edge_cases():
    """The multi-pattern scan behind CoreBPE::encode (lib.rs:375-442) and the disallowed check (core.py:120-124):
    specials longer than 16 bytes, a thousand reserved specials (o200k_harmony style), specials at document ends,
    adjacent and self-overlapping occurrences, look-alikes, and the leftmost disallowed special in a batch."""
    import tiktoken_b200
    pat, ranks, _, _ = vu.load_encoding("o200k_base", allow_real=False)
    base = max(ranks.values()) + 1
    special = {"<|endoftext|>": base, "<|endofprompt|>": base + 1, "<|a|>": base + 2, "aXa": base + 3,
               "<|start_of_a_very_long_special_token_name|>": base + 4}
    special.update({f"<|reserved_{i}|>": base + 10 + i for i in range(1000)})
    e = tiktoken_b200.Encoding("sp_edge", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)
    o = _oracle(ranks, special, pat)
    allowed = set(special)
    docs = ["<|endoftext|>", "<|endoftext|><|endoftext|>", "x<|a|>", "<|a|>x", "a  <|endoftext|>b", "a  b",
            "<|start_of_a_very_long_special_token_name|> tail", "head <|reserved_7|><|reserved_999|> <|reserved_1000|>",
            "aXaXa aXaXaXa XaXaX", "<|endoftext", "|endoftext|>", "<|<|a|>|>", "", "日本語<|a|>日本語" * 50,
            "   <|endofprompt|>\n\n  \n<|a|>   ", "<|a|>" * 300, "no specials here at all " * 100]
    assert e.encode_batch(docs, allowed_special="all") == [o.encode(d, allowed) for d in docs]
    for only in ({"<|a|>"}, {"aXa"}, {"<|reserved_7|>", "<|endoftext|>"}):
        assert e.encode_batch(docs, allowed_special=only, disallowed_special=()) == [o.encode(d, only) for d in docs]
    for d in docs:                                                   # the single-text entry point of py.rs:34-49
        assert e.encode(d, allowed_special="all") == o.encode(d, allowed)
    # default policy: everything not allowed is disallowed -> ValueError naming the LEFTMOST offender of the batch
    with pytest.raises(ValueError, match="disallowed special token '<\\|a\\|>'"):
        e.encode_batch(["fine", "x <|a|> then <|endoftext|>", "<|endoftext|>"], allowed_special={"<|endoftext|>"})
    with pytest.raises(ValueError, match="disallowed special token '<\\|reserved_5\\|>'"):
        e.encode_batch(["fine", "<|reserved_5|>"])
    assert e.encode_batch(["fine", "no <| specials |> here"]) == [o.encode_ordinary("fine"), o.encode_ordinary("no <| specials |> here")]
    # a special split across two documents is not a special
    assert e.encode_batch(["<|endof", "text|>"], allowed_special="all") == [o.encode_ordinary("<|endof"), o.encode_ordinary("text|>")]
    # array form: zero-copy pinned result, same tokens
    text = np.frombuffer("".join(docs).encode(), np.uint8)
    off = np.zeros(len(docs) + 1, np.uint64)
    off[1:] = np.cumsum([len(d.encode()) for d in docs])
    with e.encode_packed(text, off, allowed_special="all") as buf:
        flat = [t for d in docs for t in o.encode(d, allowed)]
        assert buf.tokens().tolist() == flat


def test_queued_device_calls_and_count_buffer():
    import torch
    import tiktoken_b200
    pat, ranks, special, _ = vu.load_encoding("cl100k_base", allow_real=False)
    e = tiktoken_b200.Encoding("async_dev", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)
    o = _oracle(ranks, special, pat)
    core = e._core_bpe
    stream = torch.cuda.Stream()
    inputs = [corpus.config2(nbytes=(3 + k) << 20, seed=50 + k) for k in range(3)]
    with torch.cuda.stream(stream):
        counts = torch.zeros((3, 2), dtype=torch.int64, device="cuda")
        sets = []
        for k, (text, off) in enumerate(inputs):
            d_text = torch.from_numpy(text).cuda(); d_off = torch.from_numpy(off.astype(np.int64)).cuda()
            d_tok = torch.empty(len(text), dtype=torch.int32, device="cuda"); d_toff = torch.empty(len(off), dtype=torch.int64, device="cuda")
            sets.append((d_text, d_off, d_tok, d_toff))
        stream.synchronize()
        # settle the work-space sizes with one synchronous call on the largest input, then queue three without waiting
        core.encode_device(sets[2][0].data_ptr(), len(inputs[2][0]), sets[2][1].data_ptr(), len(inputs[2][1]) - 1,
                           sets[2][2].data_ptr(), sets[2][3].data_ptr(), stream.cuda_stream)
        for k, (text, off) in enumerate(inputs):
            d_text, d_off, d_tok, d_toff = sets[k]
            core.encode_device_async(d_text.data_ptr(), len(text), d_off.data_ptr(), len(off) - 1, d_tok.data_ptr(),
                                     d_toff.data_ptr(), counts[k].data_ptr(), stream.cuda_stream)
        n_last = core.device_wait()
    stream.synchronize()
    for k, (text, off) in enumerate(inputs):
        exp_t, exp_o = o.encode_ordinary_batch_np(text, off, CORES)
        assert counts[k].tolist() == [len(exp_t), len(off) - 1]
        assert np.array_equal(sets[k][2][:len(exp_t)].cpu().numpy().view(np.uint32), exp_t)
        assert np.array_equal(sets[k][3].cpu().numpy().astype(np.uint64), exp_o)
    assert n_last == int(counts[2, 0])



def test_one_process_multi_gpu_engine():
    """SURVEY 8(b)/(e): ONE engine over several GPUs behind the same C ABI -- chunks round-robin over the devices,
    every chunk's tokens at its final offset of one pinned buffer.  Needs two devices."""
    import tiktoken_b200
    from tiktoken_b200 import _lib
    ndev = int(_lib.lib().b200bpe_device_count())
    if ndev < 2:
        pytest.skip("needs at least two CUDA devices")
    pat, ranks, special, _ = vu.load_encoding("cl100k_base", allow_real=False)
    e = tiktoken_b200.Encoding("multi", pat_str=pat, mergeable_ranks=ranks, special_tokens=special, devices=list(range(min(ndev, 8))))
    assert e._core_bpe.devices == list(range(min(ndev, 8)))
    o = _oracle(ranks, special, pat)
    text, off = corpus.config2(nbytes=160 << 20, seed=99)
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, CORES)
    for _ in range(2):
        assert _same(e.encode_ordinary_packed(text, off), exp_t, exp_o)
    docs = [text[int(off[i]):int(off[i + 1])].tobytes().decode() for i in range(40)] + ["", "<|endoftext|> x"]
    assert e.encode_batch(docs, allowed_special="all") == [o.encode(d, set(special)) for d in docs]
    small, soff = corpus.config4(n_docs=50_000, seed=3)
    exp_t, exp_o = o.encode_ordinary_batch_np(small, soff, CORES)
    assert _same(e.encode_ordinary_packed(small, soff), exp_t, exp_o)


def test_trim_releases_and_the_engine_keeps_working():
    import tiktoken_b200
    pat, ranks, special, _ = vu.load_encoding("p50k_base", allow_real=False)
    e = tiktoken_b200.Encoding("trim", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)
    o = _oracle(ranks, special, pat)
    text, off = corpus.config5(nbytes=3 << 20, seed=11)
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, 1)
    assert _same(e.encode_ordinary_packed(text, off), exp_t, exp_o)
    e._core_bpe.trim()                                   # work-spaces and pooled pinned blocks are gone, tables stay
    assert _same(e.encode_ordinary_packed(text, off), exp_t, exp_o)
    assert e.decode_bytes(exp_t) == text.tobytes()


def test_reference_loaders_feed_the_engine(tmp_path, monkeypatch):
    """`tiktoken/load.py` stays (north star): a `.tiktoken` file read by the reference's `load_tiktoken_bpe`, the same file
    parsed in C (`Encoding.from_tiktoken_file`, SURVEY 8(f)-4) and a gpt2-style data-gym pair (`vocab.bpe` + `encoder.json`,
    `load.py:89-144`: single-byte ranks follow the printable-first order, not the byte values) all construct engines on
    the GPU whose output equals the oracle's on the same ranks."""
    import gzip
    import json
    import tiktoken.load as ref_load
    import tiktoken_b200
    monkeypatch.setenv("TIKTOKEN_CACHE_DIR", "")                                    # plain local reads, no cache directory
    text = corpus.generate(corpus.ENGLISH, 5, 3 << 20)
    off = corpus.docs_fixed(text, 40_000, at_space=True)[1]
    special = {"<|endoftext|>": 50256}
    # ---- .tiktoken: reference loader -> dict -> engine; C parser -> flat arrays -> engine
    src = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "vocab", "r50k_like.tiktoken.gz")
    path = str(tmp_path / "r50k_like.tiktoken")
    with open(path, "wb") as f:
        f.write(gzip.open(src).read())
    ranks = ref_load.load_tiktoken_bpe(path)
    o = _oracle(ranks, special, vu.R50K_PAT)
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, CORES)
    e_dict = tiktoken_b200.Encoding("by_ref_loader", pat_str=vu.R50K_PAT, mergeable_ranks=ranks, special_tokens=special)
    e_file = tiktoken_b200.Encoding.from_tiktoken_file("by_c_parser", path, pat_str=vu.R50K_PAT, special_tokens=special)
    assert _same(e_dict.encode_ordinary_packed(text, off), exp_t, exp_o)
    assert _same(e_file.encode_ordinary_packed(text, off), exp_t, exp_o)
    assert e_file.n_vocab == e_dict.n_vocab and e_file.decode_bytes(exp_t[:1000].tolist()) == e_dict.decode_bytes(exp_t[:1000].tolist())
    # ---- data-gym: re-rank the single bytes the gpt2 way, write merges + encoder.json, read them back with the reference
    order = [b for b in range(256) if chr(b).isprintable() and chr(b) != " "]
    g2b, n = {chr(b): b for b in order}, 0
    for b in range(256):
        if b not in order:
            order.append(b)
            g2b[chr(256 + n)] = b
            n += 1
    b2g = {b: c for c, b in g2b.items()}
    enc_gym = lambda bs: "".join(b2g[x] for x in bs)
    small = {t: r for t, r in ranks.items() if len(t) == 1 or r < 256 + 6000}         # the first 6000 merges are enough here
    gym = {bytes([b]): i for i, b in enumerate(order)}
    merges, cur = [], dict(gym)
    for tok, _ in sorted(((t, r) for t, r in small.items() if len(t) > 1), key=lambda x: x[1]):
        parts = [bytes([x]) for x in tok]                                           # BPE of the token under the ranks so far -> its two parents
        while len(parts) > 2:
            best = min(range(len(parts) - 1), key=lambda i: (cur.get(parts[i] + parts[i + 1], 1 << 60), i))
            if parts[best] + parts[best + 1] not in cur:
                break
            parts[best:best + 2] = [parts[best] + parts[best + 1]]
        if len(parts) != 2:
            continue                                                               # not reachable by merges of earlier tokens: leave it out
        merges.append((parts[0], parts[1]))
        cur[tok] = len(cur)
    vocab_bpe, encoder_json = str(tmp_path / "vocab.bpe"), str(tmp_path / "encoder.json")
    with open(vocab_bpe, "w", encoding="utf-8") as f:
        f.write("#version: 0.2\n" + "".join(f"{enc_gym(a)} {enc_gym(b)}\n" for a, b in merges))
    with open(encoder_json, "w", encoding="utf-8") as f:
        json.dump({enc_gym(t): r for t, r in cur.items()}, f)
    gym_ranks = ref_load.data_gym_to_mergeable_bpe_ranks(vocab_bpe, encoder_json)
    assert gym_ranks == cur and gym_ranks[b"!"] == 0 and len(merges) > 4000
    e_gym = tiktoken_b200.Encoding("by_data_gym", pat_str=vu.R50K_PAT, mergeable_ranks=gym_ranks, special_tokens={"<|endoftext|>": len(cur)})
    o2 = _oracle(gym_ranks, {}, vu.R50K_PAT)
    exp_t, exp_o = o2.encode_ordinary_batch_np(text, off, CORES)
    assert _same(e_gym.encode_ordinary_packed(text, off), exp_t, exp_o)
