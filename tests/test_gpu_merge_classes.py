"""Every long-piece merge kernel the engine can select, at every vocabulary edge, bit-exact against the oracle.

Pieces of more than 16 bytes go to one kernel per length class, and to another family of kernels when the largest rank
is 2^22 or above.  Each kernel has its own whole-piece probe, its own report of a single byte the vocabulary lacks and
its own rank packing.  The inputs of merge_class_inputs.py (checked on the CPU by test_merge_class_inputs.py) have long
tokens that only the probe can produce, near misses of them, adversarial merge pieces and a vocabulary without one
single byte, in every rank layout.  Every case asserts through CoreBPE.last_piece_classes() that all eight classes
were reached by the intended family, so that no case passes because its kernel never ran."""
import os

import numpy as np
import pytest

import merge_class_inputs as mi
import vocab_util as vu
from test_gpu_paths import _same

pytestmark = pytest.mark.gpu
CORES = os.cpu_count() or 1
BASE = mi.base_vocab()
PIECES = mi.pieces(BASE)
TEXT, OFF = mi.documents([p for _, p in PIECES])
CLS = mi.class_counts(len(p) for _, p in PIECES)         # the pre-tokeniser's split is exactly PIECES (CPU test)
# single-piece calls: every kind once per length, the adversarial batches by one member
SINGLE = list(dict.fromkeys(p for k, p in PIECES if k != "adv")) + \
    list({len(p): p for k, p in PIECES if k == "adv"}.values())
MISSING = mi.missing_byte_vocab()
_ENGINES = {}


def _ranks(vocab, layout):
    base = BASE if vocab == "base" else MISSING
    return mi.shifted(base, mi.offset(base, layout))


def _engine(vocab, layout):
    """(Encoding, Oracle, ranks, offset) of a vocabulary in a rank layout, built once per module."""
    key = (vocab, layout)
    if key not in _ENGINES:
        import tiktoken_b200
        from oracle import Oracle
        ranks = _ranks(vocab, layout)
        special = mi.special_tokens(ranks)
        e = tiktoken_b200.Encoding(f"merge_classes_{vocab}_{layout}", pat_str=vu.CL100K_PAT, mergeable_ranks=ranks,
                                   special_tokens=special)
        base = BASE if vocab == "base" else MISSING
        _ENGINES[key] = (e, Oracle(ranks, special, vu.CL100K_PAT), ranks, mi.offset(base, layout))
    return _ENGINES[key]


def _classes(e, counts, ranks, what):
    got = e._core_bpe.last_piece_classes()
    assert got == {"counts": list(counts), "lane_per_piece": mi.lane_per_piece(ranks)}, (what, got)


_BASE_OUT = {}


def _base_output():
    """Tokens and offsets of the engine on the vocabulary as built (host path)."""
    if not _BASE_OUT:
        e = _engine("base", "as_built")[0]
        buf = e.encode_ordinary_packed(TEXT, OFF)
        _BASE_OUT["t"], _BASE_OUT["o"] = np.array(buf.tokens()), np.array(buf.offsets())
        buf.close()
    return _BASE_OUT["t"], _BASE_OUT["o"]


def _check_shift(t, o, c):
    base_t, base_o = _base_output()
    assert np.array_equal(t.astype(np.int64), base_t.astype(np.int64) + c) and np.array_equal(o, base_o)


@pytest.mark.parametrize("layout", list(mi.LAYOUTS))
def test_host_path(layout):
    """encode_ordinary_packed: every class, both families, all tokens and offsets."""
    e, o, ranks, c = _engine("base", layout)
    assert all(CLS)
    exp_t, exp_o = o.encode_ordinary_batch_np(TEXT, OFF, CORES)
    buf = e.encode_ordinary_packed(TEXT, OFF)
    t, toff = np.array(buf.tokens()), np.array(buf.offsets())
    buf.close()
    _classes(e, CLS, ranks, "host path")
    assert np.array_equal(t, exp_t) and np.array_equal(toff, exp_o)
    _check_shift(t, toff, c)


@pytest.mark.parametrize("layout", list(mi.LAYOUTS))
def test_device_path(layout):
    import torch
    e, o, ranks, c = _engine("base", layout)
    exp_t, exp_o = o.encode_ordinary_batch_np(TEXT, OFF, CORES)
    d_text = torch.from_numpy(TEXT).cuda()
    d_off = torch.from_numpy(OFF.astype(np.int64)).cuda()
    d_tok = torch.full((len(TEXT),), -1, dtype=torch.int32, device="cuda")
    d_toff = torch.full((len(OFF),), -1, dtype=torch.int64, device="cuda")
    torch.cuda.synchronize()
    n = e._core_bpe.encode_device(d_text.data_ptr(), len(TEXT), d_off.data_ptr(), len(OFF) - 1, d_tok.data_ptr(),
                                  d_toff.data_ptr())
    _classes(e, CLS, ranks, "device path")
    t = d_tok[:n].cpu().numpy().view(np.uint32)
    toff = d_toff.cpu().numpy().astype(np.uint64)
    assert n == len(exp_t) and np.array_equal(t, exp_t) and np.array_equal(toff, exp_o)
    _check_shift(t, toff, c)


@pytest.mark.parametrize("layout", list(mi.LAYOUTS))
def test_single_piece(layout):
    """_encode_single_piece per piece: the piece alone in its class, its class alone in the call."""
    e, o, ranks, _ = _engine("base", layout)
    seen = set()
    for p in SINGLE:
        assert e._encode_single_piece(p) == o.encode_single_piece(p), len(p)
        cls = mi.class_counts([len(p)])
        _classes(e, cls, ranks, len(p))
        seen.update(i for i, k in enumerate(cls) if k)
    assert seen == set(range(mi.N_CLS))


@pytest.mark.parametrize("layout", [k for k in mi.LAYOUTS if mi.special_tokens(_ranks("base", k))])
def test_special_token_between_long_pieces(layout):
    """Ids of 2^24 and above: a special token (at 2^25, or just below the smallest rank of the 2^30 - 1 layout) next to
    pieces of every class, and decoded on the host maps."""
    e, o, ranks, _ = _engine("base", layout)
    hits = [p.decode() for k, p in PIECES if k == "hit"]
    docs = ["<|x|>".join(hits[::3]), hits[-1] + "<|x|>", "<|x|>"]
    got = e.encode_batch(docs, allowed_special="all")
    assert got == [o.encode(d, {"<|x|>"}) for d in docs]
    assert e.decode_batch(got) == docs


@pytest.mark.parametrize("layout", list(mi.LAYOUTS))
def test_decode_returns_the_exact_bytes(layout):
    """decode_batch and decode_packed of the results, 40 kB tokens included: on the device below 2^24, on the host
    maps at and above it."""
    e, o, ranks, _ = _engine("base", layout)
    exp_t, exp_o = o.encode_ordinary_batch_np(TEXT, OFF, CORES)
    data, boff = e.decode_packed(exp_t, exp_o)
    assert np.array_equal(data, TEXT) and np.array_equal(boff, OFF)
    docs = [exp_t[int(exp_o[d]):int(exp_o[d + 1])].tolist() for d in range(len(OFF) - 1)]
    raw = TEXT.tobytes()
    assert e.decode_bytes_batch(docs) == [raw[int(OFF[d]):int(OFF[d + 1])] for d in range(len(OFF) - 1)]
    longest = max(mi.long_tokens(BASE), key=len)
    assert e.decode_bytes_batch([[ranks[longest]], [ranks[longest]] * 2]) == [longest, longest * 2]
    with pytest.raises(KeyError):
        e.decode_bytes_batch([[max(ranks.values()) + 3]])


def test_rank_limit():
    """Ranks must be below 2^30: 2^30 - 1 builds (and encodes, above), 2^30 is refused at construction."""
    import tiktoken_b200
    assert max(_ranks("base", "top_2p30m1").values()) == mi.RANK_LIMIT - 1
    over = mi.shifted(BASE, mi.RANK_LIMIT - max(BASE.values()))
    with pytest.raises(ValueError, match="rank too large"):
        tiktoken_b200.Encoding("merge_classes_over", pat_str=vu.CL100K_PAT, mergeable_ranks=over, special_tokens={})


def test_special_token_ids_up_to_the_rank_limit():
    """Special ids obey the same limit.  The probe kernel stores an allowed special's id in the token slot of its
    piece, whose top two bits tag misses and long pieces: a special id of 2^30 came back as the tokens of some other
    piece until construction refused it.  2^30 - 1 is the largest id a slot holds."""
    import tiktoken_b200
    from oracle import Oracle
    with pytest.raises(ValueError, match="special token id too large"):
        tiktoken_b200.Encoding("merge_classes_sp_over", pat_str=vu.CL100K_PAT, mergeable_ranks=BASE,
                               special_tokens={"<|x|>": mi.RANK_LIMIT})
    special = {"<|x|>": mi.RANK_LIMIT - 1}
    e = tiktoken_b200.Encoding("merge_classes_sp_top", pat_str=vu.CL100K_PAT, mergeable_ranks=BASE,
                               special_tokens=special)
    o = Oracle(BASE, special, vu.CL100K_PAT)
    hits = [p.decode() for k, p in PIECES if k == "hit"]
    docs = ["<|x|>".join(hits[::3]), "<|x|>" + hits[0], "<|x|>"]
    got = e.encode_batch(docs, allowed_special="all")
    assert got == [o.encode(d, {"<|x|>"}) for d in docs]
    assert got[-1] == [mi.RANK_LIMIT - 1]
    assert e.decode_batch(got) == docs


# ---- a single byte the vocabulary lacks -----------------------------------------------------------------------------
FAMILIES = {"group": "as_built", "lane_per_piece": "all_ge_2p22"}
_MISSING_PIECES = {}


def _missing_pieces():
    if not _MISSING_PIECES:
        from oracle import Oracle
        ok, bad = mi.missing_byte_pieces(Oracle(MISSING, {}, vu.CL100K_PAT), MISSING)
        _MISSING_PIECES.update(ok=ok, bad=bad)
    return _MISSING_PIECES["ok"], _MISSING_PIECES["bad"]


def _missing_ok_call(e, o, ranks):
    ok, _ = _missing_pieces()
    text, off = mi.documents(ok, per_doc=4)
    exp_t, exp_o = o.encode_ordinary_batch_np(text, off, CORES)
    assert mi.RANK_MAX not in exp_t
    assert _same(e.encode_ordinary_packed(text, off), exp_t, exp_o)
    _classes(e, mi.class_counts(len(p) for p in ok), ranks, "missing byte, merged away")


@pytest.mark.parametrize("family", list(FAMILIES))
def test_missing_byte_merged_away(family):
    """Every "c" ends inside a merged token: the pseudo id of the missing byte merges like any other."""
    e, o, ranks, _ = _engine("missing", FAMILIES[family])
    assert mi.lane_per_piece(ranks) == (family == "lane_per_piece")
    _missing_ok_call(e, o, ranks)
    ok, _ = _missing_pieces()
    for p in ok:
        assert e._encode_single_piece(p) == o.encode_single_piece(p), len(p)


@pytest.mark.parametrize("cls", range(mi.N_CLS))
@pytest.mark.parametrize("family", list(FAMILIES))
def test_missing_byte_left_alone_is_an_error(family, cls):
    """One piece of class `cls` leaves a "c" alone, among pieces of every class that do not: the kernel of that class
    must report it (KeyError), and the engine stays usable."""
    e, o, ranks, _ = _engine("missing", FAMILIES[family])
    ok, bad = _missing_pieces()
    text, off = mi.documents(ok + [bad[cls]], per_doc=4)
    with pytest.raises(KeyError):
        e.encode_ordinary_packed(text, off)
    assert e._core_bpe.last_piece_classes() == {"counts": [0] * mi.N_CLS, "lane_per_piece": False}
    with pytest.raises(KeyError):
        e._encode_single_piece(bad[cls])
    _missing_ok_call(e, o, ranks)
