"""The inputs of test_gpu_merge_classes.py reach what they are meant to reach, checked with the oracle on the CPU.

  * the pre-tokeniser's split (the oracle's) yields exactly the generated pieces, and every length class holds pieces
    of every kind;
  * no long token is reachable by merges, so a kernel that skipped the whole-piece probe would give other tokens;
  * no near miss is a token, so a probe that matched too much would give other tokens;
  * every rank layout only shifts the tokens;
  * the missing-byte pieces succeed or fail as intended."""
import numpy as np
import pytest

import merge_class_inputs as mi
import vocab_util as vu
from oracle import Oracle

BASE = mi.base_vocab()
PIECES = mi.pieces(BASE)
NEAR = ("near_first", "near_last", "near_word")


def _oracle(ranks):
    return Oracle(ranks, {}, vu.CL100K_PAT)


def test_generation_is_deterministic():
    assert mi.base_vocab() == BASE and mi.pieces(BASE) == PIECES
    t1, o1 = mi.documents([p for _, p in PIECES])
    t2, o2 = mi.documents([p for _, p in PIECES])
    assert np.array_equal(t1, t2) and np.array_equal(o1, o2)


def test_split_yields_exactly_the_pieces_and_every_class_every_kind():
    o = _oracle(BASE)
    text, off = mi.documents([p for _, p in PIECES])
    raw = text.tobytes()
    got = []
    for d in range(len(off) - 1):
        doc = raw[int(off[d]):int(off[d + 1])]
        split = o.split(doc)
        assert split == ([s for p in doc.split(b"\n") for s in (p, b"\n")][:-1] if doc else [])
        got += [s for s in split if s != b"\n"]
    assert sorted(got) == sorted(p for _, p in PIECES)
    by_kind = {}
    for kind, p in PIECES:
        if len(p) >= mi.CLASS_MIN[0]:
            by_kind.setdefault("drop/add" if kind in ("drop", "add") else kind, []).append(mi.length_class(len(p)))
    for kind in ("hit", *NEAR, "drop/add", "adv"):
        for c in range(mi.N_CLS):
            assert by_kind[kind].count(c) >= 2, (kind, c)
    assert mi.class_counts(len(p) for p in got) == mi.class_counts(len(p) for _, p in PIECES)


def test_long_tokens_are_reachable_only_by_the_whole_piece_probe():
    o = _oracle(BASE)
    toks = mi.long_tokens(BASE)
    assert [len(t) for t in toks] == list(mi.TOKEN_LENS)
    for t in toks:
        assert len(o.byte_pair_split(t)) > 1, len(t)
        assert o.encode_single_piece(t) == [BASE[t]]
    hits = [p for k, p in PIECES if k == "hit"]
    assert hits == toks


def test_near_misses_are_not_tokens():
    for kind, p in PIECES:
        if kind in NEAR + ("drop", "add", "adv", "top"):
            assert p not in BASE, (kind, len(p))
    for t in mi.long_tokens(BASE):
        near = [p for k, p in PIECES if k in NEAR and len(p) == len(t)][:3]
        assert len(near) == 3 and all(sum(a != b for a, b in zip(p, t)) == 1 for p in near)
        first, last, word = near
        assert first[0] != t[0] and last[-1] != t[-1]
        i = next(i for i in range(len(t)) if word[i] != t[i])
        assert i >= 8 * ((len(t) - 1) // 8) and (i < len(t) - 1 or len(t) % 8 == 1)   # inside the last hash word


def test_top_pair_merges_at_position_1022():
    o = _oracle(BASE)
    top = [p for k, p in PIECES if k == "top"]
    assert len(top) == 1 and len(top[0]) == 1024 and top[0].endswith(mi.TOP_PAIR)
    assert BASE[mi.TOP_PAIR] == max(BASE.values())
    assert o.encode_single_piece(top[0])[-1] == BASE[mi.TOP_PAIR]


@pytest.mark.parametrize("layout", sorted(mi.LAYOUTS))
def test_layouts_only_shift_the_tokens(layout):
    c = mi.offset(BASE, layout)
    ranks = mi.shifted(BASE, c)
    top, low = max(ranks.values()), min(ranks.values())
    want = mi.LAYOUTS[layout]
    if want == "all":
        assert low == mi.GROUP_MAX_RANK
    else:
        assert top == (max(BASE.values()) if want is None else want)
    assert top < mi.RANK_LIMIT
    assert mi.lane_per_piece(ranks) == (top >= mi.GROUP_MAX_RANK)
    text, off = mi.documents([p for _, p in PIECES])
    base_t, base_o = _oracle(BASE).encode_ordinary_batch_np(text, off, 8)
    t, o = _oracle(ranks).encode_ordinary_batch_np(text, off, 8)
    assert np.array_equal(t.astype(np.int64), base_t.astype(np.int64) + c) and np.array_equal(o, base_o)


def test_every_family_and_pack_width_is_covered():
    tops = {name: max(mi.shifted(BASE, mi.offset(BASE, name)).values()) for name in mi.LAYOUTS}
    assert {mi.lane_per_piece({b"": t}) for t in tops.values()} == {False, True}
    assert {t.bit_length() for t in tops.values()} >= {22, 23, 24, 25, 30}


def test_missing_byte_pieces_succeed_or_fail_as_intended():
    ranks = mi.missing_byte_vocab()
    assert mi.MISSING not in ranks and any(mi.MISSING in t and len(t) > 1 for t in ranks)
    o = _oracle(ranks)
    ok, bad = mi.missing_byte_pieces(o, ranks)
    assert (ok, bad) == mi.missing_byte_pieces(o, ranks)
    assert sorted({mi.length_class(len(p)) for p in ok}) == list(range(mi.N_CLS))
    assert sorted(bad) == list(range(mi.N_CLS))
    shifted = _oracle(mi.shifted(ranks, mi.offset(ranks, "all_ge_2p22")))
    for p in ok:
        assert mi.MISSING in p and mi.RANK_MAX not in o.encode_single_piece(p) and p not in ranks
        assert mi.RANK_MAX not in shifted.encode_single_piece(p)
    for cls, p in bad.items():
        assert mi.length_class(len(p)) == cls and p.count(mi.MISSING) == 1
        assert o.encode_single_piece(p).count(mi.RANK_MAX) == 1
        assert shifted.encode_single_piece(p).count(mi.RANK_MAX) == 1
