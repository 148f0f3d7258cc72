"""CPU side of the completion search: the restatement in unstable_oracle.py pinned to the tiktoken wheel's
`encode_with_unstable` (tests/golden/encode_with_unstable.json), and the host classes' `encode_with_unstable_batch`
on a stub engine that answers from that restatement (special-token policy, errors, empty batch)."""
import hashlib
import json
import os

import numpy as np
import pytest

import vocab_util as vu
from oracle import Oracle
from test_host_shim_stub import StubLib
from unstable_oracle import UnstableOracle

HERE = os.path.dirname(os.path.abspath(__file__))
ENCODINGS = ["cl100k_base", "r50k_base", "p50k_base", "o200k_base"]


def _digest(comps):
    """tests/golden/make_unstable_golden.py: the first 16 hex digits of the sha256 of the sorted completions"""
    return hashlib.sha256(json.dumps(sorted(comps)).encode()).hexdigest()[:16]


@pytest.mark.parametrize("enc", ENCODINGS)
def test_restatement_matches_the_wheel_fixture(enc):
    with open(os.path.join(HERE, "golden", "encode_with_unstable.json")) as f:
        cases = json.load(f)[enc]
    assert len(cases) > 250
    pat, ranks, special, _ = vu.load_encoding(enc, allow_real=False)
    uo = UnstableOracle(Oracle(ranks, special, pat), ranks, special)
    for text, allowed, stable_exp, n, dig in cases:
        stable, comps = uo.encode_with_unstable(text, frozenset(allowed))
        assert stable == stable_exp, text
        assert len(comps) == n and len({tuple(s) for s in comps}) == n, text
        assert _digest(comps) == dig, text


class UnstableStub(StubLib):
    """StubLib plus the completion search entry points, answered by the restatement."""

    def __init__(self):
        super().__init__()
        self.groups = {}

    def b200bpe_encode_with_unstable_batch(self, h, text, doc_off, n_docs, flags, stable, comp, bad):
        o, names, dec = self.engines[h.value]
        mask = self._arr(flags, np.uint8, len(names))
        allow = frozenset(nm for nm, m in zip(names, mask) if m == 1)
        docs = self._docs(text, doc_off, n_docs)
        for d in docs:                                        # the first document's leftmost disallowed special
            hits = [(d.find(nm.encode()), i) for i, (nm, m) in enumerate(zip(names, mask)) if m == 2 and nm.encode() in d]
            if hits:
                bad._obj.value = min(hits)[1]
                return -7
        sids = self._special_ids(h)
        ranks = {b: r for r, b in dec.items() if r not in set(sids)}
        uo = UnstableOracle(o, ranks, dict(zip(names, sids)))
        st_t, st_o, c_t, c_o, grp = [], [0], [], [0], [0]
        for d in docs:
            s, comps = uo.encode_with_unstable(d.decode("utf-8"), allow)
            st_t += s
            st_o.append(len(st_t))
            for q in comps:
                c_t += q
                c_o.append(len(c_t))
            grp.append(len(c_o) - 1)
        self._new_result(stable, np.asarray(st_t, np.uint32), st_o)
        self._new_result(comp, np.asarray(c_t, np.uint32), c_o)
        self.groups[comp._obj.value] = np.asarray(grp, np.uint64)
        return 0

    def _special_ids(self, h):
        _, names, dec = self.engines[h.value]
        by_name = {b: r for r, b in dec.items()}
        return [by_name[nm.encode()] for nm in names]

    def b200bpe_result_groups(self, r, n):
        g = self.groups[getattr(r, "value", r)]
        n._obj.value = len(g) - 1
        return g.ctypes.data

    def b200bpe_last_unstable(self, h, v):
        return 0


@pytest.fixture()
def enc(monkeypatch):
    import __graft_entry__  # noqa: F401  (sys.path)
    from tiktoken_b200 import _lib, core
    stub = UnstableStub()
    monkeypatch.setattr(_lib, "lib", lambda: stub)
    monkeypatch.setattr(_lib, "last_error", lambda: "stub error")
    pat, ranks, special, _ = vu.load_encoding("cl100k_base", allow_real=False)
    e = core.Encoding("stub_unstable", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)
    return e, UnstableOracle(Oracle(ranks, special, pat), ranks, special), special


def test_special_policy_and_disallowed_message(enc):
    e, uo, special = enc
    sp = sorted(special)[0]
    texts = ["hello fanta", "x " + sp + " y", ""]
    with pytest.raises(ValueError, match="disallowed special token"):
        e.encode_with_unstable_batch(texts)
    assert e.encode_with_unstable_batch(texts, disallowed_special=()) == [uo.encode_with_unstable(t) for t in texts]
    assert e.encode_with_unstable_batch(texts, allowed_special="all") == [uo.encode_with_unstable(t, {sp}) for t in texts]
    assert e.encode_with_unstable_batch(texts, allowed_special={sp}) == [uo.encode_with_unstable(t, {sp}) for t in texts]


def test_surrogates_empty_batch_and_packed(enc):
    e, uo, _ = enc
    with pytest.raises(UnicodeEncodeError):
        e.encode_with_unstable_batch(["ok", "lone \ud800"])
    assert e.encode_with_unstable_batch([]) == []
    texts = ["The quick brown fox jumps", "é"]
    blob = "".join(texts).encode()
    off = np.asarray([0, len(texts[0].encode()), len(blob)], np.uint64)
    st, so, ct, co, grp = e.encode_with_unstable_packed(np.frombuffer(blob, np.uint8), off)
    for d, t in enumerate(texts):
        stable, comps = uo.encode_with_unstable(t)
        assert st[so[d]:so[d + 1]].tolist() == stable
        assert [ct[co[q]:co[q + 1]].tolist() for q in range(int(grp[d]), int(grp[d + 1]))] == comps


def test_per_text_method_still_raises(enc):
    e, _, _ = enc
    with pytest.raises(NotImplementedError):
        e.encode_with_unstable("hello fanta")
