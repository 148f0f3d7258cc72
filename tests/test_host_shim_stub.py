"""The host side of the boundary (tiktoken_b200/core.py + _tiktoken.py: special-token policy, packing /
unpacking through the C helper, surrogate fix-up, batch methods, decode methods, pickling) run on the CPU
against a STUB of libb200bpe whose entry points are answered by the oracle.  This is a test of the host
mirror of tiktoken/core.py, not of the engine: the product never loads this stub, and the parity tests proper
(-m gpu) go through the real library.  It mirrors the reference's own API tests (tests/test_encoding.py,
tests/test_misc.py, tests/test_pickle.py) on the synthetic vocabularies."""
import ctypes as C
import pickle

import numpy as np
import pytest

import vocab_util as vu
from oracle import Oracle


class StubLib:
    """Just enough of include/b200bpe.h, with the oracle as the engine."""

    def __init__(self):
        self.engines, self.results, self.next_id = {}, {}, 1

    # --- helpers
    @staticmethod
    def _arr(ptr, ctype, n):
        if n == 0:
            return np.zeros(0, ctype)
        return np.ctypeslib.as_array(C.cast(ptr, C.POINTER(np.ctypeslib.as_ctypes_type(ctype))), shape=(n,)).copy()

    def _new_result(self, out, tokens, offsets):
        rid = self.next_id
        self.next_id += 1
        self.results[rid] = (np.ascontiguousarray(tokens), np.ascontiguousarray(offsets, np.uint64))
        out._obj.value = rid
        return 0

    # --- engine
    def b200bpe_create_multi(self, tb, to, tr, n, sb, so, sr, ns, pat, devs, n_dev, out):
        return self.b200bpe_create(tb, to, tr, n, sb, so, sr, ns, pat, 0, out)

    def b200bpe_create(self, tb, to, tr, n, sb, so, sr, ns, pat, dev, out):
        off = self._arr(to, np.uint64, n + 1)
        blob = self._arr(tb, np.uint8, int(off[-1])).tobytes()
        rk = self._arr(tr, np.uint32, n)
        ranks = {blob[int(off[i]):int(off[i + 1])]: int(rk[i]) for i in range(n)}
        soff = self._arr(so, np.uint64, ns + 1)
        sblob = self._arr(sb, np.uint8, int(soff[-1])).tobytes()
        srk = self._arr(sr, np.uint32, ns)
        names = [sblob[int(soff[i]):int(soff[i + 1])].decode() for i in range(ns)]
        special = {nm: int(srk[i]) for i, nm in enumerate(names)}
        pat = pat.decode()
        if pat not in (vu.R50K_PAT, vu.CL100K_PAT, vu.O200K_PAT):
            return -2
        eid = self.next_id
        self.next_id += 1
        dec = {v: k for k, v in ranks.items()}
        dec.update({v: k.encode() for k, v in special.items()})
        self.engines[eid] = (Oracle(ranks, special, pat), names, dec)
        out._obj.value = eid
        return 0

    def b200bpe_destroy(self, h):
        self.engines.pop(getattr(h, "value", h), None)

    def _docs(self, text, doc_off, n_docs):
        off = self._arr(doc_off, np.uint64, n_docs + 1)
        blob = self._arr(text, np.uint8, int(off[-1])).tobytes()
        return [blob[int(off[i]):int(off[i + 1])] for i in range(n_docs)]

    def b200bpe_encode_ordinary_batch(self, h, text, doc_off, n_docs, out):
        return self.b200bpe_encode_batch(h, text, doc_off, n_docs, None, out)

    def b200bpe_encode_batch(self, h, text, doc_off, n_docs, allowed, out):
        return self.b200bpe_encode_batch_special(h, text, doc_off, n_docs, allowed, out, None)

    def b200bpe_encode_batch_special(self, h, text, doc_off, n_docs, flags, out, bad):
        """flags: 1 = allowed, 2 = disallowed (the device scan's contract, include/b200bpe.h)."""
        o, names, _ = self.engines[h.value]
        allow, deny = set(), []
        if flags is not None:
            mask = self._arr(flags, np.uint8, len(names))
            allow = {nm for nm, m in zip(names, mask) if m == 1}
            deny = [(i, nm) for i, (nm, m) in enumerate(zip(names, mask)) if m == 2]
        docs = self._docs(text, doc_off, n_docs)
        if deny:                                              # leftmost occurrence in the packed batch
            best = None
            base = 0
            for d in docs:
                for i, nm in deny:
                    k = d.find(nm.encode())
                    if k >= 0 and (best is None or base + k < best[0]):
                        best = (base + k, i)
                base += len(d)
            if best is not None:
                bad._obj.value = best[1]
                return -7
        toks, offs = [], [0]
        for d in docs:
            t = o.encode(d.decode("utf-8"), allow) if allow else o.encode_ordinary(d)
            toks.extend(t)
            offs.append(len(toks))
        return self._new_result(out, np.asarray(toks, np.uint32), offs)

    def b200bpe_encode_single_piece(self, h, piece, n, out):
        o, _, _ = self.engines[h.value]
        t = o.encode_single_piece(self._arr(piece, np.uint8, n).tobytes())
        return self._new_result(out, np.asarray(t, np.uint32), [0, len(t)])

    def b200bpe_result_tokens(self, r):
        return self.results[getattr(r, "value", r)][0].ctypes.data

    def b200bpe_result_offsets(self, r):
        return self.results[getattr(r, "value", r)][1].ctypes.data

    def b200bpe_result_n_tokens(self, r):
        return len(self.results[getattr(r, "value", r)][0])

    def b200bpe_result_n_docs(self, r):
        return len(self.results[getattr(r, "value", r)][1]) - 1

    def b200bpe_result_free(self, r):
        self.results.pop(getattr(r, "value", r), None)

    def b200bpe_decode_bytes(self, h, tokens, n, out, cap, out_len, bad):
        _, _, dec = self.engines[h.value]
        data = bytearray()
        for t in self._arr(tokens, np.uint32, n).tolist():
            if t not in dec:
                bad._obj.value = t
                return -6
            data += dec[t]
        out_len._obj.value = len(data)
        if len(data) <= cap:
            C.memmove(out.value, bytes(data), len(data))
        return 0

    def b200bpe_decode_batch(self, h, tokens, tok_off, n_docs, out, bad):
        _, _, dec = self.engines[h.value]
        off = self._arr(tok_off, np.uint64, n_docs + 1)
        toks = self._arr(tokens, np.uint32, int(off[-1])).tolist()
        data, boff = bytearray(), [0]
        for d in range(n_docs):
            for t in toks[int(off[d]):int(off[d + 1])]:
                if t not in dec:
                    bad._obj.value = t
                    return -6
                data += dec[t]
            boff.append(len(data))
        return self._new_result(out, np.frombuffer(bytes(data), np.uint8), boff)


@pytest.fixture()
def enc(monkeypatch):
    import __graft_entry__  # noqa: F401  (sys.path)
    from tiktoken_b200 import _lib, core
    stub = StubLib()
    monkeypatch.setattr(_lib, "lib", lambda: stub)
    monkeypatch.setattr(_lib, "last_error", lambda: "stub error")
    pat, ranks, special, _ = vu.load_encoding("cl100k_base", allow_real=False)
    e = core.Encoding("stub_cl100k", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)
    return e, Oracle(ranks, special, pat), special, ranks


def test_encode_methods_agree_with_the_engine_answers(enc):
    e, o, special, _ = enc
    docs = ["hello world", "", "  leading", "日本語のテキスト、です。", "it's 12345 o'clock\n\n", "x" * 300]
    assert [e.encode_ordinary(d) for d in docs] == [o.encode_ordinary(d) for d in docs]
    assert e.encode_ordinary_batch(docs) == [o.encode_ordinary(d) for d in docs]
    assert e.encode_batch(docs) == [o.encode_ordinary(d) for d in docs]
    toks, offs = e.encode_ordinary_batch_to_numpy(docs)
    assert toks.dtype == np.uint32 and offs.dtype == np.uint64 and len(offs) == len(docs) + 1
    assert [toks[int(offs[i]):int(offs[i + 1])].tolist() for i in range(len(docs))] == e.encode_ordinary_batch(docs)
    assert e.encode_to_numpy("hello world").tolist() == o.encode_ordinary("hello world")
    assert e.encode_ordinary_batch([]) == [] and e.encode_batch([]) == []


def test_special_token_policy_as_in_the_reference(enc):
    e, o, special, _ = enc
    s = "hello <|endoftext|> a  <|fim_prefix|>b"
    with pytest.raises(ValueError, match="disallowed special token"):
        e.encode(s)                                              # tiktoken/core.py:120-124
    with pytest.raises(ValueError, match="disallowed special token '<\\|endoftext\\|>'"):
        e.encode_batch(["fine", s])                              # the packed C scan, same error
    with pytest.raises(ValueError):
        e.encode_batch(["fine", s], allowed_special={"<|fim_prefix|>"})
    assert e.encode(s, disallowed_special=()) == e.encode_ordinary(s)
    assert e.encode(s, allowed_special="all") == o.encode(s, set(special))
    assert e.encode_batch([s, "x"], allowed_special="all") == [o.encode(s, set(special)), o.encode_ordinary("x")]
    only = {"<|endoftext|>"}
    assert e.encode_batch([s], allowed_special=only, disallowed_special=()) == [o.encode(s, only)]
    assert e.encode("<|endoftext|>", allowed_special="all") == [special["<|endoftext|>"]]
    assert e.eot_token == special["<|endoftext|>"] and e.special_tokens_set == set(special)
    assert e.is_special_token(special["<|endoftext|>"]) and not e.is_special_token(5)


def test_surrogates_are_replaced_like_the_reference(enc):
    e, o, _, _ = enc
    assert e.encode_ordinary("\ud83d") == o.encode_ordinary("�")       # tests/test_encoding.py:103-111
    assert e.encode("a\ud83db", disallowed_special=()) == o.encode_ordinary("a�b")
    assert e.encode_ordinary_batch(["ok", "👍", "\ud83d"]) == [
        o.encode_ordinary("ok"), o.encode_ordinary("\U0001f44d"), o.encode_ordinary("�")]


def test_decode_methods_and_errors(enc):
    e, o, special, ranks = enc
    docs = ["hello world", "", "日本語 ✓", "a\nb"]
    toks = e.encode_ordinary_batch(docs)
    assert [e.decode(t) for t in toks] == docs
    assert e.decode_batch(toks) == docs
    assert e.decode_bytes_batch(toks) == [d.encode() for d in docs]
    assert e.decode_bytes(toks[0]) == b"hello world"
    assert b"".join(e.decode_tokens_bytes(toks[2])) == docs[2].encode()
    text, offsets = e.decode_with_offsets(toks[0])
    assert text == docs[0] and offsets[0] == 0 and len(offsets) == len(toks[0])
    assert e.decode_single_token_bytes(ranks[b"a"]) == b"a"
    assert e.decode([special["<|endoftext|>"]]) == "<|endoftext|>"
    with pytest.raises(KeyError):
        e.decode_bytes([e.n_vocab + 5])
    with pytest.raises(KeyError):
        e.decode_batch([[1], [e.n_vocab + 5]])
    with pytest.raises(KeyError):
        e.decode_single_token_bytes(e.n_vocab + 5)
    data, boff = e.decode_packed(np.asarray(toks[0] + toks[2], np.uint32), np.asarray([0, len(toks[0]), len(toks[0]) + len(toks[2])], np.uint64))
    assert data.tobytes() == (docs[0] + docs[2]).encode() and boff.tolist() == [0, len(docs[0].encode()), len((docs[0] + docs[2]).encode())]


def test_single_token_and_piece_helpers(enc):
    e, o, special, ranks = enc
    assert e.encode_single_token("a") == ranks[b"a"] and e.encode_single_token(b"a") == ranks[b"a"]
    assert e.encode_single_token("<|endoftext|>") == special["<|endoftext|>"]
    with pytest.raises(KeyError):
        e.encode_single_token("definitely not one token \x00\x01")
    assert e._encode_single_piece("hello") == o.encode_single_piece(b"hello")
    assert e._encode_only_native_bpe("hello world 123") == o.encode_ordinary("hello world 123")
    assert e.token_byte_values() == sorted(ranks)
    assert e._encode_bytes(b"hello") == o.encode_ordinary("hello")
    with pytest.raises(NotImplementedError):
        e._encode_bytes(b"\xff\xfe")
    with pytest.raises(NotImplementedError):
        e.encode_with_unstable("hello")


def test_pickle_by_value_rebuilds_the_engine(enc):
    e, o, _, _ = enc
    e2 = pickle.loads(pickle.dumps(e))                           # tests/test_pickle.py
    assert e2.name == e.name and e2.encode_ordinary("hello world") == o.encode_ordinary("hello world")


def test_registry_is_the_references_and_pickles_by_reference(enc, monkeypatch):
    """`tiktoken_b200.get_encoding` serves the constructors the reference's own registry discovers among the
    `tiktoken_ext` plugins (tiktoken/registry.py) -- here one more entry, as a plugin would publish it -- builds the
    GPU-backed class once per name and pickles it by name (tiktoken/core.py:409-417)."""
    import tiktoken.registry as ref_registry
    import tiktoken_b200
    pat, ranks, special, _ = vu.load_encoding("r50k_base", allow_real=False)
    calls = []

    def ctor():
        calls.append(1)
        return {"name": "r50k_like_local", "pat_str": pat, "mergeable_ranks": ranks, "special_tokens": special}

    tiktoken_b200.list_encoding_names()                          # plugin discovery by the reference's code
    monkeypatch.setitem(ref_registry.ENCODING_CONSTRUCTORS, "r50k_like_local", ctor)
    monkeypatch.setattr(tiktoken_b200, "_REGISTRY", {})
    assert "r50k_like_local" in tiktoken_b200.list_encoding_names() and "cl100k_base" in tiktoken_b200.list_encoding_names()
    e = tiktoken_b200.get_encoding("r50k_like_local")
    assert isinstance(e, tiktoken_b200.Encoding) and tiktoken_b200.get_encoding("r50k_like_local") is e and len(calls) == 1
    assert pickle.dumps(e) == pickle.dumps(e) and len(pickle.dumps(e)) < 400          # by reference, not 50 k tokens
    assert pickle.loads(pickle.dumps(e)).encode_ordinary("hello") == e.encode_ordinary("hello")
    with pytest.raises(ValueError, match="Unknown encoding"):
        tiktoken_b200.get_encoding("no_such_encoding")
    with pytest.raises(ValueError):
        tiktoken_b200.get_encoding(5)


def test_install_swaps_the_native_module_under_the_reference_package(enc, monkeypatch):
    import tiktoken
    import tiktoken.core
    import tiktoken_b200
    from tiktoken_b200 import _tiktoken as shim
    monkeypatch.setattr(tiktoken.core, "_tiktoken", tiktoken.core._tiktoken)     # restored after the test
    tiktoken_b200.install()
    pat, ranks, special, _ = vu.load_encoding("cl100k_base", allow_real=False)
    e = tiktoken.Encoding("ref_on_b200", pat_str=pat, mergeable_ranks=ranks, special_tokens=special)
    assert isinstance(e._core_bpe, shim.CoreBPE)
    assert e.encode("hello <|endoftext|>", allowed_special="all") == enc[1].encode("hello <|endoftext|>", set(special))
