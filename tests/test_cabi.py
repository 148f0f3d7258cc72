"""The C-ABI library loads without a GPU and exports every symbol include/b200bpe.h declares;
argument / pattern validation works without touching the device."""
import ctypes as C
import os
import re

import numpy as np
import pytest

import vocab_util as vu
from conftest import ROOT, have_gpu
from tiktoken_b200 import _lib


def declared_symbols():
    hdr = open(os.path.join(ROOT, "include", "b200bpe.h")).read()
    return sorted(set(re.findall(r"\b(b200bpe_[a-z_0-9]+)\s*\(", hdr)))


def test_library_builds_and_exports_every_declared_symbol():
    so = _lib.build()
    L = C.CDLL(so)
    syms = declared_symbols()
    assert len(syms) >= 15
    for s in syms:
        assert hasattr(L, s), f"{s} declared in include/b200bpe.h but not exported"
    assert sorted(_lib.EXPORTS) == syms
    assert b"sm_90a" in _lib.lib().b200bpe_version()


def test_unsupported_pattern_is_value_error():
    from tiktoken_b200 import _tiktoken
    with pytest.raises(ValueError):
        _tiktoken.CoreBPE({bytes([i]): i for i in range(256)}, {}, r"\w+|\s+")   # no CPU regex fallback


def test_special_token_id_of_2_pow_30_is_value_error():
    """Token ids must be below 2^30, special ones included (the probe kernel tags token slots with the top two bits);
    checked before the device is touched."""
    from tiktoken_b200 import _tiktoken
    ranks = {bytes([i]): i for i in range(256)}
    with pytest.raises(ValueError, match="special token id too large"):
        _tiktoken.CoreBPE(ranks, {"<|endoftext|>": 1 << 30}, vu.CL100K_PAT)


@pytest.mark.skipif(have_gpu(), reason="checks the no-GPU failure mode")
def test_no_gpu_fails_loudly_not_silently():
    from tiktoken_b200 import _tiktoken
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        _tiktoken.CoreBPE({bytes([i]): i for i in range(256)}, {}, vu.CL100K_PAT)


def test_product_package_does_not_import_the_oracle():
    pkg = os.path.join(ROOT, "tiktoken_b200")
    for dirpath, _, files in os.walk(pkg):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h", ".cpp")):
                src = open(os.path.join(dirpath, f), errors="replace").read()
                assert "import oracle" not in src and "from oracle" not in src and "liboracle" not in src, f


def test_pack_helper_matches_python_marshalling():
    """csrc/pack_ext.c (list[str] -> packed UTF-8 + offsets, token buffers -> list[list[int]])
    agrees with the pure-Python marshalling, including the UnicodeEncodeError on lone surrogates
    that tiktoken/core.py:77,128 relies on."""
    import numpy as np
    import __graft_entry__  # noqa: F401  (sys.path)
    from tiktoken_b200 import _tiktoken as T
    if T._b200pack is None:
        import __graft_entry__ as g
        g.build()
        import importlib
        importlib.reload(T)
    assert T._b200pack is not None
    docs = ["", "hello", "héllo 日本", "", "\U0001F600 x" * 50, "a" * 100000]
    arr, off = T.CoreBPE._pack(docs)
    enc = [d.encode() for d in docs]
    assert arr.tobytes() == b"".join(enc)
    assert off.tolist() == np.concatenate([[0], np.cumsum([len(e) for e in enc])]).tolist()
    arr0, off0 = T.CoreBPE._pack([])
    assert off0.tolist() == [0]
    with pytest.raises(UnicodeEncodeError):
        T.CoreBPE._pack(["ok", "\ud83d"])
    with pytest.raises(TypeError):
        T._b200pack.pack([b"bytes"])
    toks = (np.arange(10, dtype=np.uint64) * 400000003 % (1 << 32)).astype(np.uint32)
    toff = np.asarray([0, 0, 3, 3, 10], np.uint64)
    got = T._b200pack.unpack(toks.ctypes.data, toff.ctypes.data, 4)
    assert got == [[], toks[:3].tolist(), [], toks[3:].tolist()]


def test_packed_disallowed_special_scan_matches_the_regex_check():
    """_b200pack.find_first (the batch form of the disallowed-special check, tiktoken/core.py:120-124) against
    the per-document regex search it replaces; matches never straddle documents; the host class raises the
    reference's ValueError."""
    import random
    import regex
    import __graft_entry__  # noqa: F401  (sys.path)
    from tiktoken_b200 import _tiktoken as T, core
    assert T._b200pack is not None
    sp = ["<|endoftext|>", "<|fim_prefix|>", "<|fim_middle|>", "<|fim_suffix|>", "<|endofprompt|>"]
    rx = regex.compile("|".join(regex.escape(s) for s in sp))
    rnd = random.Random(1)
    frags = ["hello ", "<|", "|>", "<|endoftext", "<|endoftext|>", "<|fim_prefix|>", "<", "é<|endofprompt|>", "x" * 50, "\n"]
    for _ in range(1500):
        docs = ["".join(rnd.choice(frags) for _ in range(rnd.randint(0, 12))) for _ in range(rnd.randint(1, 6))]
        blob, offs = T._b200pack.pack(docs)
        got = T._b200pack.find_first(blob, offs, [s.encode() for s in sp])
        exp = None
        for d, t in enumerate(docs):
            m = rx.search(t)
            if m:
                exp = (d, sp.index(m.group()))
                break
        assert (got is None) == (exp is None) and (got is None or (got[0], got[1]) == exp), docs
        # needles with different first bytes take the memmem path
        got2 = T._b200pack.find_first(blob, offs, [b"hello", b"<|endoftext|>", b"x" * 50])
        exp2 = None
        for d, t in enumerate(docs):
            hits = [(t.encode().find(n), -len(n), i) for i, n in enumerate([b"hello", b"<|endoftext|>", b"x" * 50])
                    if t.encode().find(n) >= 0]
            if hits:
                exp2 = (d, min(hits)[2])
                break
        assert (got2 is None) == (exp2 is None) and (got2 is None or (got2[0], got2[1]) == exp2), docs
    blob, offs = T._b200pack.pack(["a<|endof", "text|>b"])
    assert T._b200pack.find_first(blob, offs, [b"<|endoftext|>"]) is None



def test_host_shim_construction_paths_with_a_stub_library(monkeypatch):
    """The two ways to build an engine (dict, as tiktoken/core.py:57 does, and flattened arrays parsed in C from a
    `.tiktoken` file) hand the SAME arrays to b200bpe_create, and the table-read methods / pickling state work
    from either.  The native library is stubbed (no GPU here); everything up to and after the call is real."""
    import base64
    import gzip
    import pickle
    import __graft_entry__  # noqa: F401  (sys.path)
    from tiktoken_b200 import _tiktoken as T, core

    captured = []

    class Stub:
        def b200bpe_create_multi(self, tb, to, tr, n, sb, so, sr, ns, pat, devs, n_dev, out):
            import ctypes as C2
            blob = bytes((C2.c_uint8 * 1).from_address(tb.value)) if n == 0 else None
            off = np.ctypeslib.as_array(C2.cast(to, C2.POINTER(C2.c_uint64)), shape=(n + 1,)).copy()
            rk = np.ctypeslib.as_array(C2.cast(tr, C2.POINTER(C2.c_uint32)), shape=(max(n, 1),))[:n].copy()
            data = np.ctypeslib.as_array(C2.cast(tb, C2.POINTER(C2.c_uint8)), shape=(max(int(off[-1]), 1),))[:int(off[-1])].copy()
            captured.append((data.tobytes(), off.tolist(), rk.tolist(), n, ns, pat, blob))
            return 0

        def b200bpe_destroy(self, h):
            pass

    monkeypatch.setattr(T._lib, "lib", lambda: Stub())
    path = os.path.join(ROOT, "tests", "golden", "vocab", "r50k_like.tiktoken.gz")
    data = gzip.open(path).read()
    ranks = {base64.b64decode(t): int(r) for t, r in (ln.split() for ln in data.splitlines() if ln)}
    special = {"<|endoftext|>": 50256}
    e1 = core.Encoding("by_dict", pat_str=vu.R50K_PAT, mergeable_ranks=ranks, special_tokens=special)
    e2 = core.Encoding.from_tiktoken_file("by_file", path, pat_str=vu.R50K_PAT, special_tokens=special,
                                          explicit_n_vocab=50257)
    e3 = core.Encoding.from_tiktoken_file("by_bytes", data, pat_str=vu.R50K_PAT, special_tokens=special)
    assert captured[0][:6] == captured[1][:6] == captured[2][:6]
    for e in (e1, e2, e3):
        assert e.n_vocab == 50257 and e.max_token_value == 50256
        assert e._core_bpe.encode_single_token(b"a") == ranks[b"a"]
        assert e._core_bpe.encode_single_token(b"<|endoftext|>") == 50256
        assert e._core_bpe.decode_single_token_bytes(ranks[b"th"] if b"th" in ranks else 97) in ranks
        assert e._core_bpe.token_byte_values() == sorted(ranks)
        assert e._mergeable_ranks == ranks
        state = e.__getstate__()
        assert state["mergeable_ranks"] == ranks and state["pat_str"] == vu.R50K_PAT
        e4 = pickle.loads(pickle.dumps(e))                      # by value: rebuilds through __init__
        assert e4._mergeable_ranks == ranks and e4.name == e.name
    with pytest.raises(ValueError):
        T.CoreBPE.from_flat(np.zeros(3, np.uint8), np.asarray([0, 5], np.uint64), np.asarray([1], np.uint32), {}, vu.R50K_PAT)
