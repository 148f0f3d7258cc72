"""CPU restatement of tiktoken's `bpe_train` (tools/train_oracle.c) over the C oracle's pre-tokeniser -- TEST
INFRASTRUCTURE ONLY.  The reference's Python loop costs O(merges x corpus) in the interpreter; this one trains on
megabyte corpora in seconds, so the GPU trainer can be checked at a scale that spans several chunks."""
from __future__ import annotations

import ctypes as C
import os
import subprocess

import numpy as np

from oracle import Oracle

_ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
_SRC = os.path.join(_ROOT, "tools", "train_oracle.c")
_SO = os.path.join(_ROOT, "tools", "libtrain_oracle.so")
_LIB = None


def build(force: bool = False) -> str:
    if force or not os.path.exists(_SO) or os.path.getmtime(_SO) < os.path.getmtime(_SRC):
        subprocess.check_call(["gcc", "-O2", "-fPIC", "-shared", "-Wall", "-std=c11", "-o", _SO, _SRC])
    return _SO


def _lib():
    global _LIB
    if _LIB is None:
        L = C.CDLL(build())
        L.tro_train.restype = C.c_int64
        L.tro_train.argtypes = [C.c_void_p, C.c_void_p, C.c_uint64, C.c_uint32, C.c_void_p, C.c_uint64, C.c_void_p]
        _LIB = L
    return _LIB


def _ptr(a: np.ndarray):
    return a.ctypes.data_as(C.c_void_p)


def split_packed(pat_str: str, text: np.ndarray, doc_off: np.ndarray) -> tuple[np.ndarray, np.ndarray]:
    """Pieces of every document, document by document -> (blob uint8, piece offsets uint64[n_pieces + 1])."""
    o = Oracle({}, {}, pat_str)
    text = np.ascontiguousarray(text, np.uint8)
    doc_off = np.asarray(doc_off, np.uint64)
    starts, ends = [], []
    for d in range(len(doc_off) - 1):
        lo, hi = int(doc_off[d]), int(doc_off[d + 1])
        n = hi - lo
        if n == 0:
            continue
        a = np.ascontiguousarray(text[lo:hi])
        st = np.zeros(n + 1, np.uint64); en = np.zeros(n + 1, np.uint64)
        k = o._L.orc_split(o._h, _ptr(a), n, _ptr(st), _ptr(en), n + 1)
        starts.append(st[:k] + lo); ends.append(en[:k] + lo)
    if not starts:
        return np.zeros(1, np.uint8), np.zeros(1, np.uint64)
    st = np.concatenate(starts); en = np.concatenate(ends)
    # the three patterns match every character, so the pieces tile the documents: the text is the blob
    assert np.array_equal(st[1:], en[:-1]) and int(st[0]) == 0 and int(en[-1]) == len(text)
    return (text if len(text) else np.zeros(1, np.uint8)), np.concatenate([st, en[-1:]]).astype(np.uint64)


class NoPairLeft(ValueError):
    pass


def train_merges(pat_str: str, text: np.ndarray, doc_off: np.ndarray, vocab_size: int):
    """-> (merges uint32[n, 3] of (left id, right id, merged id), distinct words).  NoPairLeft (a ValueError) when the
    pairs run out before vocab_size, like the reference's max() of an empty Counter."""
    if vocab_size < 256:
        raise ValueError("vocab_size must be at least 256, so we can encode all bytes")
    blob, off = split_packed(pat_str, text, doc_off)
    cap = max(0, vocab_size - 256) + 4096
    out = np.zeros(3 * cap + 3, np.uint32)
    nd = np.zeros(1, np.uint64)
    k = _lib().tro_train(_ptr(blob), _ptr(off), len(off) - 1, vocab_size, _ptr(out), cap, _ptr(nd))
    if k == -1:
        raise NoPairLeft("no pair left to merge before vocab_size was reached")
    if k < 0:
        raise RuntimeError(f"train_oracle failed ({k})")
    return out[:3 * k].reshape(k, 3), int(nd[0])


def ranks_from_merges(merges) -> dict[bytes, int]:
    """The reference's dict, insertion order included, from (left id, right id, merged id) triples."""
    ranks = {bytes([i]): i for i in range(256)}
    tok = [bytes([i]) for i in range(256)]
    for left, right, mid in np.asarray(merges, np.int64).reshape(-1, 3).tolist():
        b = tok[left] + tok[right]
        if b not in ranks:
            assert mid == len(tok)
            tok.append(b)
        else:
            assert tok[mid] == b
        ranks[b] = len(ranks)
    return ranks


def bpe_train(data: str, vocab_size: int, pat_str: str) -> dict[bytes, int]:
    b = data.encode("utf-8")
    text = np.frombuffer(b, np.uint8) if b else np.zeros(0, np.uint8)
    return ranks_from_merges(train_merges(pat_str, text, np.asarray([0, len(b)], np.uint64), vocab_size)[0])


def bpe_train_packed(text: np.ndarray, doc_off: np.ndarray, vocab_size: int, pat_str: str) -> dict[bytes, int]:
    return ranks_from_merges(train_merges(pat_str, text, doc_off, vocab_size)[0])
