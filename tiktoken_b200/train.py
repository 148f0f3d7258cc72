"""BPE vocabulary training on the GPU: `tiktoken._educational.bpe_train` semantics (tiktoken/_educational.py:119-185).

    ranks = tiktoken_b200.bpe_train(text, 50_000, pat_str)                  # == bpe_train(text, 50_000, pat_str, visualise=None)
    ranks = tiktoken_b200.bpe_train_batch(docs, 50_000, pat_str)            # no piece crosses a document boundary
    ranks = tiktoken_b200.bpe_train_packed(text_u8, doc_off_u64, 50_000, pat_str)

The result is the reference's dict: the same keys, values and insertion order.  The split, the distinct-word stage and
the merge loop run on the device (kernels_train.cuh); the host rebuilds the dict from the device's merge list.
"""
from __future__ import annotations

import ctypes as C
import os
import threading
from typing import Sequence

import numpy as np

from . import _lib

# the pat_strs of tiktoken_ext/openai_public.py the pre-tokeniser implements (r50k/p50k, cl100k, o200k)
_R50K = r"""'(?:[sdmt]|ll|ve|re)| ?\p{L}++| ?\p{N}++| ?[^\s\p{L}\p{N}]++|\s++$|\s+(?!\S)|\s"""
_CL100K = r"""'(?i:[sdmt]|ll|ve|re)|[^\r\n\p{L}\p{N}]?+\p{L}++|\p{N}{1,3}+| ?[^\s\p{L}\p{N}]++[\r\n]*+|\s++$|\s*[\r\n]|\s+(?!\S)|\s"""
_O200K = "|".join([
    r"""[^\r\n\p{L}\p{N}]?[\p{Lu}\p{Lt}\p{Lm}\p{Lo}\p{M}]*[\p{Ll}\p{Lm}\p{Lo}\p{M}]+(?i:'s|'t|'re|'ve|'m|'ll|'d)?""",
    r"""[^\r\n\p{L}\p{N}]?[\p{Lu}\p{Lt}\p{Lm}\p{Lo}\p{M}]+[\p{Ll}\p{Lm}\p{Lo}\p{M}]*(?i:'s|'t|'re|'ve|'m|'ll|'d)?""",
    r"""\p{N}{1,3}""",
    r""" ?[^\s\p{L}\p{N}]+[\r\n/]*""",
    r"""\s*[\r\n]+""",
    r"""\s+(?!\S)""",
    r"""\s+""",
])
SUPPORTED_PATTERNS = (_R50K, _CL100K, _O200K)

# merges whose bytes already are a token do not grow the vocabulary; room for this many of them
_DUP_SLACK = 4096

_stats_lock = threading.Lock()
_last_stats: dict[str, float] = {}


def _check(vocab_size: int, pat_str: str) -> None:
    """The checks that need no device, in the reference's order: vocab_size first (_educational.py:123)."""
    if vocab_size < 2**8:
        raise ValueError("vocab_size must be at least 256, so we can encode all bytes")
    if pat_str not in SUPPORTED_PATTERNS:
        raise ValueError("unsupported pat_str: the GPU pre-tokeniser implements exactly the r50k/p50k, cl100k and o200k "
                         "patterns of tiktoken_ext/openai_public.py")


def _device(device: int | None) -> int:
    if device is None:
        return int(os.environ.get("B200BPE_DEVICE", os.environ.get("LOCAL_RANK", "0")))
    return int(device)


def _ranks_from_merges(merges: np.ndarray) -> dict[bytes, int]:
    """(left id, right id, merged id) per merge -> the reference's dict, insertion order included.  Each merge checks
    the device's id against the bytes: a new id for new bytes, the old id for bytes that already are a token."""
    ranks = {bytes([i]): i for i in range(256)}
    tok = list(ranks)
    for left, right, mid in merges.tolist():
        b = tok[left] + tok[right]
        if b in ranks:
            if mid >= len(tok) or tok[mid] != b:
                raise RuntimeError("internal: the device merged two different byte strings into one token")
        else:
            if mid != len(tok):
                raise RuntimeError("internal: the device gave existing bytes a new token id")
            tok.append(b)
        ranks[b] = len(ranks)           # an existing key keeps its place and takes the value len(ranks), like the reference
    return ranks


def bpe_train_packed(text_bytes: np.ndarray, doc_off: np.ndarray, vocab_size: int, pat_str: str, *,
                     device: int | None = None) -> dict[bytes, int]:
    """text_bytes uint8[N] (UTF-8 of all documents back to back), doc_off uint64[n_docs + 1].  Documents are split
    independently; the words are the pieces of document 0, then document 1, ..."""
    _check(vocab_size, pat_str)
    text = np.ascontiguousarray(text_bytes, np.uint8)
    if len(text) == 0:
        text = np.zeros(1, np.uint8)
    off = np.ascontiguousarray(doc_off, np.uint64)
    if len(off) < 1:
        raise ValueError("doc_off needs n_docs + 1 entries")
    if int(off[-1]) > len(text) or int(off[0]) != 0:
        raise ValueError("doc_off must start at 0 and end within text_bytes")
    cap = max(0, vocab_size - 256) + _DUP_SLACK
    merges = np.zeros(3 * cap + 3, np.uint32)
    n = C.c_uint64(0)
    stats = np.zeros(8, np.float64)
    L = _lib.lib()
    rc = L.b200bpe_bpe_train(text.ctypes.data, off.ctypes.data,
                             len(off) - 1, pat_str.encode("utf-8"), vocab_size, _device(device), merges.ctypes.data, cap,
                             C.byref(n), stats.ctypes.data)
    with _stats_lock:
        _last_stats.clear()
        _last_stats.update(zip(("pieces", "distinct_words", "merges", "graph_batches", "split_ms", "words_ms",
                                "merge_loop_ms", "chunks"), stats.tolist()))
    _lib.check(rc)
    return _ranks_from_merges(merges[:3 * n.value].reshape(-1, 3))


def bpe_train_batch(texts: Sequence[str], vocab_size: int, pat_str: str, *, device: int | None = None) -> dict[bytes, int]:
    """Train on several documents; UnicodeEncodeError on lone surrogates, like the reference's word.encode("utf-8")."""
    _check(vocab_size, pat_str)
    from ._tiktoken import CoreBPE
    text, off = CoreBPE._pack(list(texts))
    return bpe_train_packed(text, off, vocab_size, pat_str, device=device)


def bpe_train(data: str, vocab_size: int, pat_str: str, *, device: int | None = None) -> dict[bytes, int]:
    """`tiktoken._educational.bpe_train(data, vocab_size, pat_str, visualise=None)` on the GPU."""
    return bpe_train_batch([data], vocab_size, pat_str, device=device)


def last_train_stats() -> dict[str, float]:
    """What the most recent training call in this process did: pieces, distinct words, merges, graph batches, chunks,
    and device ms of the split, the distinct-word stage and the merge loop."""
    with _stats_lock:
        return dict(_last_stats)
