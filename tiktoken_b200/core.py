"""`tiktoken_b200.Encoding` -- the reference's own host class (`tiktoken.core.Encoding`, which STAYS: special-token
policy, surrogate fix-up, decode helpers, pickling, ...) running on the GPU engine, with the batch methods
replaced by ONE native call per batch.

What this file adds to the inherited class, and nothing else:
  * the constructor builds `tiktoken_b200._tiktoken.CoreBPE` (ctypes -> libb200bpe.so -> sm_90a kernels) where
    the reference builds the Rust extension's (tiktoken/core.py:54-57), optionally on several GPUs (`devices=`);
  * `encode_ordinary_batch` / `encode_batch` / `decode_batch` / `decode_bytes_batch` make one native call for the
    whole batch instead of a ThreadPoolExecutor over per-document calls (core.py:161-203, :334-350); `num_threads`
    is accepted and ignored (the GPU is the pool); the disallowed-special check of `encode_batch` runs inside the same
    device scan that cuts the documents at allowed specials, instead of a Python regex search per document;
  * array-returning variants (`*_to_numpy`, `*_packed`) that never build Python lists;
  * `encode_bytes_batch` / `encode_bytes_packed`: the reference's `_encode_bytes` (src/py.rs:72-115) for a batch of
    documents that need not be UTF-8, on the device.
For a process that should run the UNMODIFIED reference package on the GPU engine, see `tiktoken_b200.install()`.
"""
from __future__ import annotations

import contextlib
import threading
from typing import AbstractSet, Collection, Literal, Sequence

import numpy as np
import tiktoken.core as _ref_core          # the reference's host side (tiktoken/core.py); only its native module is replaced

from . import _tiktoken

_swap_lock = threading.RLock()


class _NativeFor:
    """Stands in for the module `tiktoken._tiktoken` while a reference constructor runs (core.py:54)."""

    def __init__(self, device, devices):
        self._kw = {"device": device, "devices": devices}

    def CoreBPE(self, mergeable_ranks, special_tokens, pat_str):
        return _tiktoken.CoreBPE(mergeable_ranks, special_tokens, pat_str, **self._kw)


@contextlib.contextmanager
def _native(device=None, devices=None):
    with _swap_lock:
        old = _ref_core._tiktoken
        _ref_core._tiktoken = _NativeFor(device, devices)
        try:
            yield
        finally:
            _ref_core._tiktoken = old


def _fix_surrogates(text: str) -> str:
    # the reference's fix-up (core.py:77-80): lone surrogates become U+FFFD
    return text.encode("utf-16", "surrogatepass").decode("utf-16", "replace")


class Encoding(_ref_core.Encoding):
    def __init__(self, name: str, *, pat_str: str, mergeable_ranks: dict[bytes, int], special_tokens: dict[str, int],
                 explicit_n_vocab: int | None = None, device: int | None = None, devices: Sequence[int] | None = None):
        self._devices = list(devices) if devices is not None else None
        self._device = device
        with _native(device, self._devices):
            super().__init__(name, pat_str=pat_str, mergeable_ranks=mergeable_ranks, special_tokens=special_tokens,
                             explicit_n_vocab=explicit_n_vocab)
        # reference v0.14.0 core.py sets this in __init__; the 0.12.0 wheel's is_special_token reads it without setting it
        self._special_token_values = set(special_tokens.values())

    @classmethod
    def from_tiktoken_file(cls, name: str, path_or_bytes, *, pat_str: str, special_tokens: dict[str, int],
                           explicit_n_vocab: int | None = None, device: int | None = None,
                           devices: Sequence[int] | None = None) -> "Encoding":
        """An Encoding straight from a `.tiktoken` vocabulary file (`base64(token) rank` per line, the format
        `tiktoken/load.py:159-171` reads; `.gz` accepted), parsed in C into the flattened arrays the engine
        takes -- the 100-200 k-entry Python dict is only built if something asks for it (pickling by value,
        `encode_single_token`, `token_byte_values`)."""
        from ._tiktoken import _b200pack
        if isinstance(path_or_bytes, (bytes, bytearray, memoryview)):
            data = bytes(path_or_bytes)
        else:
            with open(path_or_bytes, "rb") as f:
                data = f.read()
        if data[:2] == b"\x1f\x8b":
            import gzip
            data = gzip.decompress(data)
        if _b200pack is None:                          # no C helper: the reference's own parse (load.py:159-171)
            import base64
            ranks = {base64.b64decode(tok): int(r) for tok, r in (ln.split() for ln in data.splitlines() if ln)}
            return cls(name, pat_str=pat_str, mergeable_ranks=ranks, special_tokens=special_tokens,
                       explicit_n_vocab=explicit_n_vocab, device=device, devices=devices)
        blob, off, rk = _b200pack.parse_tiktoken(data)
        blob, off, rk = np.frombuffer(blob, np.uint8), np.frombuffer(off, np.uint64), np.frombuffer(rk, np.uint32)
        self = cls.__new__(cls)
        self.name = name
        self._pat_str = pat_str
        self._ranks_dict = None
        self._special_tokens = special_tokens
        self._devices = list(devices) if devices is not None else None
        self._device = device
        self.max_token_value = max(int(rk.max()) if len(rk) else 0, max(special_tokens.values(), default=0))
        if explicit_n_vocab:
            assert len(rk) + len(special_tokens) == explicit_n_vocab
            assert self.max_token_value == explicit_n_vocab - 1
        self._special_token_values = set(special_tokens.values())
        self._core_bpe = _tiktoken.CoreBPE.from_flat(blob, off, rk, special_tokens, pat_str, device=device, devices=self._devices)
        return self

    # the reference keeps the dict it was given; an Encoding built from a file only builds it on demand
    @property
    def _mergeable_ranks(self) -> dict[bytes, int]:
        if self.__dict__.get("_ranks_dict") is None:
            self.__dict__["_ranks_dict"] = self._core_bpe._encoder
        return self.__dict__["_ranks_dict"]

    @_mergeable_ranks.setter
    def _mergeable_ranks(self, value: dict[bytes, int]) -> None:
        self.__dict__["_ranks_dict"] = value

    # ---------------------------------------------------------------- special-token policy (core.py:113-124)
    def _policy(self, allowed_special, disallowed_special):
        if allowed_special == "all":
            allowed_special = self.special_tokens_set
        if disallowed_special == "all":
            disallowed_special = self.special_tokens_set - allowed_special
        if disallowed_special and not isinstance(disallowed_special, frozenset):
            disallowed_special = frozenset(disallowed_special)
        return allowed_special, disallowed_special

    def _pack(self, texts: Sequence[str]):
        try:
            return self._core_bpe._pack(list(texts))
        except UnicodeEncodeError:
            return self._core_bpe._pack([_fix_surrogates(t) for t in texts])

    # ---------------------------------------------------------------- batch encode: one native call
    def encode_ordinary_batch(self, text: list[str], *, num_threads: int = 8) -> list[list[int]]:
        t, off = self._pack(text)
        return self._core_bpe._unpack(self._core_bpe.encode_ordinary_batch_buffer(t, off))

    def encode_batch_buffer(self, text: list[str], *, allowed_special: Literal["all"] | AbstractSet[str] = set(),  # noqa: B006
                            disallowed_special: Literal["all"] | Collection[str] = "all"):
        """`encode_batch` up to the zero-copy pinned TokenBuffer (tokens uint32[T] + offsets uint64[n_docs+1])."""
        allowed_special, disallowed_special = self._policy(allowed_special, disallowed_special)
        t, off = self._pack(text)
        try:
            return self._core_bpe.encode_batch_buffer(t, off, allowed_special, disallowed_special or ())
        except _tiktoken.DisallowedSpecial as e:
            _ref_core.raise_disallowed_special_token(e.token)        # the reference's message (core.py:438-447)

    def encode_batch(self, text: list[str], *, num_threads: int = 8,
                     allowed_special: Literal["all"] | AbstractSet[str] = set(),  # noqa: B006
                     disallowed_special: Literal["all"] | Collection[str] = "all") -> list[list[int]]:
        return self._core_bpe._unpack(self.encode_batch_buffer(text, allowed_special=allowed_special,
                                                               disallowed_special=disallowed_special))

    def encode_ordinary_batch_to_numpy(self, text: list[str]):
        """-> (tokens uint32[T], offsets uint64[n_docs+1]); document d is tokens[offsets[d]:offsets[d+1]]."""
        t, off = self._pack(text)
        with self._core_bpe.encode_ordinary_batch_buffer(t, off) as buf:
            return np.array(buf.tokens()), np.array(buf.offsets())

    def encode_ordinary_packed(self, text_bytes: np.ndarray, doc_off: np.ndarray):
        """Already-packed input: uint8[N] UTF-8 + uint64[n_docs+1] -> zero-copy TokenBuffer."""
        return self._core_bpe.encode_ordinary_batch_buffer(np.ascontiguousarray(text_bytes, np.uint8),
                                                           np.ascontiguousarray(doc_off, np.uint64))

    def encode_packed(self, text_bytes: np.ndarray, doc_off: np.ndarray, *,
                      allowed_special: Literal["all"] | AbstractSet[str] = set(),  # noqa: B006
                      disallowed_special: Literal["all"] | Collection[str] = "all"):
        """`encode_batch` on already-packed input -> zero-copy TokenBuffer (special tokens handled on the device)."""
        allowed_special, disallowed_special = self._policy(allowed_special, disallowed_special)
        try:
            return self._core_bpe.encode_batch_buffer(np.ascontiguousarray(text_bytes, np.uint8),
                                                      np.ascontiguousarray(doc_off, np.uint64), allowed_special,
                                                      disallowed_special or ())
        except _tiktoken.DisallowedSpecial as e:
            _ref_core.raise_disallowed_special_token(e.token)

    def encode_bytes_batch(self, data: Sequence[bytes], *, num_threads: int = 8) -> list[list[int]]:
        """`_encode_bytes` (core.py:406-407, src/py.rs:72-115) of every document, in one native call: a document that is
        not UTF-8 is encoded up to its first ill-formed byte, and the tokens of that prefix's last piece are re-encoded
        together with the rest of the document as one piece."""
        return self._core_bpe.encode_bytes_batch(list(data))

    def encode_bytes_packed(self, data: np.ndarray, doc_off: np.ndarray):
        """`encode_bytes_batch` on packed input: uint8[N] (any bytes) + uint64[n_docs+1] -> zero-copy TokenBuffer."""
        return self._core_bpe.encode_bytes_batch_buffer(np.ascontiguousarray(data, np.uint8),
                                                        np.ascontiguousarray(doc_off, np.uint64))

    def encode_with_unstable_batch(self, text: Sequence[str], *,
                                   allowed_special: Literal["all"] | AbstractSet[str] = set(),  # noqa: B006
                                   disallowed_special: Literal["all"] | Collection[str] = "all",
                                   num_threads: int = 8) -> list[tuple[list[int], list[list[int]]]]:
        """`encode_with_unstable` (core.py:208-243) of every text, in one native call: (stable tokens, completions) per
        text.  Each distinct completion comes once, at its first position in the reference's enumeration order (the
        reference returns them in hash-set order).  Lone surrogates raise UnicodeEncodeError, as the reference's
        `encode_with_unstable` does."""
        allowed_special, disallowed_special = self._policy(allowed_special, disallowed_special)
        try:
            return self._core_bpe.encode_with_unstable_batch(list(text), allowed_special, disallowed_special or ())
        except _tiktoken.DisallowedSpecial as e:
            _ref_core.raise_disallowed_special_token(e.token)

    def encode_with_unstable_packed(self, text_bytes: np.ndarray, doc_off: np.ndarray, *,
                                    allowed_special: Literal["all"] | AbstractSet[str] = set(),  # noqa: B006
                                    disallowed_special: Literal["all"] | Collection[str] = "all"):
        """`encode_with_unstable_batch` on packed UTF-8 (uint8[N] + uint64[n_docs+1]) -> (stable tokens uint32[T],
        stable offsets uint64[n_docs+1], completion tokens uint32[K], completion offsets uint64[n_completions+1],
        groups uint64[n_docs+1]); document d's completions are numbers groups[d] .. groups[d+1]-1."""
        allowed_special, disallowed_special = self._policy(allowed_special, disallowed_special)
        try:
            sbuf, cbuf = self._core_bpe.encode_with_unstable_batch_buffer(
                np.ascontiguousarray(text_bytes, np.uint8), np.ascontiguousarray(doc_off, np.uint64), allowed_special,
                disallowed_special or ())
        except _tiktoken.DisallowedSpecial as e:
            _ref_core.raise_disallowed_special_token(e.token)
        with sbuf, cbuf:
            return (np.array(sbuf.tokens()), np.array(sbuf.offsets()), np.array(cbuf.tokens()), np.array(cbuf.offsets()),
                    np.array(cbuf.groups()))

    # ---------------------------------------------------------------- batch decode: one native call
    def decode_batch(self, batch: Sequence[Sequence[int]], *, errors: str = "replace", num_threads: int = 8) -> list[str]:
        return [b.decode("utf-8", errors=errors) for b in self._core_bpe.decode_bytes_batch(batch)]

    def decode_bytes_batch(self, batch: Sequence[Sequence[int]], *, num_threads: int = 8) -> list[bytes]:
        return self._core_bpe.decode_bytes_batch(batch)

    def decode_packed(self, tokens: np.ndarray, tok_off: np.ndarray):
        """Array form: tokens uint32[T] + offsets uint64[n_docs+1] -> (bytes uint8[B], byte offsets uint64[n_docs+1])."""
        return self._core_bpe.decode_batch_buffer(tokens, tok_off)

    # ---------------------------------------------------------------- pickling (core.py:406-427)
    def __getstate__(self) -> object:
        from . import _REGISTRY
        if self is _REGISTRY.get(self.name):
            return self.name                      # encodings obtained from get_encoding pickle by reference
        return {"name": self.name, "pat_str": self._pat_str, "mergeable_ranks": self._mergeable_ranks,
                "special_tokens": self._special_tokens, "device": self._device, "devices": self._devices}

    def __setstate__(self, value: object) -> None:
        if isinstance(value, str):
            from . import get_encoding
            self.__dict__ = get_encoding(value).__dict__
            return
        self.__init__(**value)                    # rebuilds the device tables
