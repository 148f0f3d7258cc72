"""The reference's `CoreBPE::_encode_bytes` (src/py.rs:72-115, with `_increase_last_piece_token_len`, src/lib.rs:444-481)
restated on top of the oracle's public entry points -- TEST INFRASTRUCTURE ONLY, the checker of the bytes mode.

For a document b with v = valid_up_to(b) (std::str::from_utf8; Python's strict decoder fails at the same byte):
  * v == len(b): encode_ordinary(b);
  * otherwise encode(b[:v], {}) -- the prefix is its own haystack, special-token text is ordinary text -- and take the
    tokens of its last regex piece, extended backwards over tokens made only of ' ', '\\n', '\\t' when the first of them
    is one; drop them, and encode decode_bytes(dropped) + b[v:] as ONE piece (whole-piece probe, then byte_pair_encode).
A single byte the vocabulary lacks comes back as the oracle's RANK_MAX token (0xFFFFFFFF), where the reference raises."""
from __future__ import annotations

import numpy as np

RANK_MAX = 0xFFFFFFFF
_SPACE = frozenset(b" \n\t")


def valid_up_to(data: bytes) -> int:
    """std::str::from_utf8(data).valid_up_to(), len(data) when the bytes are well-formed."""
    try:
        data.decode("utf-8")
        return len(data)
    except UnicodeDecodeError as e:
        return e.start


class BytesOracle:
    def __init__(self, oracle, mergeable_ranks: dict[bytes, int]):
        self.o = oracle
        self.dec = {r: t for t, r in mergeable_ranks.items()}

    def _all_space(self, tok: int) -> bool:
        b = self.dec.get(tok)
        return b is not None and all(c in _SPACE for c in b)

    def encode_bytes(self, data: bytes) -> list[int]:
        data = bytes(data)
        v = valid_up_to(data)
        if v == len(data):
            return self.o.encode_ordinary(data)
        prefix = data[:v]
        tokens = self.o.encode_ordinary(prefix)
        pieces = self.o.split(prefix)
        L = len(self.o.encode_single_piece(pieces[-1])) if pieces else 0
        if L and self._all_space(tokens[-L]):
            while L < len(tokens) and self._all_space(tokens[-L - 1]):
                L += 1
        unstable = b"".join(self.dec[t] for t in tokens[len(tokens) - L:]) + data[v:]
        return tokens[:len(tokens) - L] + self.o.encode_single_piece(unstable)

    def encode_bytes_batch_np(self, text: np.ndarray, doc_off: np.ndarray):
        """text uint8[N], doc_off uint64[n_docs+1] -> (tokens uint32[T], tok_off uint64[n_docs+1])"""
        text = np.ascontiguousarray(text, np.uint8)
        doc_off = np.ascontiguousarray(doc_off, np.uint64)
        raw = text.tobytes()
        t_ord, o_ord = self.o.encode_ordinary_batch_np(text, doc_off)
        parts, off = [], [0]
        for d in range(len(doc_off) - 1):
            doc = raw[int(doc_off[d]):int(doc_off[d + 1])]
            if valid_up_to(doc) == len(doc):
                part = t_ord[int(o_ord[d]):int(o_ord[d + 1])]
            else:
                part = np.asarray(self.encode_bytes(doc), np.uint32)
            parts.append(part)
            off.append(off[-1] + len(part))
        tokens = np.concatenate(parts).astype(np.uint32) if parts else np.zeros(0, np.uint32)
        return tokens, np.asarray(off, np.uint64)
