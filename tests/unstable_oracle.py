"""The reference's `CoreBPE::_encode_unstable_native` (src/lib.rs:483-599, with `encode` :375-442 and
`_increase_last_piece_token_len` :444-481) restated on top of the oracle's public entry points -- TEST INFRASTRUCTURE
ONLY, the checker of the completion search.

Per text: (tokens, L) = encode(text, allowed) where L = the tokens of the last regex piece of the final haystack (0 when
the text is empty or ends with an allowed special); L grows backwards over tokens made only of ' ', '\\n', '\\t' when the
first of the L is one (mergeable tokens only: the reference looks them up in `self.decoder`); U = their bytes; stable =
tokens[:-L].  Completions, in this order, each distinct one at its first position:
  (a) [t] for every token t whose bytes start with U, in byte order;
  (b) for i = 1 .. |U|-1 and every token t that starts with U[i:] (byte order): encode_ordinary(U[:i] + t) if that is
      UTF-8, else byte_pair_encode(U[:i] + t); kept up to the first token at which the byte count reaches |U|;
  (c) if |U| > 1 and U ends in a White_Space scalar after other bytes: byte_pair_encode(front) + byte_pair_encode(last).
A single byte the vocabulary lacks raises KeyError (the reference panics)."""
from __future__ import annotations

import bisect

import numpy as np

RANK_MAX = 0xFFFFFFFF
_SPACE = frozenset(b" \n\t")
# Rust char::is_whitespace
WHITE_SPACE = frozenset([*range(0x09, 0x0E), 0x20, 0x85, 0xA0, 0x1680, *range(0x2000, 0x200B), 0x2028, 0x2029, 0x202F,
                         0x205F, 0x3000])


def _is_utf8(b: bytes) -> bool:
    try:
        b.decode("utf-8")
        return True
    except UnicodeDecodeError:
        return False


class UnstableOracle:
    def __init__(self, oracle, mergeable_ranks: dict[bytes, int], special_tokens: dict[str, int]):
        self.o = oracle
        self.ranks = mergeable_ranks
        self.dec = {r: t for t, r in mergeable_ranks.items()}
        self.special_ids = frozenset(special_tokens.values())
        self.special_dec = {v: k.encode() for k, v in special_tokens.items()}
        self.sorted = sorted(mergeable_ranks)

    def _all_space(self, tok: int) -> bool:
        b = self.dec.get(tok)
        return b is not None and all(c in _SPACE for c in b)

    def _check(self, toks):
        if RANK_MAX in toks:
            raise KeyError("a piece needs a single-byte token that mergeable_ranks does not contain")
        return toks

    def byte_pair_encode(self, piece: bytes) -> list[int]:
        out = []
        for p in self.o.byte_pair_split(piece):
            if p not in self.ranks:
                raise KeyError(p)
            out.append(self.ranks[p])
        return out

    def _range(self, prefix: bytes):
        """the tokens (byte order) that start with prefix"""
        i = bisect.bisect_left(self.sorted, prefix)
        while i < len(self.sorted) and self.sorted[i].startswith(prefix):
            yield self.sorted[i]
            i += 1

    def stable_and_unstable(self, text: str, allowed_special=frozenset()):
        """-> (stable tokens, U)"""
        tokens = self._check(self.o.encode(text, allowed_special))
        if not text or not tokens or tokens[-1] in self.special_ids:
            return tokens, b""
        k = len(tokens)
        while k > 0 and tokens[k - 1] not in self.special_ids:
            k -= 1
        hay = b"".join(self.dec[t] for t in tokens[k:])
        L = len(self.o.encode_single_piece(self.o.split(hay)[-1]))
        if self._all_space(tokens[-L]):
            while L < len(tokens) and self._all_space(tokens[-L - 1]):
                L += 1
        U = b"".join(self.dec[t] if t in self.dec else self.special_dec[t] for t in tokens[len(tokens) - L:])
        return tokens[:len(tokens) - L], U

    def completions(self, U: bytes) -> list[list[int]]:
        if not U:
            return []
        seqs = [[self.ranks[t]] for t in self._range(U)]
        cands = []                       # (index into seqs, P, UTF-8?)
        for i in range(1, len(U)):
            for t in self._range(U[i:]):
                P = U[:i] + t
                cands.append((len(seqs), P, _is_utf8(P)))
                seqs.append(None)
        utf8 = [c for c in cands if c[2]]
        if utf8:                         # every UTF-8 candidate of the text in one oracle call
            blob = b"".join(c[1] for c in utf8)
            off = np.zeros(len(utf8) + 1, np.uint64)
            off[1:] = np.cumsum([len(c[1]) for c in utf8])
            tok, toff = self.o.encode_ordinary_batch_np(np.frombuffer(blob, np.uint8), off)
            for j, c in enumerate(utf8):
                seqs[c[0]] = self._check(tok[int(toff[j]):int(toff[j + 1])].tolist())
        for c in cands:
            if not c[2]:
                seqs[c[0]] = self.byte_pair_encode(c[1])
        for q, s in enumerate(seqs[len(seqs) - len(cands):], len(seqs) - len(cands)):
            keep, n = [], 0
            for t in s:
                keep.append(t)
                n += len(self.dec[t])
                if n >= len(U):
                    break
            seqs[q] = keep
        if len(U) > 1:
            last = U.decode("utf-8")[-1]
            front = U[:len(U) - len(last.encode("utf-8"))]
            if front and ord(last) in WHITE_SPACE:
                seqs.append(self.byte_pair_encode(front) + self.byte_pair_encode(last.encode("utf-8")))
        seen, out = set(), []
        for s in seqs:
            t = tuple(s)
            if t not in seen:
                seen.add(t)
                out.append(list(s))
        return out

    def encode_with_unstable(self, text: str, allowed_special=frozenset()):
        stable, U = self.stable_and_unstable(text, allowed_special)
        return stable, self.completions(U)
