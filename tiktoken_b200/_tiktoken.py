"""Drop-in for tiktoken's native module `tiktoken._tiktoken` (reference: src/py.rs).

`CoreBPE(mergeable_ranks, special_tokens, pat_str)` has the constructor and the methods
`tiktoken/core.py` calls on `self._core_bpe` (core.py:57,76,127,161,259,273,301,358,393),
plus two batched entry points (`encode_ordinary_batch`, `encode_batch`) that the host class
uses instead of a thread pool: one native call per batch, executed by hand-written sm_90a
kernels through the C ABI of libb200bpe.so.  No CPU fallback exists.
"""
from __future__ import annotations

import ctypes as C
import threading

import numpy as np

from . import _lib

try:                                    # C marshalling helper (csrc/pack_ext.c), built by __graft_entry__.build()
    from . import _b200pack
except ImportError:                     # host marshalling only -- the kernels never depend on it
    _b200pack = None


def _ptr(a: np.ndarray):
    return C.c_void_p(a.ctypes.data)


def _flatten_bytes(items: list[bytes]):
    blob = b"".join(items)
    off = np.zeros(len(items) + 1, dtype=np.uint64)
    if items:
        np.cumsum(np.fromiter((len(b) for b in items), dtype=np.uint64, count=len(items)), out=off[1:])
    arr = np.frombuffer(blob, dtype=np.uint8) if blob else np.zeros(1, np.uint8)
    return arr, off


class _NativeView:
    """Exposes native memory through the array interface and keeps its TokenBuffer alive for as long as
    any ndarray built on it exists (np.asarray(view).base is this object)."""

    def __init__(self, owner, ptr: int, n: int, typestr: str):
        self._owner = owner
        self.__array_interface__ = {"data": (ptr, True), "shape": (n,), "typestr": typestr, "version": 3}


class TokenBuffer:
    """Owns one native result; exposes tokens / offsets without copying (the role of TiktokenBuffer,
    src/py.rs:186-249).  Lifetime: the buffer holds its CoreBPE, and every array handed out holds the buffer,
    so neither `enc.encode_ordinary_packed(t, o).tokens()` nor dropping the Encoding first can dangle (the
    native handle is reference-counted as well: b200bpe_destroy defers to the last b200bpe_result_free).
    `close()` frees the native memory NOW: arrays obtained before it must not be used afterwards."""

    def __init__(self, L, handle, owner=None):
        self._L, self._h, self._owner = L, handle, owner
        self.n_tokens = int(L.b200bpe_result_n_tokens(handle))
        self.n_docs = int(L.b200bpe_result_n_docs(handle))

    def tokens(self) -> np.ndarray:
        if self.n_tokens == 0 or not self._h:
            return np.zeros(0, np.uint32)
        p = self._L.b200bpe_result_tokens(self._h)
        return np.asarray(_NativeView(self, int(p), self.n_tokens, "<u4"))

    def offsets(self) -> np.ndarray:
        if not self._h:
            raise ValueError("TokenBuffer is closed")
        p = self._L.b200bpe_result_offsets(self._h)
        return np.asarray(_NativeView(self, int(p), self.n_docs + 1, "<u8"))

    def close(self):
        if self._h:
            self._L.b200bpe_result_free(self._h)
            self._h = None
        self._owner = None

    def __enter__(self):
        return self

    def __exit__(self, *exc):
        self.close()

    def __del__(self):
        self.close()


class CompletionBuffer(TokenBuffer):
    """The completions of `encode_with_unstable_batch_buffer`: `tokens()` holds every completion's tokens back to back,
    `offsets()` their boundaries (`n_docs` is the number of completions), `groups()` per input document the range of
    its completions (uint64[n_inputs + 1])."""

    def groups(self) -> np.ndarray:
        if not self._h:
            raise ValueError("CompletionBuffer is closed")
        n = C.c_uint64(0)
        p = self._L.b200bpe_result_groups(self._h, C.byref(n))
        return np.asarray(_NativeView(self, int(p), int(n.value) + 1, "<u8"))


class DisallowedSpecial(ValueError):
    """The text contains a special token that the call disallows; `.token` names it.  The host class turns it into
    the reference's message (tiktoken/core.py:431-438)."""

    def __init__(self, token: str):
        super().__init__(f"Encountered text corresponding to disallowed special token {token!r}.")
        self.token = token


class CoreBPE:
    def __init__(self, mergeable_ranks: dict[bytes, int], special_tokens: dict[str, int], pat_str: str,
                 device: int | None = None, devices: list[int] | None = None):
        """Same positional arguments as the reference's `CoreBPE(encoder, special_tokens_encoder, pattern)`
        (src/py.rs:16-23).  `device` / `devices` (keyword, optional) choose the GPU(s): one engine can span several
        GPUs of the box (b200bpe_create_multi), documents then shard over them inside every batch call."""
        toks = list(mergeable_ranks.keys())
        blob, off = _flatten_bytes(toks)
        ranks = np.fromiter((mergeable_ranks[t] for t in toks), dtype=np.uint32, count=len(toks))
        self._create(blob, off, ranks, special_tokens, pat_str, device, devices)
        self._encoder_dict = mergeable_ranks

    @classmethod
    def from_flat(cls, tok_bytes: np.ndarray, tok_off: np.ndarray, tok_rank: np.ndarray, special_tokens: dict[str, int],
                  pat_str: str, device: int | None = None, devices: list[int] | None = None) -> "CoreBPE":
        """Construct from the flattened vocabulary (token i = tok_bytes[tok_off[i]:tok_off[i+1]], rank
        tok_rank[i]) -- what `_b200pack.parse_tiktoken` produces from a `.tiktoken` file -- without a Python
        dict of 100-200 k bytes objects ("next" row: vocabulary parsing, tiktoken/load.py:159-171).  The dict the
        table-read methods need is built on first use."""
        self = cls.__new__(cls)
        blob = np.ascontiguousarray(tok_bytes, np.uint8)
        off = np.ascontiguousarray(tok_off, np.uint64)
        ranks = np.ascontiguousarray(tok_rank, np.uint32)
        if len(off) != len(ranks) + 1 or (len(off) and int(off[-1]) > len(blob)):
            raise ValueError("inconsistent flattened vocabulary")
        self._create(blob if len(blob) else np.zeros(1, np.uint8), off, ranks, special_tokens, pat_str, device, devices)
        self._encoder_dict = None
        self._flat = (blob, off, ranks)
        return self

    def _create(self, blob: np.ndarray, off: np.ndarray, ranks: np.ndarray, special_tokens: dict[str, int], pat_str: str,
                device: int | None, devices: list[int] | None = None):
        L = _lib.lib()
        self._L = L
        n_tok = len(ranks)
        self._special_names = list(special_tokens.keys())
        sblob, soff = _flatten_bytes([s.encode("utf-8") for s in self._special_names])
        sranks = np.asarray([special_tokens[s] for s in self._special_names], dtype=np.uint32)
        if len(sranks) == 0:
            sranks = np.zeros(1, np.uint32)
        if devices is None:
            if device is None:
                import os
                device = int(os.environ.get("B200BPE_DEVICE", os.environ.get("LOCAL_RANK", "0")))
            devices = [int(device)]
        devs = np.asarray(list(devices), dtype=np.int32)
        h = C.c_void_p()
        rc = L.b200bpe_create_multi(_ptr(blob), _ptr(off), _ptr(ranks if n_tok else np.zeros(1, np.uint32)),
                                    n_tok, _ptr(sblob), _ptr(soff), _ptr(sranks), len(self._special_names),
                                    pat_str.encode("utf-8"), _ptr(devs), len(devs), C.byref(h))
        _lib.check(rc)                      # ValueError for an unsupported pat_str / duplicate ranks
        self._h = h
        self.device = int(devs[0])
        self.devices = [int(d) for d in devs]
        self._special = special_tokens
        self._n_ids = max(int(ranks.max()) + 1 if n_tok else 0, max(special_tokens.values(), default=-1) + 1)   # ids are < this
        self._int_cache = None
        self._decoder = None
        self._flat = None
        self._lock = threading.Lock()

    @property
    def _encoder(self) -> dict[bytes, int]:
        if self._encoder_dict is None:
            blob, off, ranks = self._flat
            raw, o = blob.tobytes(), off.tolist()
            self._encoder_dict = {raw[o[i]:o[i + 1]]: r for i, r in enumerate(ranks.tolist())}
        return self._encoder_dict

    def __del__(self):
        h = getattr(self, "_h", None)
        if h:
            self._L.b200bpe_destroy(h)
            self._h = None

    # ---- batched native calls (replace ThreadPoolExecutor fan-out, core.py:164-206) ----------
    def encode_ordinary_batch_buffer(self, text: np.ndarray, doc_off: np.ndarray) -> TokenBuffer:
        """text: uint8[N] concatenated UTF-8, doc_off: uint64[n_docs+1] -> TokenBuffer."""
        res = C.c_void_p()
        rc = self._L.b200bpe_encode_ordinary_batch(self._h, _ptr(text), _ptr(doc_off), len(doc_off) - 1,
                                                   C.byref(res))
        _lib.check(rc)
        return TokenBuffer(self._L, res, self)

    def encode_batch_buffer(self, text: np.ndarray, doc_off: np.ndarray, allowed_special, disallowed_special=()) -> TokenBuffer:
        """CoreBPE::encode for a batch (lib.rs:375-442) plus, when `disallowed_special` is given, the check that
        `Encoding.encode` runs first (core.py:120-124) -- one device scan for both.  Raises the reference's
        ValueError (through `disallowed_error`) naming the leftmost disallowed special."""
        flags = self._special_flags(allowed_special, disallowed_special)
        res = C.c_void_p()
        bad = C.c_int32(-1)
        rc = self._L.b200bpe_encode_batch_special(self._h, _ptr(text), _ptr(doc_off), len(doc_off) - 1, _ptr(flags),
                                                  C.byref(res), C.byref(bad))
        if rc == _lib.ESPECIAL:
            raise DisallowedSpecial(self._special_names[bad.value])
        _lib.check(rc)
        return TokenBuffer(self._L, res, self)

    def _special_flags(self, allowed_special, disallowed_special) -> np.ndarray:
        flags = np.zeros(len(self._special_names) + 1, np.uint8)
        for i, s in enumerate(self._special_names):
            if s in allowed_special:
                flags[i] = 1
            elif s in disallowed_special:
                flags[i] = 2
        return flags

    def encode_with_unstable_batch_buffer(self, text: np.ndarray, doc_off: np.ndarray, allowed_special,
                                          disallowed_special=()) -> tuple[TokenBuffer, CompletionBuffer]:
        """CoreBPE::_encode_unstable_native (lib.rs:483-599) for every document, with the disallowed check of
        encode_batch_buffer: (stable tokens, completions).  Each distinct completion of a document comes once, at its
        first position in the reference's enumeration order."""
        flags = self._special_flags(allowed_special, disallowed_special)
        stable, comp = C.c_void_p(), C.c_void_p()
        bad = C.c_int32(-1)
        rc = self._L.b200bpe_encode_with_unstable_batch(self._h, _ptr(text if len(text) else np.zeros(1, np.uint8)),
                                                        _ptr(doc_off), len(doc_off) - 1, _ptr(flags), C.byref(stable),
                                                        C.byref(comp), C.byref(bad))
        if rc == _lib.ESPECIAL:
            raise DisallowedSpecial(self._special_names[bad.value])
        _lib.check(rc)
        return TokenBuffer(self._L, stable, self), CompletionBuffer(self._L, comp, self)

    def encode_with_unstable_batch(self, texts: list[str], allowed_special, disallowed_special=()):
        """-> [(stable tokens, [completion, ...]), ...]; UnicodeEncodeError on lone surrogates (py.rs:120 takes &str)."""
        text, off = self._pack(texts)
        sbuf, cbuf = self.encode_with_unstable_batch_buffer(text, off, allowed_special, disallowed_special)
        grp = cbuf.groups().tolist()
        stable = self._unpack(sbuf)
        comps = self._unpack(cbuf)
        return [(stable[d], comps[grp[d]:grp[d + 1]]) for d in range(len(stable))]

    def encode_bytes_batch_buffer(self, text: np.ndarray, doc_off: np.ndarray) -> TokenBuffer:
        """CoreBPE::_encode_bytes (src/py.rs:72-115) for every document: text uint8[N] need not be UTF-8, doc_off
        uint64[n_docs+1] -> TokenBuffer.  Well-formed documents get exactly the tokens of encode_ordinary_batch_buffer;
        KeyError when an unstable piece needs a single byte the vocabulary lacks."""
        res = C.c_void_p()
        rc = self._L.b200bpe_encode_bytes_batch(self._h, _ptr(text if len(text) else np.zeros(1, np.uint8)), _ptr(doc_off),
                                                len(doc_off) - 1, C.byref(res))
        _lib.check(rc)
        return TokenBuffer(self._L, res, self)

    def encode_bytes_batch(self, docs: list[bytes]) -> list[list[int]]:
        text, off = _flatten_bytes([bytes(d) for d in docs])
        return self._unpack(self.encode_bytes_batch_buffer(text, off))

    @staticmethod
    def _pack(texts: list[str]):
        """list[str] -> (uint8 blob, uint64 offsets); UnicodeEncodeError on lone surrogates, like the
        `&str` extraction of py.rs:30,36 (core.py:77,128 catch it and retry)."""
        if _b200pack is not None:
            blob, offs = _b200pack.pack(texts)
            arr = np.frombuffer(blob, dtype=np.uint8) if blob else np.zeros(1, np.uint8)
            return arr, np.frombuffer(offs, dtype=np.uint64)
        enc = [t.encode("utf-8") for t in texts]
        return _flatten_bytes(enc)

    def _unpack(self, buf: TokenBuffer) -> list[list[int]]:
        if _b200pack is not None and buf.n_tokens:
            cache = self._int_cache
            if cache is None:                     # the int objects of all token ids, shared by every list this engine returns
                cache = self._int_cache = list(range(min(int(self._n_ids), 1 << 20)))
            out = _b200pack.unpack(buf.tokens().ctypes.data, buf.offsets().ctypes.data, buf.n_docs, cache)
            buf.close()
            return out
        toks = buf.tokens().tolist()
        off = buf.offsets().tolist()
        out = [toks[off[i]:off[i + 1]] for i in range(buf.n_docs)]
        buf.close()
        return out

    def encode_ordinary_batch(self, texts: list[str]) -> list[list[int]]:
        text, off = self._pack(texts)
        return self._unpack(self.encode_ordinary_batch_buffer(text, off))

    def encode_batch(self, texts: list[str], allowed_special) -> list[list[int]]:
        text, off = self._pack(texts)
        return self._unpack(self.encode_batch_buffer(text, off, allowed_special))

    # ---- the per-text methods of src/py.rs -----------------------------------------------------
    def encode_ordinary(self, text: str) -> list[int]:                      # py.rs:29-32
        return self.encode_ordinary_batch([text])[0]

    def encode(self, text: str, allowed_special) -> list[int]:              # py.rs:34-49
        return self.encode_batch([text], allowed_special)[0]

    def encode_to_tiktoken_buffer(self, text: str, allowed_special):        # py.rs:51-70
        t, off = self._pack([text])
        buf = self.encode_batch_buffer(t, off, allowed_special)
        arr = np.array(buf.tokens(), dtype=np.uint32)                      # 1-D 'I' buffer, read-only
        buf.close()
        arr.flags.writeable = False
        return arr

    def encode_single_piece(self, piece: bytes) -> list[int]:               # py.rs:145-150
        if len(piece) == 0:
            return []
        a = np.frombuffer(piece, dtype=np.uint8)
        res = C.c_void_p()
        _lib.check(self._L.b200bpe_encode_single_piece(self._h, _ptr(a), len(piece), C.byref(res)))
        buf = TokenBuffer(self._L, res, self)
        out = buf.tokens().tolist()
        buf.close()
        return out

    def encode_single_token(self, piece: bytes) -> int:                     # py.rs:133-143 (table read)
        r = self._encoder.get(bytes(piece))
        if r is not None:
            return r
        try:
            s = bytes(piece).decode("utf-8")
        except UnicodeDecodeError:
            raise KeyError(bytes(piece)) from None
        if s in self._special:
            return self._special[s]
        raise KeyError(bytes(piece))

    def _encode_bytes(self, data: bytes) -> list[int]:                      # py.rs:72-115
        try:
            text = data.decode("utf-8")
        except UnicodeDecodeError:
            raise NotImplementedError(
                "_encode_bytes on invalid UTF-8 (unstable-token path, src/py.rs:79-112) is out of scope "
                "of the GPU encoder") from None
        return self.encode_ordinary(text)

    def encode_with_unstable(self, text: str, allowed_special):             # py.rs:117-131
        raise NotImplementedError("encode_with_unstable (completion search, src/lib.rs:444-599) is out of scope")

    def decode_bytes(self, tokens) -> bytes:                                 # py.rs:156-162
        arr = np.ascontiguousarray(np.asarray(tokens, dtype=np.uint32))
        n = len(arr)
        if n == 0:
            return b""
        out_len = C.c_uint64(0)
        bad = C.c_uint32(0)
        cap = max(64, 8 * n)
        while True:
            out = np.empty(cap, np.uint8)
            rc = self._L.b200bpe_decode_bytes(self._h, _ptr(arr), n, _ptr(out), cap, C.byref(out_len), C.byref(bad))
            if rc == _lib.EKEY:
                raise KeyError(f"Invalid token for decoding: {bad.value}")
            _lib.check(rc)
            if out_len.value <= cap:
                return out[:out_len.value].tobytes()
            cap = int(out_len.value)

    def decode_batch_buffer(self, tokens: np.ndarray, tok_off: np.ndarray):
        """Device gather ("next" row): tokens uint32[T] + tok_off uint64[n_docs+1] -> (bytes uint8[B], byte_off
        uint64[n_docs+1]).  KeyError on an unknown id, like decode_bytes."""
        tokens = np.ascontiguousarray(tokens, np.uint32)
        tok_off = np.ascontiguousarray(tok_off, np.uint64)
        res = C.c_void_p()
        bad = C.c_uint32(0)
        rc = self._L.b200bpe_decode_batch(self._h, _ptr(tokens if len(tokens) else np.zeros(1, np.uint32)), _ptr(tok_off),
                                          len(tok_off) - 1, C.byref(res), C.byref(bad))
        if rc == _lib.EKEY:
            raise KeyError(f"Invalid token for decoding: {bad.value}")
        _lib.check(rc)
        n_bytes = int(self._L.b200bpe_result_n_tokens(res))
        n_docs = int(self._L.b200bpe_result_n_docs(res))
        data = np.ctypeslib.as_array(C.cast(self._L.b200bpe_result_tokens(res), C.POINTER(C.c_uint8)),
                                     shape=(max(n_bytes, 1),))[:n_bytes].copy()
        off = np.ctypeslib.as_array(C.cast(self._L.b200bpe_result_offsets(res), C.POINTER(C.c_uint64)),
                                    shape=(n_docs + 1,)).copy()
        self._L.b200bpe_result_free(res)
        return data, off

    def decode_bytes_batch(self, batch) -> list[bytes]:
        lens = np.fromiter((len(t) for t in batch), dtype=np.uint64, count=len(batch))
        off = np.zeros(len(batch) + 1, np.uint64)
        np.cumsum(lens, out=off[1:])
        toks = np.zeros(int(off[-1]), np.uint32)
        for i, t in enumerate(batch):
            toks[int(off[i]):int(off[i + 1])] = np.asarray(t, dtype=np.uint32)
        data, boff = self.decode_batch_buffer(toks, off)
        raw = data.tobytes()
        return [raw[int(boff[i]):int(boff[i + 1])] for i in range(len(batch))]

    def decode_single_token_bytes(self, token: int) -> bytes:                # py.rs:164-172
        if self._decoder is None:
            self._decoder = {v: k for k, v in self._encoder.items()}
            self._decoder.update({v: k.encode("utf-8") for k, v in self._special.items()})
        try:
            return self._decoder[token]
        except KeyError:
            raise KeyError(str(token)) from None

    def token_byte_values(self) -> list[bytes]:                              # py.rs:178-183
        return sorted(self._encoder.keys())

    # ---- measurement hooks ----------------------------------------------------------------------
    def last_timings(self) -> dict:
        ms = (C.c_float * 9)()
        n = C.c_uint32(0)
        self._L.b200bpe_last_timings(self._h, ms, C.byref(n))
        keys = ["mark_docs_ms", "pretok_ms", "long_ms", "encode_ms", "device_total_ms", "h2d_ms", "d2h_ms", "gather_ms", "probe_ms"]
        d = {k: float(ms[i]) for i, k in enumerate(keys)}
        d["launches"] = int(n.value)
        return d

    def last_reruns(self) -> dict:
        """What the most recent encode call had to redo: `grown` names the work-spaces it grew and re-ran ("miss",
        "slow", "long"), `reruns` counts pipeline re-runs over all chunks and devices, `token_passes` is 2 when the
        host token buffer had to be re-sized.  Every encode call, `encode_device_async` included, starts from zeros."""
        grown, reruns, passes = C.c_uint32(0), C.c_uint32(0), C.c_uint32(0)
        _lib.check(self._L.b200bpe_last_reruns(self._h, C.byref(grown), C.byref(reruns), C.byref(passes)))
        names = {_lib.GREW_MISS: "miss", _lib.GREW_SLOW: "slow", _lib.GREW_LONG: "long"}
        return {"grown": {s for bit, s in names.items() if grown.value & bit}, "reruns": int(reruns.value),
                "token_passes": int(passes.value)}

    def last_piece_classes(self) -> dict:
        """Which long-piece merge kernels the most recent encode call ran: `counts[c]` = pieces of length class c
        (17..32, 33..64, 65..128, 129..256, 257..1024, 1025..4096, 4097..32768 and more bytes) of the runs whose output
        it returned, `lane_per_piece` = the lane-per-piece kernels of vocabularies with ranks of 2^22 and above merged
        them.  Zeros after a call that failed."""
        counts, lane = (C.c_uint64 * 8)(), C.c_int32(0)
        _lib.check(self._L.b200bpe_last_piece_classes(self._h, counts, C.byref(lane)))
        return {"counts": [int(x) for x in counts], "lane_per_piece": bool(lane.value)}

    def last_bytes_repairs(self) -> int:
        """Documents the most recent encode_bytes_batch* call found not to be well-formed UTF-8 and repaired (0 after any
        other call)."""
        n = C.c_uint64(0)
        _lib.check(self._L.b200bpe_last_bytes_repairs(self._h, C.byref(n)))
        return int(n.value)

    def last_unstable(self) -> dict:
        """What the most recent encode_with_unstable_batch* call did: documents with unstable bytes, candidates encoded,
        candidates that took byte_pair_encode, candidate rounds and completions returned (zeros after any other call)."""
        v = (C.c_uint64 * 5)()
        _lib.check(self._L.b200bpe_last_unstable(self._h, v))
        return dict(zip(["docs", "encoded", "bpe_candidates", "rounds", "completions"], (int(x) for x in v)))

    def last_miss_memo(self) -> dict:
        """What the per-call miss memo did in the most recent encode call: `misses` = pieces of up to 16 bytes that are
        not tokens (a single byte only when the vocabulary lacks it), `merged` = those merged (one per distinct piece, plus
        16-byte and unplaced ones; the others copy their owner's tokens), `unplaced` = pieces the memo did not place (no
        room, or it had stopped because it was full or did not pay).  Summed over chunks and devices; zeros after a call
        that failed."""
        v = [C.c_uint64(0) for _ in range(3)]
        _lib.check(self._L.b200bpe_last_miss_memo(self._h, *(C.byref(x) for x in v)))
        return {"misses": int(v[0].value), "merged": int(v[1].value), "unplaced": int(v[2].value)}

    def trim(self) -> None:
        """Give the engine's grow-only device work-spaces and pooled pinned blocks back (tables stay)."""
        _lib.check(self._L.b200bpe_trim(self._h))

    def table_bytes(self) -> dict:
        b = (C.c_uint64 * 4)()
        self._L.b200bpe_table_bytes(self._h, b)
        return {"piece_table": int(b[0]), "pair_table": int(b[1]), "long_token_table": int(b[2]), "unicode": int(b[3])}

    def encode_device_async(self, d_text_ptr: int, n_bytes: int, d_doc_off_ptr: int, n_docs: int, d_tokens_ptr: int,
                            d_tok_off_ptr: int, d_counts_ptr: int = 0, stream: int = 0) -> None:
        """Enqueue only (no host synchronisation); `d_counts_ptr`: optional device uint64[2] <- {n_tokens, n_docs}."""
        _lib.check(self._L.b200bpe_encode_device_async(self._h, C.c_void_p(d_text_ptr), n_bytes, C.c_void_p(d_doc_off_ptr),
                                                       n_docs, C.c_void_p(d_tokens_ptr), C.c_void_p(d_tok_off_ptr),
                                                       C.c_void_p(d_counts_ptr), C.c_void_p(stream)))

    def device_wait(self) -> int:
        n = C.c_uint64(0)
        _lib.check(self._L.b200bpe_device_wait(self._h, C.byref(n)))
        return int(n.value)

    def encode_device(self, d_text_ptr: int, n_bytes: int, d_doc_off_ptr: int, n_docs: int, d_tokens_ptr: int,
                      d_tok_off_ptr: int, stream: int = 0) -> int:
        """Device-resident path (pointers are raw CUDA device addresses); returns n_tokens."""
        n = C.c_uint64(0)
        rc = self._L.b200bpe_encode_device(self._h, C.c_void_p(d_text_ptr), n_bytes, C.c_void_p(d_doc_off_ptr),
                                           n_docs, C.c_void_p(d_tokens_ptr), C.c_void_p(d_tok_off_ptr), C.byref(n),
                                           C.c_void_p(stream))
        _lib.check(rc)
        return int(n.value)
