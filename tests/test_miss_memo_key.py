"""The miss memo's key (memo_key in bpe_device.cuh, host build through hostcheck.cpp): equal keys mean equal pieces.

Every string of 1..15 bytes over {NUL, 'a', 0xFF} up to length 10, plus random ones of every length, gets a key of its
own; no key is all zero (an empty memo slot); a 16-byte piece is not memoised."""
import ctypes as C
import itertools
import random


def _key(H, piece: bytes):
    out = (C.c_uint32 * 4)()
    rc = H.hc_memo_key(piece, len(piece), out)
    return rc, tuple(out)


def test_memo_key_is_injective_and_never_empty(hostcheck):
    H = hostcheck
    H.hc_memo_key.restype = C.c_int
    H.hc_memo_key.argtypes = [C.c_char_p, C.c_uint32, C.c_void_p]
    pieces = [bytes(t) for n in range(1, 11) for t in itertools.product((0, 0x61, 0xFF), repeat=n)]
    rnd = random.Random(3)
    pieces += [bytes(rnd.choice((0, 0, 1, 0x61, 0xFF)) for _ in range(n)) for n in range(1, 16) for _ in range(2000)]
    pieces = set(pieces)
    seen = {}
    for pc in pieces:
        rc, k = _key(H, pc)
        assert rc == 1 and any(k), pc
        assert k[3] >> 24 == len(pc)
        assert seen.setdefault(k, pc) == pc, (pc, seen[k])
    assert len(seen) == len(pieces)
    assert _key(H, b"\0" * 16)[0] == 0 and _key(H, bytes(range(16)))[0] == 0
