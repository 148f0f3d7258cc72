"""CPU-only check of the two piece tables (bpe_tables.h): tokens of 1..11 bytes in the narrow table (16-byte slots),
12..16 bytes in the wide table (32-byte slots), probed through the same issue / finish pair the probe kernel runs."""
import ctypes as C
import random

import vocab_util as vu
from test_host_tables import make_tables

MAXR = 0xFFFFFFFF


def _bind(H):
    H.hc_piece_lookup.restype = C.c_uint32
    H.hc_piece_lookup.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32]
    H.hc_piece_slots.restype = None
    H.hc_piece_slots.argtypes = [C.c_void_p, C.POINTER(C.c_uint64), C.POINTER(C.c_uint64)]


def test_every_short_token_is_found_in_its_table(hostcheck):
    _bind(hostcheck)
    for name in ("cl100k_base", "o200k_base", "r50k_base"):
        _, ranks, _, _ = vu.load_encoding(name, allow_real=False)
        h, rc = make_tables(hostcheck, ranks)
        assert rc == 0
        short = {t: r for t, r in ranks.items() if len(t) <= 16}
        n_narrow = sum(1 for t in short if len(t) <= 11)
        n_wide = len(short) - n_narrow
        assert n_narrow and n_wide
        for t, r in short.items():
            assert hostcheck.hc_piece_lookup(h, t, len(t)) == r, (name, t)
        narrow, wide = C.c_uint64(0), C.c_uint64(0)
        hostcheck.hc_piece_slots(h, C.byref(narrow), C.byref(wide))
        assert narrow.value >= 3 * n_narrow and wide.value >= 3 * n_wide          # load <= 1/3 in both tables
        # absent pieces of every length miss, including ones that differ from a token only in the length byte's place
        rnd = random.Random(7)
        toks = list(short)
        tried = 0
        while tried < 20000:
            t = rnd.choice(toks)
            k = rnd.randint(1, 16)
            p = (t + bytes(rnd.randrange(256) for _ in range(16)))[:k]
            if rnd.random() < 0.3 and len(t) < 16:
                p = t + b"\0"                                                   # zero byte appended: same key words
            if p in ranks:
                continue
            tried += 1
            assert hostcheck.hc_piece_lookup(h, p, len(p)) == MAXR, (name, p)
        hostcheck.hc_tables_free(h)
