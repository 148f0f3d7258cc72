import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
for p in (ROOT, os.path.join(ROOT, "tests")):
    if p not in sys.path:
        sys.path.insert(0, p)


def pytest_configure(config):
    config.addinivalue_line("markers", "gpu: needs a CUDA device (run on an H100 with -m gpu)")


def _build_hostcheck() -> str:
    csrc = os.path.join(ROOT, "tiktoken_b200", "csrc")
    so = os.path.join(csrc, "libb200bpe_hostcheck.so")
    srcs = [os.path.join(csrc, f) for f in ("hostcheck.cpp", "pretok_rules.cuh", "pretok_fast.cuh", "text_access.cuh", "bpe_device.cuh",
                                            "bpe_tables.h", "unicode_classes.inc")]
    if not os.path.exists(so) or any(os.path.getmtime(s) > os.path.getmtime(so) for s in srcs):
        subprocess.check_call(["g++", "-O2", "-fPIC", "-shared", "-std=c++17", "-o", so, srcs[0]])
    return so


@pytest.fixture(scope="session")
def hostcheck():
    import ctypes as C
    H = C.CDLL(_build_hostcheck())
    H.hc_piece_starts.argtypes = [C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p]
    H.hc_piece_starts_fast.argtypes = [C.c_int, C.c_void_p, C.c_int64, C.c_void_p, C.c_int64, C.c_void_p, C.c_void_p]
    H.hc_tables_new.restype = C.c_void_p
    H.hc_tables_new.argtypes = [C.c_void_p, C.c_void_p, C.c_void_p, C.c_uint32, C.c_void_p]
    H.hc_tables_free.argtypes = [C.c_void_p]
    H.hc_encode_short.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32, C.c_void_p]
    H.hc_encode_mid.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32, C.c_uint32, C.c_void_p]
    H.hc_pair_lookup.restype = C.c_uint32
    H.hc_pair_lookup.argtypes = [C.c_void_p, C.c_uint32, C.c_uint32]
    H.hc_pair_buckets.restype = C.c_uint64
    H.hc_pair_buckets.argtypes = [C.c_void_p]
    H.hc_tables_pairs.restype = C.c_uint64
    H.hc_tables_pairs.argtypes = [C.c_void_p]
    H.hc_probe_long.restype = C.c_uint32
    H.hc_probe_long.argtypes = [C.c_void_p, C.c_char_p, C.c_uint32]
    return H


_HAVE_GPU = None


def have_gpu() -> bool:
    """CUDA device present?  Asked of the engine's own library (cudaGetDeviceCount), not of torch: the
    engine does not need torch."""
    global _HAVE_GPU
    if _HAVE_GPU is None:
        try:
            from tiktoken_b200 import _lib
            _lib.build()
            _HAVE_GPU = int(_lib.lib().b200bpe_device_count()) > 0
        except Exception:
            _HAVE_GPU = False
    return _HAVE_GPU


def pytest_collection_modifyitems(config, items):
    """`-m gpu` tests are skipped (not failed) on a machine without a CUDA device."""
    if have_gpu():
        return
    skip = pytest.mark.skip(reason="needs a CUDA device (the engine has no CPU fallback)")
    for item in items:
        if "gpu" in item.keywords:
            item.add_marker(skip)
