"""ctypes binding of libb200bpe.so (C ABI in include/b200bpe.h).

This is the binding a tiktoken maintainer would add in place of the PyO3 module
(src/py.rs): plain pointers and sizes, the GIL is released for the duration of every call
(ctypes.CDLL does that), errors come back as status codes + a thread-local message.
The library is built in-tree by `build()` (nvcc, sm_90a only).  There is no fallback: if the
shared object or a CUDA device is missing the import / constructor raises.
"""
from __future__ import annotations

import ctypes as C
import os
import subprocess

_CSRC = os.path.join(os.path.dirname(os.path.abspath(__file__)), "csrc")
_SO = os.path.join(_CSRC, "libb200bpe.so")
_SOURCES = ["b200bpe.cu", "dev_common.cuh", "kernels_pretok.cuh", "kernels_long.cuh", "kernels_mid.cuh", "kernels_pmerge.cuh", "kernels_encode.cuh",
            "kernels_special.cuh", "kernels_decode.cuh", "kernels_bytes.cuh", "kernels_unstable.cuh", "kernels_train.cuh", "utf8_check.cuh", "bpe_device.cuh", "bpe_tables.h", "pretok_rules.cuh",
            "pretok_fast.cuh", "text_access.cuh", "unicode_classes.inc", "doc_seams.h"]

OK, EINVAL, EPATTERN, EDUPRANK, ECUDA, ENOBYTE, EKEY, ESPECIAL, ECAPACITY, ENOPAIR = 0, -1, -2, -3, -4, -5, -6, -7, -8, -9

NVCC_FLAGS = ["-gencode", "arch=compute_90a,code=sm_90a", "-O3", "-lineinfo", "-std=c++17",
              "-shared", "-Xcompiler", "-fPIC"]


def build(force: bool = False) -> str:
    """Compile libb200bpe.so for sm_90a with nvcc (cross-compiles without a GPU)."""
    srcs = [os.path.join(_CSRC, s) for s in _SOURCES] + [
        os.path.join(os.path.dirname(_CSRC), "..", "include", "b200bpe.h")]
    stale = force or not os.path.exists(_SO) or any(
        os.path.getmtime(s) > os.path.getmtime(_SO) for s in srcs if os.path.exists(s))
    if stale:
        nvcc = os.environ.get("NVCC", "/usr/local/cuda/bin/nvcc")
        if not os.path.exists(nvcc):
            nvcc = "nvcc"
        subprocess.check_call([nvcc] + NVCC_FLAGS + ["-o", _SO, os.path.join(_CSRC, "b200bpe.cu")])
    return _SO


_lib = None


def lib() -> C.CDLL:
    global _lib
    if _lib is not None:
        return _lib
    so = os.environ.get("B200BPE_LIB") or _SO        # development: A/B builds of the same sources (tools/ab.sh)
    if not os.path.exists(so):
        raise RuntimeError(
            f"{so} is missing: build it with `python -c 'import __graft_entry__ as g; g.build()'` "
            "(tiktoken_b200 has no CPU fallback)")
    L = C.CDLL(so)
    vp, u64, u32, i32 = C.c_void_p, C.c_uint64, C.c_uint32, C.c_int
    L.b200bpe_create.restype = i32
    L.b200bpe_create.argtypes = [vp, vp, vp, u32, vp, vp, vp, u32, C.c_char_p, i32, C.POINTER(vp)]
    L.b200bpe_create_multi.restype = i32
    L.b200bpe_create_multi.argtypes = [vp, vp, vp, u32, vp, vp, vp, u32, C.c_char_p, vp, i32, C.POINTER(vp)]
    L.b200bpe_trim.restype = i32
    L.b200bpe_trim.argtypes = [vp]
    L.b200bpe_n_devices.restype = i32
    L.b200bpe_n_devices.argtypes = [vp]
    L.b200bpe_encode_batch_special.restype = i32
    L.b200bpe_encode_batch_special.argtypes = [vp, vp, vp, u64, vp, C.POINTER(vp), C.POINTER(C.c_int32)]
    L.b200bpe_special_name.restype = C.c_char_p
    L.b200bpe_special_name.argtypes = [vp, C.c_int32]
    L.b200bpe_encode_device_async.restype = i32
    L.b200bpe_encode_device_async.argtypes = [vp, vp, u64, vp, u64, vp, vp, vp, vp]
    L.b200bpe_device_wait.restype = i32
    L.b200bpe_device_wait.argtypes = [vp, C.POINTER(u64)]
    L.b200bpe_count_batch.restype = i32
    L.b200bpe_count_batch.argtypes = [vp, vp, vp, u64, vp, vp, C.POINTER(C.c_int32)]
    L.b200bpe_encode_device_special_async.restype = i32
    L.b200bpe_encode_device_special_async.argtypes = [vp, vp, u64, vp, u64, vp, vp, vp, vp, vp]
    L.b200bpe_device_wait_special.restype = i32
    L.b200bpe_device_wait_special.argtypes = [vp, C.POINTER(u64), C.POINTER(C.c_int32)]
    L.b200bpe_destroy.restype = None
    L.b200bpe_destroy.argtypes = [vp]
    L.b200bpe_encode_ordinary_batch.restype = i32
    L.b200bpe_encode_ordinary_batch.argtypes = [vp, vp, vp, u64, C.POINTER(vp)]
    L.b200bpe_encode_batch.restype = i32
    L.b200bpe_encode_batch.argtypes = [vp, vp, vp, u64, vp, C.POINTER(vp)]
    L.b200bpe_encode_device.restype = i32
    L.b200bpe_encode_device.argtypes = [vp, vp, u64, vp, u64, vp, vp, C.POINTER(u64), vp]
    L.b200bpe_encode_bytes_batch.restype = i32
    L.b200bpe_encode_bytes_batch.argtypes = [vp, vp, vp, u64, C.POINTER(vp)]
    L.b200bpe_last_bytes_repairs.restype = i32
    L.b200bpe_last_bytes_repairs.argtypes = [vp, C.POINTER(u64)]
    L.b200bpe_encode_with_unstable_batch.restype = i32
    L.b200bpe_encode_with_unstable_batch.argtypes = [vp, vp, vp, u64, vp, C.POINTER(vp), C.POINTER(vp), C.POINTER(C.c_int32)]
    L.b200bpe_result_groups.restype = vp
    L.b200bpe_result_groups.argtypes = [vp, C.POINTER(u64)]
    L.b200bpe_last_unstable.restype = i32
    L.b200bpe_last_unstable.argtypes = [vp, vp]
    L.b200bpe_last_miss_memo.restype = i32
    L.b200bpe_last_miss_memo.argtypes = [vp, C.POINTER(u64), C.POINTER(u64), C.POINTER(u64)]
    L.b200bpe_last_doc_seams.restype = i32
    L.b200bpe_last_doc_seams.argtypes = [vp, C.POINTER(u64), C.POINTER(u64)]
    L.b200bpe_encode_single_piece.restype = i32
    L.b200bpe_encode_single_piece.argtypes = [vp, vp, u64, C.POINTER(vp)]
    L.b200bpe_result_tokens.restype = vp
    L.b200bpe_result_tokens.argtypes = [vp]
    L.b200bpe_result_offsets.restype = vp
    L.b200bpe_result_offsets.argtypes = [vp]
    L.b200bpe_result_n_tokens.restype = u64
    L.b200bpe_result_n_tokens.argtypes = [vp]
    L.b200bpe_result_n_docs.restype = u64
    L.b200bpe_result_n_docs.argtypes = [vp]
    L.b200bpe_result_free.restype = None
    L.b200bpe_result_free.argtypes = [vp]
    L.b200bpe_decode_bytes.restype = i32
    L.b200bpe_decode_bytes.argtypes = [vp, vp, u64, vp, u64, C.POINTER(u64), C.POINTER(u32)]
    L.b200bpe_decode_batch.restype = i32
    L.b200bpe_decode_batch.argtypes = [vp, vp, vp, u64, C.POINTER(vp), C.POINTER(u32)]
    L.b200bpe_last_timings.restype = i32
    L.b200bpe_last_timings.argtypes = [vp, vp, C.POINTER(u32)]
    L.b200bpe_last_reruns.restype = i32
    L.b200bpe_last_reruns.argtypes = [vp, C.POINTER(u32), C.POINTER(u32), C.POINTER(u32)]
    L.b200bpe_last_piece_classes.restype = i32
    L.b200bpe_last_piece_classes.argtypes = [vp, vp, C.POINTER(i32)]
    L.b200bpe_table_bytes.restype = i32
    L.b200bpe_table_bytes.argtypes = [vp, vp]
    L.b200bpe_device_count.restype = i32
    L.b200bpe_device_count.argtypes = []
    L.b200bpe_bpe_train.restype = i32
    L.b200bpe_bpe_train.argtypes = [vp, vp, u64, C.c_char_p, u32, i32, vp, u64, C.POINTER(u64), vp]
    L.b200bpe_last_error.restype = C.c_char_p
    L.b200bpe_version.restype = C.c_char_p
    _lib = L
    return L


EXPORTS = [
    "b200bpe_create", "b200bpe_destroy", "b200bpe_encode_ordinary_batch", "b200bpe_encode_batch",
    "b200bpe_encode_device", "b200bpe_encode_single_piece", "b200bpe_result_tokens",
    "b200bpe_result_offsets", "b200bpe_result_n_tokens", "b200bpe_result_n_docs", "b200bpe_result_free",
    "b200bpe_decode_bytes", "b200bpe_decode_batch", "b200bpe_last_timings", "b200bpe_table_bytes", "b200bpe_last_error",
    "b200bpe_version", "b200bpe_device_count", "b200bpe_create_multi", "b200bpe_n_devices", "b200bpe_encode_batch_special",
    "b200bpe_special_name", "b200bpe_encode_device_async", "b200bpe_device_wait", "b200bpe_trim", "b200bpe_last_reruns",
    "b200bpe_last_piece_classes", "b200bpe_encode_bytes_batch", "b200bpe_last_bytes_repairs", "b200bpe_last_miss_memo",
    "b200bpe_encode_with_unstable_batch", "b200bpe_result_groups", "b200bpe_last_unstable", "b200bpe_bpe_train",
    "b200bpe_count_batch", "b200bpe_encode_device_special_async", "b200bpe_device_wait_special",
    "b200bpe_last_doc_seams",
]

GREW_MISS, GREW_SLOW, GREW_LONG = 1, 2, 4       # B200BPE_GREW_* (b200bpe_last_reruns)


def last_error() -> str:
    return (lib().b200bpe_last_error() or b"").decode("utf-8", "replace")


def check(rc: int) -> None:
    """Map C status codes onto the exception types the reference raises (SURVEY.md 8(b))."""
    if rc == OK:
        return
    msg = last_error()
    if rc in (EINVAL, EPATTERN, EDUPRANK, ESPECIAL, ENOPAIR):
        raise ValueError(msg)
    if rc == EKEY:
        raise KeyError(msg)
    if rc == ENOBYTE:
        raise KeyError(msg)
    raise RuntimeError(msg)
