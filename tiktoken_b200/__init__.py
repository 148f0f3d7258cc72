"""tiktoken_b200 -- H100-native BPE encoder behind tiktoken's API (encode hot path only).

    from tiktoken_b200 import Encoding          # tiktoken.Encoding's constructor (+ device= / devices=)
    enc = Encoding("my_enc", pat_str=..., mergeable_ranks=..., special_tokens=...)
    enc.encode_ordinary_batch(docs)             # one native call -> sm_90a kernels

    tiktoken_b200.get_encoding("cl100k_base")   # the reference's registry + plugins, GPU-backed Encoding
    tiktoken_b200.install()                     # or: run the UNMODIFIED `tiktoken` package on the GPU engine

    tiktoken_b200.bpe_train(text, 50_000, pat)  # tiktoken._educational.bpe_train on the GPU (train.py)

`tiktoken_b200._tiktoken.CoreBPE` is the drop-in for the Rust extension (see INTEGRATION.md).  Everything the
north star says stays -- tiktoken/core.py's host class, tiktoken/registry.py, tiktoken/load.py, the tiktoken_ext
plugins -- is the reference's own code, imported, not re-typed.
"""
from __future__ import annotations

import threading

from .core import Encoding  # noqa: F401
from .train import bpe_train, bpe_train_batch, bpe_train_packed, last_train_stats  # noqa: F401

__version__ = "0.2.0"

_REGISTRY: dict[str, Encoding] = {}
_lock = threading.RLock()


def _constructors():
    import tiktoken.registry as ref           # the reference's plugin discovery (tiktoken/registry.py:28-60), untouched
    if ref.ENCODING_CONSTRUCTORS is None:
        with ref._lock:
            if ref.ENCODING_CONSTRUCTORS is None:
                ref._find_constructors()
    return ref.ENCODING_CONSTRUCTORS


def get_encoding(encoding_name: str, **device_kw) -> Encoding:
    """`tiktoken.get_encoding` with the GPU-backed class: same names, same plugin constructors
    (tiktoken_ext.openai_public, ...), one cached instance per name."""
    if not isinstance(encoding_name, str):
        raise ValueError(f"Expected a string in get_encoding, got {type(encoding_name)}")
    with _lock:
        if encoding_name in _REGISTRY:
            return _REGISTRY[encoding_name]
        ctors = _constructors()
        if encoding_name not in ctors:
            raise ValueError(f"Unknown encoding {encoding_name}.\nPlugins found: {sorted(ctors)}")
        enc = Encoding(**ctors[encoding_name](), **device_kw)
        _REGISTRY[encoding_name] = enc
        return enc


def list_encoding_names() -> list[str]:
    return list(_constructors())


def install() -> None:
    """Make the unmodified `tiktoken` package use the GPU engine from now on: `tiktoken.core._tiktoken` (the one
    name through which tiktoken/core.py reaches its native module, core.py:7,54) becomes `tiktoken_b200._tiktoken`.
    Every `tiktoken.Encoding` constructed afterwards -- `tiktoken.get_encoding(...)` included -- runs on the GPU.
    This is what shipping `tiktoken/_tiktoken.py` = this shim in place of the Rust extension does (INTEGRATION.md)."""
    import tiktoken.core
    from . import _tiktoken
    tiktoken.core._tiktoken = _tiktoken
