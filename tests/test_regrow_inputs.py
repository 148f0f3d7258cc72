"""The inputs of test_gpu_regrow.py reach the paths they are meant to reach.

Every recipe of regrow_inputs.py is recounted on the CPU (pieces from the oracle's split, undecided pre-tokeniser
positions from the span evaluator the pre-tokeniser kernel runs, tokens from the oracle) and compared with the
engine's first-run capacities: it must exceed the one it is built for by at least 1.25x and stay under all the others.
If the sizing in b200bpe.cu changes, this fails before a GPU test passes for the wrong reason."""
import numpy as np
import pytest

import regrow_inputs as ri
from oracle import Oracle

_ORACLES = {}


def _oracle(kind):
    if kind not in _ORACLES:
        pat, ranks, special = ri.vocabulary(kind)
        _ORACLES[kind] = (Oracle(ranks, special, pat), ranks)
    return _ORACLES[kind]


def _check(need, cap, exceeds, what):
    for k in cap:
        if k in exceeds:
            assert need[k] >= 1.25 * cap[k], f"{what}: {k} {need[k]} does not exceed {cap[k]} by 1.25x"
        else:
            assert need[k] < cap[k], f"{what}: {k} {need[k]} is not under {cap[k]}"


@pytest.mark.parametrize("name", sorted(ri.RECIPES))
def test_recipe_exceeds_exactly_its_capacity(name, hostcheck):
    gen, vocab, exceeds = ri.RECIPES[name]
    text, off = gen()
    again, off2 = gen()
    assert np.array_equal(text, again) and np.array_equal(off, off2)          # deterministic in the seed
    assert len(text) <= 32 << 20 and len(off) > 2
    o, ranks = _oracle(vocab)
    need = ri.measure(o, ranks, hostcheck, text, off)
    _check(need, ri.caps(len(text)), exceeds, name)


def test_batch_overflows_every_chunk_and_the_token_buffer(hostcheck):
    """With 1 MiB chunks every document of the batch is one chunk, and each overflows the work-space of its recipe."""
    text, off, kinds = ri.batch()
    assert len(text) <= 32 << 20 and set(kinds) == {"miss", "slow", "long", "tokens"}
    o, ranks = _oracle(ri.BATCH_VOCAB)
    for d, kind in enumerate(kinds):
        lo, hi = int(off[d]), int(off[d + 1])
        if kind == "long":
            assert hi - lo > 1 << 20
        else:
            assert hi - lo <= 1 << 20 and (d + 1 == len(kinds) or int(off[d + 2]) - lo > 1 << 20)   # alone in its chunk
        doc = np.ascontiguousarray(text[lo:hi])
        need = ri.measure(o, ranks, hostcheck, doc, np.asarray([0, hi - lo], np.uint64))
        cap = ri.caps(hi - lo)
        del need["tokens"], cap["tokens"]                     # the token buffer is sized per call, not per chunk
        exceeds = set() if kind == "tokens" else ri.RECIPES[kind][2]
        _check(need, cap, exceeds, f"document {d} ({kind})")
    total = len(o.encode_ordinary_batch_np(text, off, 8)[0])
    assert total >= 1.1 * ri.caps(len(text))["tokens"]
