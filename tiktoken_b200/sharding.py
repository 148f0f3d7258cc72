"""Document sharding across the GPUs of one box (SURVEY.md 8(e)).

Documents are independent haystacks, so the encode path shards embarrassingly: rank r encodes a
contiguous range of documents chosen to balance BYTES, with its own replica of the rank tables.
The only exchange is one all-gather of (n_tokens, n_docs) per rank (NCCL over NVLink when the
process group is NCCL), from which every rank derives the global token offset of its shard; no
token payload crosses NVLink.
"""
from __future__ import annotations

import numpy as np


def shard_ranges(doc_off: np.ndarray, world: int) -> list[tuple[int, int]]:
    """Contiguous document ranges [lo, hi) per rank with ~equal bytes.  A single huge document
    cannot be split (one haystack), so ranks may receive empty ranges."""
    doc_off = np.asarray(doc_off, dtype=np.uint64)
    n_docs = len(doc_off) - 1
    total = int(doc_off[-1])
    cuts = [0]
    for r in range(1, world):
        target = total * r // world
        # first document whose START is >= target keeps prefix sums balanced
        d = int(np.searchsorted(doc_off[:-1], target, side="left"))
        cuts.append(min(max(d, cuts[-1]), n_docs))
    cuts.append(n_docs)
    return [(cuts[r], cuts[r + 1]) for r in range(world)]


def local_view(text: np.ndarray, doc_off: np.ndarray, lo: int, hi: int):
    """Slice the packed batch to documents [lo, hi) and rebase the offsets."""
    doc_off = np.asarray(doc_off, dtype=np.uint64)
    b0, b1 = int(doc_off[lo]), int(doc_off[hi])
    return text[b0:b1], (doc_off[lo:hi + 1] - doc_off[lo]).astype(np.uint64)


def gather_counts(n_tokens: int, n_docs: int, rank: int, world: int, device=None):
    """All-gather (n_tokens, n_docs) of every rank -> (counts[world,2], token_base, doc_base)."""
    import torch
    import torch.distributed as dist
    if world == 1 or not dist.is_initialized():
        counts = np.asarray([[n_tokens, n_docs]], dtype=np.int64)
        return counts, 0, 0
    mine = torch.tensor([n_tokens, n_docs], dtype=torch.int64, device=device or "cpu")
    allc = [torch.zeros_like(mine) for _ in range(world)]
    dist.all_gather(allc, mine)
    counts = torch.stack(allc).cpu().numpy()
    return counts, int(counts[:rank, 0].sum()), int(counts[:rank, 1].sum())


def encode_sharded(encode_packed, text: np.ndarray, doc_off: np.ndarray, rank: int, world: int, device=None):
    """Encode this rank's shard with `encode_packed(text, doc_off) -> (tokens, tok_off)` and locate it
    in the global output.  Returns a dict with the local arrays and the global placement."""
    lo, hi = shard_ranges(doc_off, world)[rank]
    ltext, loff = local_view(text, doc_off, lo, hi)
    tokens, tok_off = encode_packed(ltext, loff)
    counts, token_base, doc_base = gather_counts(int(len(tokens)), hi - lo, rank, world, device)
    return {"doc_range": (lo, hi), "tokens": tokens, "tok_off": tok_off, "token_base": token_base,
            "doc_base": doc_base, "counts": counts, "total_tokens": int(counts[:, 0].sum())}


class CountExchange:
    """The same all-gather as `gather_counts`, posted asynchronously so that a stream of batches does not stop
    for it: `post()` after batch k, `wait()` (any time later) returns (counts[world,2], token_base, doc_base) of
    that batch.  All buffers are allocated ONCE (a ring of `depth` send / receive pairs): a post costs one
    `all_gather_into_tensor` and nothing else.  The send buffer of slot k can be handed to the engine as the
    `d_counts` of `b200bpe_encode_device_async` (`send_ptr(k)`): the pipeline's last kernel writes {n_tokens, n_docs}
    there and `post_device()` enqueues the all-gather behind it on the same stream -- the host never sees the
    counts.  With an NCCL group the exchange runs next to the kernels of the following batch."""

    def __init__(self, rank: int, world: int, device=None, depth: int = 8):
        self.rank, self.world, self.depth = rank, world, depth
        self._pending = []
        self._k = 0
        import torch
        import torch.distributed as dist
        self.active = world > 1 and dist.is_initialized()
        self._dev = device or "cpu"
        self._send = torch.zeros((depth, 2), dtype=torch.int64, device=self._dev)
        self._recv = torch.zeros((depth, max(world, 1), 2), dtype=torch.int64, device=self._dev)
        pin = self._dev != "cpu" and torch.cuda.is_available()
        self._host = torch.zeros((depth, 2), dtype=torch.int64, pin_memory=pin)

    def _slot(self) -> int:
        if len(self._pending) >= self.depth:
            raise RuntimeError("CountExchange ring is full: wait() before posting more")
        k = self._k
        self._k = (k + 1) % self.depth
        return k

    def send_ptr(self, k: int | None = None) -> int:
        """Device address of the next (or given) slot's send buffer, for `encode_device_async(d_counts_ptr=...)`."""
        return int(self._send[self._k if k is None else k].data_ptr())

    def post(self, n_tokens: int, n_docs: int) -> None:
        """Counts known on the host."""
        k = self._slot()
        if not self.active:
            self._pending.append((None, k, (int(n_tokens), int(n_docs))))
            return
        self._host[k, 0] = int(n_tokens); self._host[k, 1] = int(n_docs)
        self._send[k].copy_(self._host[k], non_blocking=True)
        self._post(k)

    def post_device(self) -> None:
        """Counts already written into `send_ptr()` by work enqueued on the current stream."""
        k = self._slot()
        if not self.active:
            self._pending.append((None, k, None))
            return
        self._post(k)

    def _post(self, k: int) -> None:
        import torch.distributed as dist
        work = dist.all_gather_into_tensor(self._recv[k].view(-1), self._send[k], async_op=True)
        self._pending.append((work, k, None))

    def wait(self):
        work, k, local = self._pending.pop(0)
        if work is None:
            if local is None:
                local = tuple(int(x) for x in self._send[k].cpu().tolist())
            return np.asarray([local], dtype=np.int64), 0, 0
        work.wait()
        counts = self._recv[k].cpu().numpy().copy()
        return counts, int(counts[:self.rank, 0].sum()), int(counts[:self.rank, 1].sum())

    def drain(self):
        out = []
        while self._pending:
            out.append(self.wait())
        return out


def gpu_numa_cpus(device_index: int) -> list[int] | None:
    """CPUs of the NUMA node the GPU hangs off (sysfs), or None when the platform does not say."""
    try:
        import torch
        p = torch.cuda.get_device_properties(device_index)
        bdf = f"{p.pci_domain_id:04x}:{p.pci_bus_id:02x}:{p.pci_device_id:02x}.0"
        node = int(open(f"/sys/bus/pci/devices/{bdf}/numa_node").read().strip())
        if node < 0:
            return None
        cpus: list[int] = []
        for part in open(f"/sys/devices/system/node/node{node}/cpulist").read().strip().split(","):
            a, _, b = part.partition("-")
            cpus.extend(range(int(a), int(b or a) + 1))
        return cpus or None
    except Exception:
        return None


def bind_to_gpu_numa(device_index: int) -> dict:
    """Pin this process to the CPUs next to its GPU BEFORE it allocates pinned host buffers: first touch then puts
    them on that node, and H2D / D2H do not cross the inter-socket link (ranks whose buffers sit on one node share that
    node's memory and link bandwidth).  Returns what was done, for the bench line."""
    import os
    cpus = gpu_numa_cpus(device_index)
    if not cpus:
        return {"bound": False, "why": "no NUMA information for the device"}
    try:
        allowed = sorted(set(cpus) & set(os.sched_getaffinity(0)))
        if not allowed:
            return {"bound": False, "why": "node CPUs not in the allowed set"}
        os.sched_setaffinity(0, allowed)
        return {"bound": True, "cpus": f"{allowed[0]}-{allowed[-1]} ({len(allowed)})"}
    except Exception as e:                                     # noqa: BLE001
        return {"bound": False, "why": str(e)}
