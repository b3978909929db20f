"""An in-process stand-in for the part of ``torch.distributed`` that ``pinot_b200.distributed`` uses, so the cross-GPU
combine runs end to end on ONE GPU (or on none): every simulated rank is a thread with its own facade over one shared
rendezvous.

Semantics follow torch's:

* ``reduce`` writes only ``dst``'s tensor, ``all_reduce`` every rank's; the ranks' tensors are combined in rank order
  (rank 0 first), so float sums are deterministic;
* ``all_gather_object`` / ``broadcast_object_list`` move objects through a pickle round trip;
* CUDA tensors (the views ``device_buffers`` puts over the library's tables) are read and written with torch ops, and the
  device is synchronised before a collective reads them and before it returns, so the library's own streams see the
  result.

Every collective waits at most ``timeout`` seconds.  A rank that raises aborts the rendezvous: its peers fail at their next
(or current) collective instead of hanging.  Each facade counts the collectives its rank issued (``calls``).
"""
from __future__ import annotations

import pickle
import threading
import time
from dataclasses import dataclass, field
from typing import Callable, List, Optional

TIMEOUT_S = 120.0      # longest wait inside one collective
DEADLINE_S = 900.0     # longest run of all ranks


class ReduceOp:
    SUM = "sum"
    MAX = "max"
    MIN = "min"


class LoopbackAborted(RuntimeError):
    """A peer failed, or a collective waited longer than the timeout."""


class Rendezvous:
    """The meeting point of `world` ranks: one slot per rank and a barrier, used twice per collective."""

    def __init__(self, world: int, timeout: float = TIMEOUT_S):
        self.world, self.timeout = world, timeout
        self.slots: List[object] = [None] * world
        self.barrier = threading.Barrier(world, timeout=timeout)

    def wait(self, what: str) -> None:
        try:
            self.barrier.wait()
        except threading.BrokenBarrierError:
            raise LoopbackAborted(f"{what}: a peer failed or the collective timed out") from None

    def abort(self) -> None:
        self.barrier.abort()


def _sync(t) -> None:
    if t.is_cuda:
        import torch
        torch.cuda.synchronize(t.device)


def _combine(parts, op):
    import torch
    acc = parts[0].clone()
    for p in parts[1:]:
        if op == ReduceOp.SUM:
            acc += p
        elif op == ReduceOp.MAX:
            acc = torch.maximum(acc, p)
        elif op == ReduceOp.MIN:
            acc = torch.minimum(acc, p)
        else:
            raise ValueError(op)
    return acc


class LoopbackDist:
    """One rank's facade: get_rank, get_world_size, ReduceOp, reduce, all_reduce, all_gather_object,
    broadcast_object_list."""

    ReduceOp = ReduceOp

    def __init__(self, rdv: Rendezvous, rank: int):
        self.rdv, self.rank = rdv, rank
        self.calls: List[str] = []   # the collectives this rank issued, in order

    def get_rank(self) -> int:
        return self.rank

    def get_world_size(self) -> int:
        return self.rdv.world

    def _exchange(self, what: str, payload) -> list:
        """Posts `payload`, returns every rank's (rank order) once all have posted.  The caller must call
        self.rdv.wait() again after it has finished reading the peers' payloads."""
        self.calls.append(what)
        self.rdv.slots[self.rank] = payload
        self.rdv.wait(what)
        return list(self.rdv.slots)

    def _reduce(self, what: str, tensor, op, write: bool) -> None:
        _sync(tensor)
        parts = self._exchange(what, tensor)
        out = _combine(parts, op)
        _sync(out)
        self.rdv.wait(what)            # every rank has read every tensor: now they may be overwritten
        if write:
            tensor.copy_(out)
            _sync(tensor)
        self.rdv.wait(what)            # slots are free for the next collective

    def reduce(self, tensor, dst: int = 0, op=ReduceOp.SUM) -> None:
        self._reduce("reduce", tensor, op, self.rank == dst)

    def all_reduce(self, tensor, op=ReduceOp.SUM) -> None:
        self._reduce("all_reduce", tensor, op, True)

    def all_gather_object(self, object_list: list, obj) -> None:
        parts = self._exchange("all_gather_object", pickle.dumps(obj))
        self.rdv.wait("all_gather_object")
        for i, p in enumerate(parts):
            object_list[i] = pickle.loads(p)

    def broadcast_object_list(self, object_list: list, src: int = 0) -> None:
        parts = self._exchange("broadcast_object_list", pickle.dumps(list(object_list)) if self.rank == src else None)
        self.rdv.wait("broadcast_object_list")
        object_list[:] = pickle.loads(parts[src])


@dataclass
class RankOutcome:
    value: object = None
    error: Optional[BaseException] = None
    calls: List[str] = field(default_factory=list)


def run_ranks(world: int, fn: Callable[[LoopbackDist], object], timeout: float = TIMEOUT_S,
              deadline: float = DEADLINE_S) -> List[RankOutcome]:
    """Runs fn(dist) on `world` threads, one per rank, and returns each rank's outcome (value or the exception it raised,
    and the collectives it issued).  A rank that raises aborts the rendezvous so that no peer waits for it.  Threads are
    joined within `deadline` seconds; a thread still alive then is reported as a failure of the whole run (the rendezvous
    is aborted, so it leaves at its next collective)."""
    rdv = Rendezvous(world, timeout)
    dists = [LoopbackDist(rdv, r) for r in range(world)]
    out = [RankOutcome() for _ in range(world)]

    def body(r: int) -> None:
        try:
            out[r].value = fn(dists[r])
        except BaseException as e:   # noqa: BLE001 -- reported to the caller
            out[r].error = e
            rdv.abort()

    threads = [threading.Thread(target=body, args=(r,), name=f"loopback-rank{r}", daemon=True) for r in range(world)]
    for t in threads:
        t.start()
    end = time.monotonic() + deadline
    for t in threads:
        t.join(max(0.0, end - time.monotonic()))
    alive = [t.name for t in threads if t.is_alive()]
    if alive:
        rdv.abort()
        for t in threads:
            t.join(timeout)
        raise RuntimeError(f"loopback ranks did not finish: {alive}")
    for r in range(world):
        out[r].calls = dists[r].calls
    return out


def values(outcomes: List[RankOutcome]) -> list:
    """The ranks' values; re-raises the first rank's error (the one that aborted the others, not a peer's abort)."""
    first = next((o.error for o in outcomes if o.error is not None and not isinstance(o.error, LoopbackAborted)), None)
    first = first or next((o.error for o in outcomes if o.error is not None), None)
    if first is not None:
        raise first
    return [o.value for o in outcomes]
