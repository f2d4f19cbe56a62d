"""Ranks of the sharded bundle adjustment as threads of one process: `world` calls of `bundle.solve(..., rank=r,
world=W, allreduce=...)` on one device, joined by an all-reduce that works like NCCL's and checks that the ranks
agree on what they exchange.

* One device token (a lock) is held by a rank for its whole solve and given up only inside the all-reduce, after the
  device is idle: the ranks' kernels (cooperative PCG launches, persistent Schur kernels) never share the SMs, and the
  run does not depend on how the threads are scheduled.
* Every rank copies its buffer to the host and waits at a barrier; every rank then sums the copies in rank order in
  fp64 (so every rank gets the same bits) and writes the sum back.  Ranks whose `count` differs at the same call raise
  together; a rank that never arrives makes the barrier time out, which raises in the others (no hang).  Each rank logs
  the counts of its calls, and `run_ranks` fails with the logs side by side unless they are identical.
* `device=None`: the buffers are host pointers (numpy arrays, as in the gloo branch of opensfm_b200.dist), so the
  exchange can be exercised without a GPU.

Not a test module: the test files import it (pytest puts tests/ on sys.path)."""
from __future__ import annotations

import copy
import ctypes
import threading
from typing import Any, Callable, List, Optional

import numpy as np


class RankFailure(AssertionError):
    """The ranks failed or disagreed; the message holds every rank's error and the all-reduce counts side by side."""


class Exchange:
    """The all-reduce of `world` in-process ranks (see the module docstring)."""

    def __init__(self, world: int, device: Optional[int] = 0, timeout: float = 120.0):
        self.world, self.device, self.timeout = int(world), device, float(timeout)
        self.token = threading.Lock()
        self.cond = threading.Condition()
        self.generation, self.arrived, self.broken = 0, 0, False
        self.slots: List[Optional[np.ndarray]] = [None] * self.world
        self.counts: List[Optional[int]] = [None] * self.world
        self.logs: List[List[int]] = [[] for _ in range(self.world)]
        self.errors: List[Optional[BaseException]] = [None] * self.world   # raised in a rank's all-reduce
        self.finished = [False] * self.world

    def allreduce(self, rank: int) -> Callable[[int, int, int], None]:
        """The `allreduce(ptr, count, stream)` callable of rank `rank`."""

        def fn(ptr: int, count: int, stream: int) -> None:
            try:
                self._exchange(rank, int(ptr), int(count))
            except BaseException as e:
                self.errors[rank] = e
                with self.cond:   # the other ranks raise at once instead of waiting for the timeout
                    self.broken = True
                    self.cond.notify_all()
                raise

        return fn

    def _wait(self, rank: int, k: int, count: int) -> None:
        """A barrier of the `world` ranks that gives up when a rank failed or finished its solve, or on the timeout."""
        with self.cond:
            gen = self.generation
            self.arrived += 1
            if self.arrived == self.world:
                self.arrived, self.generation = 0, gen + 1
                self.cond.notify_all()
                return
            self.cond.wait_for(lambda: self.generation != gen or self.broken or any(self.finished), self.timeout)
            if self.generation != gen:
                return
            gone = [r for r in range(self.world) if self.finished[r]]
            failed = [r for r in range(self.world) if self.errors[r] is not None]
            why = ("rank(s) %s had finished their solve" % gone if gone else
                   "rank(s) %s failed" % failed if failed else
                   "not every rank arrived within %g s" % self.timeout)
            self.broken = True
            self.cond.notify_all()
        raise RankFailure("all-reduce #%d (count %d) on rank %d: %s" % (k, count, rank, why))

    def _exchange(self, rank: int, ptr: int, count: int) -> None:
        k = len(self.logs[rank])
        self.logs[rank].append(count)
        on_device = self.device is not None
        if on_device:
            import torch

            from opensfm_b200.dist import _CudaPtr

            torch.cuda.synchronize(self.device)
            dev = None
            if count > 0:
                dev = torch.as_tensor(_CudaPtr(ptr, count), device="cuda:%d" % self.device)
                mine = dev.cpu().numpy()
            else:
                mine = np.zeros(0)
            self.token.release()
        else:
            host = np.ctypeslib.as_array((ctypes.c_double * count).from_address(ptr)) if count > 0 else np.zeros(0)
            mine = host.copy()
        try:
            self.slots[rank], self.counts[rank] = mine, count
            self._wait(rank, k, count)
            if len(set(self.counts)) != 1:
                raise RankFailure("all-reduce #%d: the ranks' counts differ: %s" % (
                    k, ", ".join("rank %d: %d" % (r, c) for r, c in enumerate(self.counts))))
            acc = self.slots[0].copy()
            for r in range(1, self.world):
                acc += self.slots[r]
            self._wait(rank, k, count)   # every rank has read every slot before the next call overwrites its own
        finally:
            if on_device:
                self.token.acquire()
        if on_device:
            if count > 0:
                dev.copy_(torch.from_numpy(acc))
            torch.cuda.synchronize(self.device)
        else:
            host[:] = acc

    def finish(self, rank: int) -> None:
        """Rank `rank` left its solve: a rank still exchanging waits for it in vain, so it raises now."""
        with self.cond:
            self.finished[rank] = True
            self.cond.notify_all()

    def report(self, results_errors: List[Optional[BaseException]]) -> str:
        lines = []
        for r in range(self.world):
            e = self.errors[r] or results_errors[r]
            if e is not None:
                lines.append("rank %d: %s: %s" % (r, type(e).__name__, e))
        n = max(len(l) for l in self.logs)
        first = next((k for k in range(n) if len({tuple(l[k:k + 1]) for l in self.logs}) > 1), None)
        lines.append("all-reduce counts (call: %s)%s" % (" | ".join("rank %d" % r for r in range(self.world)),
                                                          "" if first is None else ", first difference at #%d" % first))
        lo = 0 if first is None else max(0, first - 12)   # the calls just before the first difference, and after it
        hi = n if first is None else min(n, first + 4)
        if first is None and n > 16:
            lo = n - 16
        if lo > 0:
            lines.append("  (%d earlier calls agree)" % lo)
        for k in range(lo, hi):
            row = " | ".join("%8s" % (l[k] if k < len(l) else "-") for l in self.logs)
            lines.append("  #%-3d %s%s" % (k, row, "   <--" if k == first else ""))
        return "\n".join(lines)


def run_threads(world: int, body: Callable[[int, Callable[[int, int, int], None]], Any], device: Optional[int] = 0,
                timeout: float = 120.0) -> List[Any]:
    """body(rank, allreduce) in `world` threads, each holding the device token for its whole call (device mode).
    Returns the bodies' results in rank order; raises RankFailure when a rank failed or the ranks' all-reduce counts
    differ."""
    ex = Exchange(world, device, timeout)
    results: List[Any] = [None] * world
    errors: List[Optional[BaseException]] = [None] * world

    def main(r: int) -> None:
        try:
            if device is not None:
                with ex.token:
                    results[r] = body(r, ex.allreduce(r))
            else:
                results[r] = body(r, ex.allreduce(r))
        except BaseException as e:
            errors[r] = e
        finally:
            ex.finish(r)

    threads = [threading.Thread(target=main, args=(r,), name="rank%d" % r) for r in range(world)]
    for t in threads:
        t.start()
    for t in threads:
        t.join()
    if any(e is not None for e in errors) or any(e is not None for e in ex.errors) or \
            any(l != ex.logs[0] for l in ex.logs):
        raise RankFailure("world %d:\n%s" % (world, ex.report(errors)))
    return results


def run_ranks(pb, world: int, device: int = 0, timeout: float = 120.0, **solve_kw) -> List[dict]:
    """bundle.solve of `pb` sharded over `world` in-process ranks on `device` (each rank solves its own deep copy);
    the results in rank order."""
    from opensfm_b200 import bundle

    def body(r, allreduce):
        return bundle.solve(copy.deepcopy(pb), device=device, rank=r, world=world, allreduce=allreduce, **solve_kw)

    return run_threads(world, body, device=device, timeout=timeout)
