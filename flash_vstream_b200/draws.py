"""Where every k-means draw comes from: the package's RNG contract, in one place.

The reference's k-means draw `torch.randperm` for the initial centroids (LLaVA compress_functions.py:134 on the tensor's
device, :93 on the CPU; Qwen :211) and one `random.randint` per cluster that ends an iteration EMPTY (LLaVA :152 and
:107, Qwen :258).  That count is only known on the device after the Lloyd loop, so the kernels take every possible refill
up front: `refill_candidates` draws them from a private clone of the source's `random`, and the source is then advanced
by exactly the count the device consumed — lazily through `Refills.consumed_from` (a pinned read-back, applied at the
source's next draw or by `settle()`), or eagerly through `consume` when the count is already on the host.

A `DrawSource` is either
  * `GLOBAL`: torch's default generators and the `random` module, what the reference's functions draw from.  The mirrored
    functions of both model families and the single-stream model share it, as the reference's would; or
  * `DrawSource(seed, device)`: a torch CPU state, a CUDA state for `device` (none for "cpu") and a `random.Random(seed)`,
    for a `StreamPool` stream (in the reference each stream is its own process).  It draws what `GLOBAL` draws after
    `torch.manual_seed(seed); random.seed(seed)`.

Invariants:
  1. Every draw settles its source first, so it starts where the reference's generator would be.
  2. Global `random` is only ever advanced, never set: a user's `random.seed()` between two calls is never undone.
  3. An owned source never changes global torch or `random` state.
  4. Every site draws the values the reference draws from the same generator positions.
"""
from __future__ import annotations

import random
from typing import Optional

import numpy as np
import torch


def to_device(values, dtype, device) -> torch.Tensor:
    """host integers -> a numpy-`dtype` tensor on `device`, through pinned memory on a GPU (a pageable H2D copy would
    serialise the stream; pinning needs a GPU)"""
    t = torch.from_numpy(np.ascontiguousarray(values, dtype=dtype))
    if torch.device(device).type == "cuda":
        t = t.pin_memory()
    return t.to(device, non_blocking=True)


class Refills:
    """The refill candidates of one `refill_candidates` call; tell it how many the device consumed."""

    def __init__(self, source: "DrawSource", T: int):
        self._source, self._T = source, T

    def consumed_from(self, info: torch.Tensor):
        """info: the k-means kernel's int32 [4] (info[1] = refills consumed).  A device tensor is read back asynchronously;
        the source is advanced at its next draw or settle()."""
        if info.is_cuda:
            info_h = torch.empty(4, dtype=torch.int32).pin_memory()
            info_h.copy_(info[:4], non_blocking=True)
            ev = torch.cuda.Event()
            ev.record()
        else:
            info_h, ev = info[:4], None
        self._source._pending.append((self._T, info_h, ev))


class DrawSource:
    """DrawSource(): the global generators.  DrawSource(seed, device): generators of its own (see the module docstring)."""

    def __init__(self, seed: Optional[int] = None, device=None):
        self._pending = []        # (T, info int32 [4] on the host, event | None): consumed counts not yet applied
        self.owned = seed is not None
        if not self.owned:
            self.py, self.device = random, None
            return
        self.device = torch.device(device)
        g = torch.Generator()
        g.manual_seed(seed)
        self.cpu, self.cuda = g.get_state(), None
        if self.device.type == "cuda":
            gc = torch.Generator(device=self.device)
            gc.manual_seed(seed)
            self.cuda = gc.get_state()
        self.py = random.Random(seed)

    def settle(self):
        """Advance `random` by the refills the device consumed in the calls made so far.  Blocks on their read-backs."""
        while self._pending:
            T, info_h, ev = self._pending.pop(0)
            if ev is not None:
                ev.synchronize()
            self._advance(T, int(info_h[1]))

    def _advance(self, T: int, count: int):
        for _ in range(count):
            self.py.randint(0, T - 1)

    def randperm(self, n: int, device) -> torch.Tensor:
        """torch.randperm(n, device=device) on this source's torch generators"""
        self.settle()
        if not self.owned:
            return torch.randperm(n, device=device)
        cuda = [self.device] if self.cuda is not None else []
        with torch.random.fork_rng(devices=cuda):           # the caller's states come back on the way out
            torch.set_rng_state(self.cpu)
            if cuda:
                torch.cuda.set_rng_state(self.cuda, self.device)
            perm = torch.randperm(n, device=device)
            self.cpu = torch.get_rng_state()
            if cuda:
                self.cuda = torch.cuda.get_rng_state(self.device)
        return perm

    def refill_candidates(self, T: int, n: int, device):
        """n draws of random.randint(0, T - 1) from a private clone of this source's `random`, as int32 on `device`, and
        the `Refills` handle through which the consumed count advances the source."""
        self.settle()
        clone = random.Random()
        clone.setstate(self.py.getstate())
        return to_device([clone.randint(0, T - 1) for _ in range(n)], np.int32, device), Refills(self, T)

    def consume(self, T: int, count: int):
        """advance the source by `count` refills of a k-means over T rows, the count already read back to the host"""
        self.settle()
        self._advance(T, count)

    def randints(self, lo: int, hi: int, n: int) -> list:
        """n draws of random.randint(lo, hi), each consumed as drawn (the coin flips of the drop variants)"""
        self.settle()
        return [self.py.randint(lo, hi) for _ in range(n)]

    def snapshot(self, device="cpu"):
        """The source's position, without settling: (torch CPU state, CUDA state or None, `random` state or None, the
        refill counts still owed, device).  For the global source `device` names the CUDA generator to include, and
        `random` is not part of it."""
        if self.owned:
            return self.cpu, self.cuda, self.py.getstate(), list(self._pending), self.device
        dev = torch.device(device)
        return torch.get_rng_state(), torch.cuda.get_rng_state(dev) if dev.type == "cuda" else None, None, None, dev

    def rewind(self, snap):
        """Back to `snap`: the torch states, and an owned source's `random` with the counts it owed then (a settle since
        is undone with them, so nothing is applied twice or lost).  The global `random` keeps its position, and every
        count it still owes stays owed."""
        cpu, cuda, py, pending, dev = snap
        if self.owned:
            self.cpu, self.cuda, self._pending = cpu, cuda, list(pending)
            self.py.setstate(py)
            return
        torch.set_rng_state(cpu)
        if cuda is not None:
            torch.cuda.set_rng_state(cuda, dev)


GLOBAL = DrawSource()
