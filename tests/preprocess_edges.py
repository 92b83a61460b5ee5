"""Poisoned neighbours and guarded outputs for tests/test_preprocess_edges_gpu.py (pure torch: the host tests run the
checker on the CPU).

Every call of the sweep runs twice, once per poison.  The frames of each job sit at the start of a buffer whose tail
holds the poison byte, the workspace (and a tail past the size the call is given) is filled with it, and the output
sits inside a buffer whose guard elements before the first job and after the last hold the output sentinel.  A kernel
that reads past its frames or reads workspace it never wrote gives different bytes under the two poisons; an output
element it never writes keeps the run's sentinel, so it differs between the runs too; a store outside the outputs
changes a guard.  uint8 outputs take the poison bytes as sentinels; f16 / fp32 outputs take NaNs with two different
payloads (the value table is finite, so no written element is NaN).  Everything is compared as integers, bit for bit."""
from __future__ import annotations

import torch

POISON = (0x00, 0xFF)                                                  # frame tails and workspace, per run
SENTINEL = {torch.uint8: (0x00, 0xFF), torch.float16: (0x7D5A, 0xFEA5), torch.float32: (0x7FC0A5A5, 0xFFA55A5A)}
GUARD = 512                                                            # output guard elements on either side
TAIL = 4096                                                            # poison bytes past frames and workspace
_INT = {1: torch.uint8, 2: torch.int16, 4: torch.int32}


def as_int(t: torch.Tensor) -> torch.Tensor:
    """the bits of `t` as a same-width integer tensor"""
    return t.view(_INT[t.element_size()])


def signed(bits: int, dtype) -> int:
    """`bits` as the integer as_int shows for a dtype-wide element"""
    n = 8 * torch.empty((), dtype=dtype).element_size()
    return bits - (1 << n) if dtype != torch.uint8 and bits >= 1 << (n - 1) else bits


def poisoned_frames(frames: torch.Tensor, run: int) -> torch.Tensor:
    """a flat uint8 buffer: the bytes of `frames`, then TAIL bytes of the run's poison"""
    n = frames.numel()
    buf = torch.full((n + TAIL,), POISON[run], dtype=torch.uint8, device=frames.device)
    buf[:n].copy_(frames.reshape(-1))
    return buf


def poisoned_workspace(nbytes: int, run: int, device) -> torch.Tensor:
    """nbytes of workspace and TAIL more, all the run's poison (a call is given only the first nbytes)"""
    return torch.full((nbytes + TAIL,), POISON[run], dtype=torch.uint8, device=device)


def guarded_output(n: int, dtype, run: int, device) -> tuple[torch.Tensor, torch.Tensor]:
    """(buffer, view): GUARD + n + GUARD elements of the run's sentinel; view is the n in the middle"""
    buf = torch.empty(n + 2 * GUARD, dtype=dtype, device=device)
    as_int(buf).fill_(signed(SENTINEL[dtype][run], dtype))
    return buf, buf[GUARD:GUARD + n]


def report(name: str, outs, workspaces=(), ws_bytes: int = 0, frames=(), frame_bytes=()) -> list[str]:
    """the problems of one call run under both poisons: `outs` the two guarded output buffers; `workspaces` the two
    workspaces (ws_bytes given to the call, the tail past it must keep the poison); `frames` the two runs' poisoned
    frame buffers of each job ([run][job]) with the job's frame bytes (the tails must keep the poison)"""
    probs = []
    dtype = outs[0].dtype
    n = outs[0].numel() - 2 * GUARD
    for run, buf in enumerate(outs):
        ib, s = as_int(buf), signed(SENTINEL[dtype][run], dtype)
        bad = torch.cat([ib[:GUARD], ib[GUARD + n:]]) != s
        if bool(bad.any()):
            where = int(bad.nonzero()[0])
            where = where - GUARD if where < GUARD else n + where - GUARD
            probs.append(f"{name}: run {run}: {int(bad.sum())} output guard elements changed (first at element {where} "
                         f"of the output)")
    a, b = (as_int(o)[GUARD:GUARD + n] for o in outs)
    diff = a != b
    if bool(diff.any()):
        left = int(((a == signed(SENTINEL[dtype][0], dtype)) & (b == signed(SENTINEL[dtype][1], dtype))).sum())
        probs.append(f"{name}: {int(diff.sum())} output elements differ between the two poisons, {left} of them still "
                     f"the sentinel (never written); first at element {int(diff.nonzero()[0])}")
    for run, ws in enumerate(workspaces):
        bad = ws[ws_bytes:] != POISON[run]
        if bool(bad.any()):
            probs.append(f"{name}: run {run}: {int(bad.sum())} workspace bytes past the {ws_bytes} given were written")
    for run, bufs in enumerate(frames):
        for j, (buf, nb) in enumerate(zip(bufs, frame_bytes)):
            if bool((buf[nb:] != POISON[run]).any()):
                probs.append(f"{name}: run {run}: the poison past job {j}'s frames was written")
    return probs
