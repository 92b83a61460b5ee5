"""The host tier of a two-tier frame bank, shared by the LLaVA bank (ops.StreamBank) and the Qwen2-VL stream state
(qwen/stream_state.py): the first `device_frames` frames of a stream stay in HBM, later ones go to pinned host chunks
of `chunk_frames` frames each and never move again.  `placement` is the arithmetic, `HostChunks` the chunks."""
from __future__ import annotations

import ctypes as C
import numbers
from typing import Optional

import torch

from . import _lib as L

CHUNK_BYTES = 1 << 28     # pinned host memory per chunk of spilled frames (the host allocator rounds up to a power of two)


def check_device_frames(v, who: str = "device_frames") -> Optional[int]:
    """None (every frame stays in HBM) or an integer >= 0; ValueError otherwise"""
    if v is None:
        return None
    if isinstance(v, bool) or not isinstance(v, numbers.Integral) or v < 0:
        raise ValueError(f"{who} must be an integer >= 0 or None, got {v!r}")
    return int(v)


def chunk_frames(frame_bytes: int, chunk_bytes: int = CHUNK_BYTES) -> int:
    """frames per host chunk: as many whole frames as fit in chunk_bytes, at least one"""
    return max(1, chunk_bytes // frame_bytes)


def placement(n0: int, t: int, device_frames: Optional[int], per_chunk: int):
    """Where frames [n0, n0 + t) of the two-tier bank go, as (chunk, dst, src, count) spans: chunk -1 is the device tier
    (dst = frame index), chunk c >= 0 the c-th host chunk (dst = frame within the chunk); src = frame within the clip.
    Frames below device_frames stay in HBM; frame f >= device_frames is frame f - device_frames of the host tier."""
    cap = n0 + t if device_frames is None else device_frames
    k = max(0, min(t, cap - n0))
    spans = [(-1, n0, 0, k)] if k else []
    s = k
    while s < t:
        c, off = divmod(n0 + s - cap, per_chunk)
        cnt = min(t - s, per_chunk - off)
        spans.append((c, off, s, cnt))
        s += cnt
    return spans


def host_device_ptr(t: torch.Tensor) -> int:
    """the mapped device address of a pinned host tensor (what a kernel dereferences for a zero-copy read)"""
    assert not t.is_cuda
    out = C.c_void_p()
    L.check(L.load().fvs_host_device_ptr(t.data_ptr(), C.byref(out)), "fvs_host_device_ptr")
    return out.value


class HostChunks:
    """The host tier of a frame bank: frames [0, n) of the tier in pinned chunks of `per_chunk` frames each, allocated
    on first use.  A frame is one row of each of its parts (the Qwen2-VL full-resolution bank: x rows and merged rows;
    every other bank: one part), and chunk c is one flat buffer [F part-0 rows | F part-1 rows | ...], F = per_chunk,
    which kernels read in place through its mapped device pointer.  Empty until lay_out() fixes the frame layout."""

    def __init__(self):
        self.chunks: list = []
        self.n = 0                            # frames written (or left as slots) so far
        self.dtype, self.shapes, self.per_chunk, self.frame_elems = None, (), 0, 0
        self._ptrs: list = []                 # mapped device pointers of the chunks, taken on first request
        self._table: Optional[torch.Tensor] = None
        self._in_table = 0

    def lay_out(self, dtype, shapes, chunk_bytes: int = CHUNK_BYTES) -> "HostChunks":
        """frames of one row of `shapes[p]` elements of dtype per part; per_chunk from chunk_bytes"""
        self.dtype, self.shapes = dtype, tuple(torch.Size(s) for s in shapes)
        self.frame_elems = sum(s.numel() for s in self.shapes)
        self.per_chunk = chunk_frames(self.frame_elems * dtype.itemsize, chunk_bytes)
        return self

    def view(self, c: int, part: int = 0) -> torch.Tensor:
        """the rows of `part` in chunk c, [per_chunk, *shapes[part]]"""
        F, off = self.per_chunk, sum(s.numel() for s in self.shapes[:part])
        return self.chunks[c][F * off: F * (off + self.shapes[part].numel())].view(F, *self.shapes[part])

    def write(self, first: int, parts=None, t: int = 0):
        """frames [first, first + t) of the tier from parts[p], the rows [t, *shapes[p]] of each part (device or host:
        asynchronous copies on the current stream, ordered before any later kernel that reads them); parts None: t
        slots left unwritten.  Chunks are allocated on first use."""
        if parts is not None:
            t = parts[0].shape[0]
        for c, dst, s, cnt in placement(first, t, 0, self.per_chunk):
            while len(self.chunks) <= c:
                self.chunks.append(torch.empty(self.per_chunk * self.frame_elems, dtype=self.dtype, pin_memory=True))
            for p, rows in enumerate(parts or ()):
                self.view(c, p)[dst: dst + cnt].copy_(rows[s: s + cnt], non_blocking=True)
        self.n = max(self.n, first + t)

    def ptrs(self) -> tuple:
        """the chunks' mapped device pointers, a host list (qwen.ops.TieredBank)"""
        self._ptrs += [host_device_ptr(b) for b in self.chunks[len(self._ptrs):]]
        return tuple(self._ptrs)

    def table(self, device) -> Optional[torch.Tensor]:
        """the chunks' mapped device pointers as a device int64 table (the gather, scatter and pixel-gather jobs), None
        while there is no chunk.  Built on first request and grown by doubling; new entries are stream-ordered fills,
        so no host wait."""
        ptrs = self.ptrs()
        k = self._in_table
        if len(ptrs) > k and (self._table is None or self._table.numel() < len(ptrs)):
            tab = torch.zeros(max(16, 2 * len(ptrs)), dtype=torch.int64, device=device)
            if k:
                tab[:k].copy_(self._table[:k])
            self._table = tab
        for i in range(k, len(ptrs)):
            self._table[i].fill_(ptrs[i])
        self._in_table = len(ptrs)
        return self._table

    def to_host(self, device_rows: Optional[torch.Tensor], part: int = 0) -> torch.Tensor:
        """the whole bank of `part` as one pinned host tensor: device_rows (the device tier, None when empty) D2H, then
        the tier's n frames H2H once the pending copies have landed (synchronises the current stream)"""
        n_dev = 0 if device_rows is None else device_rows.shape[0]
        out = torch.empty((n_dev + self.n,) + tuple(self.shapes[part]), dtype=self.dtype, pin_memory=True)
        if n_dev:
            out[:n_dev].copy_(device_rows, non_blocking=True)
        torch.cuda.current_stream().synchronize()
        for c in range(len(self.chunks)):
            s = c * self.per_chunk
            cnt = min(self.per_chunk, self.n - s)
            out[n_dev + s: n_dev + s + cnt].copy_(self.view(c, part)[:cnt])
        return out

    def nbytes(self) -> int:
        return sum(b.numel() * b.element_size() for b in self.chunks)
