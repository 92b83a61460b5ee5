"""Placement arithmetic of a two-tier frame bank, shared by the LLaVA bank (ops.StreamBank) and the Qwen2-VL stream state
(qwen/stream_state.py): the first `device_frames` frames of a stream stay in HBM, later ones go to pinned host chunks
of `chunk_frames` frames each and never move again.  How each family lays out and allocates its chunks is its own."""
from __future__ import annotations

import numbers
from typing import Optional

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
