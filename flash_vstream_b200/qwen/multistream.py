"""Many Qwen2-VL video streams on one GPU: `QwenStreamPool`, the Qwen2-VL counterpart of multistream.StreamPool
(DESIGN.md §3.15).

One `step` is one round over the listed streams, each with one clip:
  1. every clip is validated before anything is enqueued;
  2. temporal_pool builds each clip's half-resolution rows;
  3. ONE fvs_qwen_vit_encode call (QwenVisionBlocksB200) encodes all clips: the segments of one (h, w) form one grid entry
     whose t is their sum, so each resolution gets one attention launch.  A round that needs more than 16 grid entries or
     more than `TOWER_ROWS` rows is split into several calls (plan_tower_calls);
  4. ONE PatchMerger call merges every stream's new full-resolution frames;
  5. each stream's memory step is enqueued, the round waits ONCE for all their read-backs, and each stream is completed
     (QwenStreamState.complete).  Every stream runs QwenStreamState.enqueue_input; then ONE stream_state.enqueue_csm call
     steps the CSM half of every stream past its CSM length (ordered k-means, klarge retrieval, DAM gather, PatchMerger
     rows) as one job table per kernel (fvs_qwen_*_multi, DESIGN.md §3.17), and the round's read-backs land in one
     pinned [S, 8] buffer with one copy.  A round of fewer than BATCH_MIN_JOBS such streams makes one one-item call per
     stream instead, as a stream stepped alone does.

Exact by construction: the tower is invariant to batch composition (§3.7) and the merger is row-wise (§3.5), so a pool
stream gets the bits it gets alone through QwenStreamState with the same draws, however the round is composed or split.

RNG: each stream owns a `draws.DrawSource` seeded by `open(seed)` (contract in draws.py), so a stream draws what the
single-stream path draws after `torch.manual_seed(seed); random.seed(seed)` and never touches the global generators.
"""
from __future__ import annotations

import os
from typing import Optional

import torch

from .. import _lib as L
from ..draws import DrawSource
from . import ops as Q
from .stream_state import (_KMEANS_METHODS, PATCH_DIM, QwenStreamState, _rest_finish, check_compact_pixels,
                           check_device_frames, check_full_res_bank, check_lazy_full_res, enqueue_csm)
from .vision_tower import QwenVisionBlocksB200

MAX_GRIDS = 16            # grid entries one fvs_qwen_vit_encode call takes
TOWER_ROWS = 65536        # rows of one tower call (its workspace is about 30 KB per row at 1280 wide)


def plan_tower_calls(clips, max_rows: int, max_grids: int = MAX_GRIDS):
    """clips: per clip, its segments [(t, h, w), ...].  -> one (grids, places) per tower call: grids = [(t, h, w)] with
    every (h, w) of the call once and t summed over its segments; places = [(clip index, [first output row of each of its
    segments])].  Clips are taken in the order of their grids, so clips of one resolution share calls; a call takes
    clips while it stays within `max_grids` entries and `max_rows` rows (a clip larger than `max_rows` goes alone)."""
    order = sorted(range(len(clips)), key=lambda i: [(h, w) for _, h, w in clips[i]])
    calls, cur, keys, rows = [], [], set(), 0
    for i in order:
        ck = {(h, w) for _, h, w in clips[i]}
        n = sum(t * h * w for t, h, w in clips[i])
        if cur and (len(keys | ck) > max_grids or rows + n > max_rows):
            calls.append(cur)
            cur, keys, rows = [], set(), 0
        cur.append(i)
        keys |= ck
        rows += n
    if cur:
        calls.append(cur)
    return [_call_layout(clips, members) for members in calls]


def _call_layout(clips, members):
    tsum = {}                                             # (h, w) -> summed t, in first-seen order
    for i in members:
        for t, h, w in clips[i]:
            tsum[(h, w)] = tsum.get((h, w), 0) + t
    base, r = {}, 0
    for (h, w), t in tsum.items():
        base[(h, w)] = r
        r += t * h * w
    places = []
    for i in members:
        offs = []
        for t, h, w in clips[i]:
            offs.append(base[(h, w)])
            base[(h, w)] += t * h * w
        places.append((i, offs))
    return [(t, h, w) for (h, w), t in tsum.items()], places


def encode_picked(states, readbacks: torch.Tensor, max_rows: int = TOWER_ROWS):
    """The full-resolution half of a lazy_full_res round (DESIGN.md §3.18), for states whose retrieval is enqueued
    (state._lazy_ctx): ONE fvs_qwen_pick_plan_multi call plans every state's first-time frames (count of states[k] to
    slot 7 of readbacks[k], pinned int32 [>= len(states), 8]); the round's ONE host wait, when a count or a k-means
    read-back is still on its way (a DAM that is the whole bank plans the frames not yet encoded, and an empty DAM,
    spatial_length 0, nothing: counts the host knows); then the planned frames' pixel rows go through one fvs_qwen_pixel_gather_multi, the tower and the
    PatchMerger per tower call (plan_tower_calls), and fvs_qwen_bank_scatter_multi writes them into the banks.  Last,
    the DAM gathers and the CSM merger of every state (stream_state._rest_finish).  The tower, the first state's, is
    invariant to batch composition (§3.7) and the merger row-wise (§3.5), so each frame gets the bits of the eager
    path.
    A state without full_res_bank (§3.19) plans the picks its previous DAM does not hold (a DAM that is the whole bank
    plans the frames the previous one did not have, a count the host knows).  Its tower and merger rows are not
    scattered anywhere: they stay as the state's fresh rows, which the DAM gather reads beside the previous DAM, and are
    dropped after it.  A state with compact_pixels (§3.20) gathers its codes with their table, decoded into the rows a
    store of tower-dtype rows would give."""
    if any(st._lazy_ctx["n_spa"] and st.tower is None for st in states):     # refused before any mask byte is set
        raise NotImplementedError("lazy_full_res: no full-resolution tower was given to the stream state")
    addr = Q.host_device_ptr(readbacks)
    jobs, counts = [], []
    for k, st in enumerate(states):
        c = st._lazy_ctx
        n_spa, n = c["n_spa"], st.n_frames
        st._plan = torch.empty(max(1, n_spa), dtype=torch.int64, device=st.encoded.buf.device)
        if n_spa == 0:                     # spatial_length 0: nothing is ever retrieved, so nothing is encoded
            counts.append(0)
            continue
        # a DAM that is the whole bank is frames [0, n) (spatial_picks returns arange while n <= spatial_length)
        whole = n_spa == n
        count = addr + (k * 8 + 7) * readbacks.element_size()
        prev = None if st.full_res_bank else st._prev_dam          # a bank holds every encoded frame: the mask says it
        if not st.full_res_bank and st.re_encodes is None:
            st.re_encodes = torch.zeros(1, dtype=torch.int64, device=st._plan.device)
        jobs.append((None if whole else c["picks"], n_spa, st.encoded.buf, n, st._plan, count,
                     1 if st.full_res_bank else 2, None if prev is None else prev[0], st.re_encodes))
        if not whole:
            counts.append(None)
        else:                              # the frames not yet encoded; without a bank, those the previous DAM lacks
            counts.append(n - (st.n_encoded if st.full_res_bank else 0 if prev is None else prev[0].numel()))
    if jobs:
        Q.pick_plan_multi(jobs)
    if any(v is None for v in counts) or any(st._pending for st in states):
        done = torch.cuda.Event()
        done.record()
        done.synchronize()
    counts = [int(readbacks[k, 7]) if v is None else v for k, v in enumerate(counts)]
    todo = [(st, n) for st, n in zip(states, counts) if n]
    for st, n in todo:
        st.n_encoded += n
    if todo:
        tower, merger = todo[0][0].tower, todo[0][0].merger
        for grids, places in plan_tower_calls([[(n, *st.grid)] for st, n in todo], max_rows):
            rows = sum(t * h * w for t, h, w in grids)
            inp = torch.empty(rows, PATCH_DIM, dtype=todo[0][0].pixels.out_dtype, device=todo[0][0].encoded.buf.device)
            gathers = []                   # one kind: the states of a round share compact_pixels
            for i, (off,) in places:
                st, n = todo[i]
                px = st.pixels
                gathers.append((st._plan, n, st.n_frames, px.base, px.table, px.chunk_frames,
                                inp[off: off + n * st.grid[0] * st.grid[1]], px.frame_elems, px.values))
            Q.pixel_gather_multi(gathers)
            feats = tower(inp, grids)
            merged = merger(feats) if len(todo[0][0].bank_tier.shapes) > 1 else None
            scatters = []
            for i, (off,) in places:
                st, n = todo[i]
                r = n * st.grid[0] * st.grid[1]
                rows = (feats[off: off + r], None if merged is None else merged[off // 4: (off + r) // 4])
                if st.full_res_bank:
                    scatters.append(st._scatter_args(n, *rows))
                else:
                    st._fresh = (st._plan, n) + rows
            if scatters:
                Q.bank_scatter_multi(scatters)
    ctxs = []
    for st in states:
        ctxs.append((st, st._lazy_ctx))
        st._lazy_ctx, st._in_round = None, False
    _rest_finish(ctxs)
    for st in states:
        st._fresh = None                   # the DAM holds the fresh rows it picked now


class _Stream:
    """one pool stream; it has what qwen.serve.export_qwen_memory reads of a host (visual, stream_state), so it can be
    exported like one"""

    def __init__(self, visual, state: QwenStreamState):
        self.visual, self.stream_state = visual, state


class QwenStreamPool:
    """A pool of Qwen2-VL streams sharing one realtime host's vision side (visual: VisualB200 with a QwenVisionBlocksB200
    tower, its FlashMemory config and PatchMerger).

    `open(seed)` -> sid; `step({sid: (pixel_values_videos, video_grid_thw), ...})` advances the listed streams by one clip
    each (what the Qwen2-VL processor returns: patch rows [t*h*w, 1176] and one (t, h, w) grid); `state(sid)` is the
    stream's QwenStreamState, `as_list(sid)` its 13-item list; `stream(sid)` can be handed to qwen.serve.export_qwen_memory.
    `checkpoint(sid)` / `open(checkpoint=)` suspend and resume a stream; `close(sid)` drops it.  Configs and towers the
    batched round does not cover raise NotImplementedError naming the knob: stream them through the host's single-stream
    path.  `device_frames` and `small_device_frames` apply to every stream, as `fvs_bank_device_frames` and
    `fvs_bank_small_device_frames` do to the host's stream (DESIGN.md §3.13).  TOWER_ROWS bounds the rows of one tower
    call (its workspace is about 30 KB per row at 1280 wide).  `preprocess` (a preprocess.Qwen2VLFramePreprocessor):
    `step` also takes decoded uint8 frames [T, H, W, 3] per stream (any mix of sizes, host or device); the round's clips
    go through ONE `preprocess.many` call, and each stream's rows and grid then make its (pixel_values_videos,
    video_grid_thw).  `lazy_full_res` (QwenStreamState's): the round runs the full-resolution tower once, after its one
    host wait, on only the frames some stream's DAM picks for the first time (encode_picked, DESIGN.md §3.18).
    `full_res_bank=False` (with lazy_full_res): every stream keeps no full-resolution or merged rows beyond its DAM, and
    the round's one tower pass also re-encodes the picks a stream's previous DAM does not hold (§3.19).
    `compact_pixels=True` (with lazy_full_res and a Qwen2VLFramePreprocessor): the round's frames come out of
    `preprocess.many` as uint8 codes, ONE fvs_qwen_pixel_decode call makes the tower's rows of the whole round from
    them, and each stream keeps the codes, half the pinned bytes of tower-dtype rows; its re-encodes decode as they
    gather (§3.20).  Rounds of (pixels, grid) clips are refused.  The knobs are the pool's: eager, lazy and bank-less
    streams do not share a pool."""

    TOWER_ROWS = TOWER_ROWS
    BATCH_MIN_JOBS = 4        # fewer k-means streams in a round take one enqueue_csm call each

    def __init__(self, model, device_frames: Optional[int] = None, max_streams: Optional[int] = None,
                 small_device_frames: Optional[int] = None, preprocess=None, lazy_full_res: bool = False,
                 full_res_bank: bool = True, compact_pixels: bool = False):
        visual = model.visual
        flash, tower = visual.flash_memory, visual.encode_patches
        if not isinstance(tower, QwenVisionBlocksB200):
            raise NotImplementedError("QwenStreamPool: visual.encode_patches is not a QwenVisionBlocksB200 tower, which the "
                                      "batched round encodes through; stream this host through its single-stream path")
        if flash.temporal_method not in _KMEANS_METHODS:
            raise NotImplementedError(f"QwenStreamPool: flash_memory_temporal_method={flash.temporal_method!r} is outside "
                                      f"what the batched round covers ({', '.join(_KMEANS_METHODS)}); stream it through "
                                      f"the host's single-stream path")
        if flash.temporal_poolsize != 2:
            raise NotImplementedError(f"QwenStreamPool: flash_memory_temporal_poolsize={flash.temporal_poolsize} is outside "
                                      f"what the batched round covers (2); stream it through the host's single-stream path")
        self.device = torch.device(visual.get_device())
        if self.device.type != "cuda":
            raise L.FvsError("QwenStreamPool needs the vision side on a CUDA device (no CPU fallback)")
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        self.visual, self.flash, self.merger, self.tower = visual, flash, visual.merger, tower
        self.device_frames = check_device_frames(device_frames, "device_frames")
        self.small_device_frames = check_device_frames(small_device_frames, "small_device_frames")
        self.lazy_full_res = check_lazy_full_res(lazy_full_res, flash)
        self.full_res_bank = check_full_res_bank(full_res_bank, self.lazy_full_res)
        self.compact_pixels = check_compact_pixels(compact_pixels, self.lazy_full_res)
        if self.compact_pixels:
            from ..preprocess import Qwen2VLFramePreprocessor
            if not isinstance(preprocess, Qwen2VLFramePreprocessor):
                raise ValueError("QwenStreamPool: compact_pixels=True needs preprocess=Qwen2VLFramePreprocessor(...): the "
                                 "codes are what it makes of uint8 frames")
        self.max_streams = max_streams
        self.preprocess = preprocess
        self._readbacks: Optional[torch.Tensor] = None     # pinned int32 [S, 8]: the round's read-backs
        self._streams: dict[int, _Stream] = {}
        self._next = 0

    # ---- streams -------------------------------------------------------------------------------------------------------
    def open(self, seed: Optional[int] = None, *, checkpoint=None) -> int:
        """A new stream -> its sid.  With `checkpoint` (of `checkpoint(sid)`, from this pool or another, on any device, or
        of a host's save_video_stream()), the stream continues where the checkpoint left it: its state and, when the
        checkpoint carries them, its generators.  A checkpoint without them (from the single-stream host, whose draws come
        from the global generators) needs `seed=` for the generators the stream draws from from here on."""
        if self.max_streams is not None and len(self._streams) >= self.max_streams:
            raise RuntimeError(f"QwenStreamPool is full ({self.max_streams} streams)")
        if checkpoint is not None and checkpoint.rng is None and seed is None:
            raise ValueError("QwenStreamPool.open: this checkpoint carries no draw source (single-stream host): pass seed=")
        if checkpoint is None:
            state = QwenStreamState(self.flash, self.merger, device_frames=self.device_frames,
                                    small_device_frames=self.small_device_frames, lazy_full_res=self.lazy_full_res,
                                    full_res_bank=self.full_res_bank, compact_pixels=self.compact_pixels)
        else:
            state = QwenStreamState.restore(checkpoint, self.flash, self.merger, self.device, device_frames=self.device_frames,
                                            small_device_frames=self.small_device_frames,
                                            lazy_full_res=self.lazy_full_res, full_res_bank=self.full_res_bank,
                                            compact_pixels=self.compact_pixels, pixel_table=self._pixel_table())
        state.tower = self.tower
        state.pixel_table = self._pixel_table()
        if seed is None and checkpoint is None:
            seed = int.from_bytes(os.urandom(8), "little") >> 1
        rng = DrawSource(int(seed) if seed is not None else 0, self.device)
        if checkpoint is not None and checkpoint.rng is not None:
            r = checkpoint.rng
            rng.cpu = r["cpu"].clone()
            rng.cuda = r["cuda"].clone() if rng.cuda is not None and r["cuda"] is not None else rng.cuda
            rng.py.setstate(r["py"])
        state.rng = rng
        sid = self._next
        self._next += 1
        self._streams[sid] = _Stream(self.visual, state)
        return sid

    def checkpoint(self, sid: int):
        """The stream as a StreamCheckpoint in pinned host memory: its QwenStreamState and its draw source (settled first,
        so no consumed refill count is lost or applied twice).  Suspend = checkpoint(sid) then close(sid); resume =
        open(checkpoint=...) here or in another pool, or a host's load_video_stream()."""
        from .. import checkpoint as CK
        state = self._streams[sid].stream_state
        state.rng.settle()
        ck = state.checkpoint()
        ck.rng = CK.rng_state(state.rng)
        return ck

    def close(self, sid: int):
        del self._streams[sid]

    def __len__(self):
        return len(self._streams)

    def stream(self, sid: int) -> _Stream:
        return self._streams[sid]

    def state(self, sid: int) -> QwenStreamState:
        return self._streams[sid].stream_state

    def as_list(self, sid: int):
        """the stream's 13-item `video_embedding_memory` list (QwenStreamState.as_list)"""
        return self._streams[sid].stream_state.as_list()

    def _pixel_table(self):
        """compact_pixels: the preprocessor's value table on the pool's device (None otherwise)"""
        return self.preprocess.device_table(self.device) if self.compact_pixels else None

    # ---- one round -----------------------------------------------------------------------------------------------------
    def _validate(self, sid, clip):
        """-> (pixel rows on the device in the tower's dtype, t, h, w); raises before anything is enqueued"""
        if sid not in self._streams:
            raise KeyError(f"QwenStreamPool.step: no stream {sid}")
        pix, thw = clip
        thw = torch.as_tensor(thw).reshape(-1, 3)
        if thw.shape[0] != 1:
            raise ValueError(f"QwenStreamPool.step: stream {sid}: one clip per stream (got {thw.shape[0]} grids)")
        t, h, w = (int(v) for v in thw[0].tolist())
        if t < 1 or h < 1 or w < 1 or h % 2 or w % 2:
            raise ValueError(f"QwenStreamPool.step: stream {sid}: bad grid (t, h, w) = ({t}, {h}, {w})")
        for name, side in (("pad_h", h), ("pad_w", w)):            # the reference's temporal_pool (pool size 2)
            if (side // 2) % 2:
                raise NotImplementedError(f"Performing temporal pool, {name} > 0, {name}={(side // 2) % 2}")
        if pix.numel() != t * h * w * PATCH_DIM:
            raise ValueError(f"QwenStreamPool.step: stream {sid}: {tuple(pix.shape)} pixels do not match the grid "
                             f"({t}, {h}, {w})")
        if pix.is_cuda and pix.device != self.device:
            raise ValueError(f"QwenStreamPool.step: stream {sid}: pixels on {pix.device}, the pool is on {self.device}")
        grid = self._streams[sid].stream_state.grid
        if grid is not None and grid != (h, w):
            raise ValueError(f"QwenStreamPool.step: stream {sid}: grid {(h, w)} differs from the stream's grid {grid}")
        return pix, t, h, w

    def _encode(self, items, codes=None):
        """items: [(pixels, t, h, w)] -> per item (x_new [t*h*w, D], small_new [t*h*w/4, D]) through as few tower calls
        as plan_tower_calls allows; with lazy_full_res, (the pixel rows [t*h*w, 1176] on the device, small_new): only the
        half-resolution rows go through the tower here; with compact_pixels, (the item's codes, small_new)"""
        rows, segs, fulls = [], [], []
        for pix, t, h, w in items:
            full = pix.type(self.visual.get_dtype()).to(self.device, non_blocking=True).view(-1, PATCH_DIM)
            small, _ = self.flash.temporal_pool(full, [t, h, w])
            fulls.append(full)
            if self.lazy_full_res:
                rows.append((small,))
                segs.append([(t, h // 2, w // 2)])
            else:
                rows.append((full, small))
                segs.append([(t, h, w), (t, h // 2, w // 2)])
        out = [None] * len(items)
        for grids, places in plan_tower_calls(segs, self.TOWER_ROWS):
            pieces = sorted(((off, rows[i][k]) for i, offs in places for k, off in enumerate(offs)), key=lambda p: p[0])
            feats = self.tower(torch.cat([p for _, p in pieces]) if len(pieces) > 1 else pieces[0][1], grids)
            for i, offs in places:
                out[i] = tuple(feats[off: off + r.shape[0]] for off, r in zip(offs, rows[i]))
        if self.lazy_full_res:
            out = [(full, o[0]) for full, o in zip(fulls if codes is None else codes, out)]
        return out

    def step(self, clips: dict, draws: Optional[dict] = None):
        """One round: one clip for every stream in `clips` ({sid: (pixel_values_videos, video_grid_thw)}); the other
        streams do not move.  draws={sid: dict} replays a stream's draws (the `draws` of QwenStreamState.step).  A refused
        round raises before anything is enqueued: no stream moves and no generator advances.  A stream whose clip raises
        while being completed (ZeroDivisionError on an empty cluster, as the reference) is left as the single-stream
        path leaves it; every other stream completes, and then the round raises one error naming the failing sids
        (`.errors`: sid -> exception).  With `preprocess`, a round of uint8 frames ({sid: [T, H, W, 3]}) is pre-processed
        in one call first; a round mixing them with (pixels, grid) clips is refused, and so is a round of (pixels, grid)
        clips in a compact_pixels pool."""
        draws = draws or {}
        sids = list(clips)
        frames = {not isinstance(clips[sid], (tuple, list)) for sid in sids}
        if len(frames) > 1:
            raise ValueError("QwenStreamPool.step: one round takes uint8 frames or (pixels, grid) clips for every stream, "
                             "not a mix")
        codes = None
        if frames == {True}:
            if self.preprocess is None:
                raise ValueError("QwenStreamPool.step: uint8 frames need a pool made with "
                                 "preprocess=Qwen2VLFramePreprocessor(...)")
            for sid in sids:
                if sid not in self._streams:
                    raise KeyError(f"QwenStreamPool.step: no stream {sid}")
            out, rows, grids = self.preprocess.many([clips[sid] for sid in sids], codes=self.compact_pixels)
            if self.compact_pixels:              # one decode of the round's codes into the rows the tower reads
                out = out.to(self.device, non_blocking=True)
                full, r, codes, rows = Q.pixel_decode(out, self._pixel_table(), self.visual.get_dtype()), 0, [], []
                for g in grids:
                    n = int(torch.prod(g))
                    codes.append(out[r: r + n])
                    rows.append(full[r: r + n])
                    r += n
            clips = dict(zip(sids, zip(rows, grids)))
        items = [self._validate(sid, clips[sid]) for sid in sids]
        if codes is None and self.compact_pixels:
            raise ValueError("QwenStreamPool.step: a compact_pixels pool keeps uint8 codes, which only uint8 frames give: "
                             "(pixels, grid) clips are refused")
        feats = self._encode(items, codes)
        merged = [None] * len(sids)
        if self.lazy_full_res:
            self._readback_rows(len(sids))
            states = [self._streams[sid].stream_state for sid in sids]
            for st in states:
                st._in_round = True
            try:
                self._enqueue_memory(sids, items, feats, merged, draws)
            finally:
                started = [st for st in states if st._lazy_ctx is not None]
                for st in states:
                    st._in_round = False
                if started:                            # the round's one host wait is in there
                    encode_picked(started, self._readbacks, self.TOWER_ROWS)
            self._complete(sids)
            return
        if self.flash.spatial_length > 0 and self.merger is not None:
            xs = [x for x, _ in feats]
            m = self.merger(torch.cat(xs) if len(xs) > 1 else xs[0])
            r = 0
            for k, x in enumerate(xs):
                merged[k] = m[r: r + x.shape[0] // 4]
                r += x.shape[0] // 4
        pending = self._enqueue_memory(sids, items, feats, merged, draws)
        if pending:                                    # the round's one host wait: every stream's read-back has landed
            done = torch.cuda.Event()
            done.record()
            done.synchronize()
        self._complete(sids)

    def _enqueue_memory(self, sids, items, feats, merged, draws) -> bool:
        """every listed stream's memory step, enqueued; -> whether any stream reads back.  The streams whose clip needs
        the CSM k-means (past the CSM length) are collected and stepped by one enqueue_csm call, or, in a round of fewer
        than BATCH_MIN_JOBS of them, by one one-item call each (a job table does not pay off there, DESIGN.md §4); the
        others (memory still filling) run their pass-through inside enqueue_input.  Should a stream's enqueue_input
        raise, the streams collected before it are enqueued first, so the round leaves every stream as stepping each
        stream alone would."""
        reqs = []                                      # (state, k-means request) of the round
        try:
            for k, sid in enumerate(sids):
                st = self._streams[sid]
                _, t, h, w = items[k]
                pub = st.__dict__.get("_qwen_publication")
                if pub is not None and st.stream_state.n_frames == 0:
                    pub.new_stream()
                _, req = st.stream_state.enqueue_input(feats[k][0], feats[k][1], t, (h, w), (h // 2, w // 2),
                                                       st.stream_state.n_frames, draws=draws.get(sid), merged=merged[k])
                if req is not None:
                    reqs.append((st.stream_state, req))
        finally:
            if reqs:
                n = len(reqs)
                self._readback_rows(n)
                if n >= self.BATCH_MIN_JOBS:
                    enqueue_csm(reqs, self._readbacks)
                else:
                    for i, item in enumerate(reqs):
                        enqueue_csm([item], self._readbacks[i: i + 1])
        return bool(reqs)

    def _readback_rows(self, n: int):
        if self._readbacks is None or self._readbacks.shape[0] < n:
            self._readbacks = torch.empty(max(n, 2 * (0 if self._readbacks is None else self._readbacks.shape[0])), 8,
                                          dtype=torch.int32).pin_memory()

    def _complete(self, sids):
        """complete every enqueued stream of the round and publish it; then raise one error for those that raised"""
        errors = {}
        for sid in sids:
            st = self._streams[sid]
            try:
                st.stream_state.complete()
            except Exception as e:                     # noqa: BLE001 - reported below, once every stream is completed
                errors[sid] = e
                continue
            pub = st.__dict__.get("_qwen_publication")
            if pub is not None:
                pub.publish(st.stream_state)
        if errors:
            kinds = {type(e) for e in errors.values()}
            cls = kinds.pop() if len(kinds) == 1 and ZeroDivisionError in kinds else RuntimeError
            err = cls(f"QwenStreamPool.step: stream(s) {sorted(errors)} raised: "
                      + "; ".join(f"{sid}: {type(e).__name__}: {e}" for sid, e in errors.items()))
            err.errors = errors
            raise err from next(iter(errors.values()))
