"""Device-resident state of the Qwen2-VL streaming Flash Memory and its per-clip update — the GPU-resident form of
FlashVStreamQwen2VLModel.embed_new_video_clip (Flash-VStream-Qwen/models/vstream_qwen2vl_realtime.py:548-630).

The reference rebuilds its 13-item state list from host-driven pieces every clip (cat old + new, k-means whose cluster
count, member lists, timestamps and ordering are computed on the CPU from `.item()` / `.cpu()` reads, a merger pass over
all 6480 memory tokens) and parks the list on the CPU in between.  Here the state is one object in HBM and a clip is ONE
enqueue pass with ONE 32-byte read-back at its end:

  * every shape of a step is known on the host beforehand (frames per clip, carried centroids = min(frames so far, T0),
    retrieved frames = min(frames so far, S0)), so the host never has to ask the device how large something is;
  * the data-dependent scalars of the k-means — number of distinct rows, exit iteration, refill draws consumed, empty
    clusters — are produced on the device and copied, together, into pinned memory after the last kernel of the step has
    been enqueued; the step is published once that copy has landed and says the enqueued work was the right work;
  * the right work is the common case: the reference draws `torch.randperm(n_unique)` for the initial centroids, so the
    step assumes all T rows are distinct (n_unique == T), draws randperm(T) and runs the non-degenerate branch; should the
    read-back show duplicates, the torch generators are rewound and the clip is redone through the synchronous path
    (weighted_kmeans_ordered_feature), which handles every branch of the reference;
  * timestamps (mean member index), their ordering and the sorted gather run on the device (fvs_qwen_kmeans_finalize); the
    member lists the reference returns are materialised lazily — nothing in the streaming step reads them;
  * the PatchMerger is row-wise over groups of 4 tokens: DAM rows are verbatim bank frames, so each frame is merged once,
    when it enters the bank, and a step merges only its new frames and the CSM centroids (2160 + 144 t of the 6480 + 144 t
    rows) and gathers the retrieved frames' merged rows.

`RealtimeStreamingMixin` (vstream_qwen2vl_realtime.py of this package) keeps the reference's method names and the 13-item
list on top of this object.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from . import compress_functions as CF
from . import ops as Q
from .. import ops as O
from ..draws import GLOBAL, to_device
from ..host_tier import CHUNK_BYTES, HostChunks, check_device_frames, chunk_frames, placement  # noqa: F401

_KMEANS_METHODS = ("kmeans_ordered", "fast_kmeans_ordered")
PATCH_DIM = 3 * 2 * 14 * 14           # elements of one full-resolution pixel row (what the tower reads)


class RowBank:
    """append-only row store in HBM with capacity doubling; `rows()` is a view of the filled part"""

    def __init__(self):
        self.buf: Optional[torch.Tensor] = None
        self.n = 0

    def append(self, rows: torch.Tensor) -> torch.Tensor:
        need = self.n + rows.shape[0]
        if self.buf is None or need > self.buf.shape[0] or self.buf.dtype != rows.dtype:
            cap = max(need, 2 * (self.buf.shape[0] if self.buf is not None else 0))
            new = torch.empty((cap,) + tuple(rows.shape[1:]), dtype=rows.dtype, device=rows.device)
            if self.buf is not None and self.n:
                new[: self.n].copy_(self.buf[: self.n])
            self.buf = new
        self.buf[self.n: need].copy_(rows)
        self.n = need
        return self.buf[: self.n]

    def rows(self) -> torch.Tensor:
        return self.buf[: self.n]


class QwenStreamState:
    """flash: the streaming FlashMemory (temporal_length / spatial_length in frames, methods); merger: PatchMerger.
    device_frames: how many frames of the full-resolution and merged banks stay in HBM (None: all of them).  Later frames
    are copied to pinned host chunks as they arrive and never move again; a step reads only its retrieved frames from
    them (fvs_qwen_dam_gather_multi).
    small_device_frames: how many frames of the half-resolution bank stay in HBM (None: all of them).  Later frames go to
    pinned host chunks of their own; the klarge retrieval sweeps them in place over PCIe (fvs_qwen_klarge_retrieve_tiered),
    once per step, twice with the cosine metric.  The two caps are independent; results are bit-identical either way.
    lazy_full_res: keep each clip's full-resolution pixel rows in pinned host chunks instead of its tower features, and
    run the full-resolution tower on a frame only the first time the DAM picks it (DESIGN.md §3.18); step() then takes
    the pixel rows in place of x_new, and the tower.  The published bits are the eager state's.
    full_res_bank: False (with lazy_full_res only) keeps no full-resolution or merged row of the frames the stream
    encodes: the step gathers its DAM from the previous DAM and from this step's tower output, and re-encodes a pick the
    previous DAM does not hold from its pixel rows (DESIGN.md §3.19).  Same bits again.
    compact_pixels: True (with lazy_full_res only) keeps each pixel row as the uint8 codes of FVS_PRE_QWEN_CODES, half
    the bytes of the tower dtype: step() then takes the codes [t * h * w, 1176] in place of the pixel rows, and
    `pixel_table` (the pre-processor's float32 [3, 256] device table) is what they decode through, on each re-encode,
    into the rows the tower would have read (DESIGN.md §3.20).  Same bits again."""

    CHUNK_BYTES = CHUNK_BYTES

    def __init__(self, flash, merger, device_frames=None, small_device_frames=None, lazy_full_res=False,
                 full_res_bank=True, compact_pixels=False):
        self.flash, self.merger = flash, merger
        self.device_frames = check_device_frames(device_frames)
        self.small_device_frames = check_device_frames(small_device_frames, "small_device_frames")
        self.lazy_full_res = check_lazy_full_res(lazy_full_res, flash)
        self.full_res_bank = check_full_res_bank(full_res_bank, self.lazy_full_res)
        self.compact_pixels = check_compact_pixels(compact_pixels, self.lazy_full_res)
        self.pixel_table = None               # compact_pixels: device float32 [3, 256], what the codes decode through
        self.rng = GLOBAL                     # the draws.DrawSource of every k-means draw (a QwenStreamPool stream owns one)
        self.reset()

    def reset(self):
        self.bank_x, self.bank_small, self.bank_merged = RowBank(), RowBank(), RowBank()
        self.bank_tier = HostChunks()         # frames >= device_frames: x rows and (a part of their own) merged rows
        self.small_tier = HostChunks()        # half-resolution frames >= small_device_frames
        self._prev_dam = None                 # (spa_positions, spa_x, DAM rows of video_embeds) before the current step
        self.host_fetches = None              # device int64 [1]: retrieved frames read from the host chunks so far
        self.n_frames = 0
        self.grid = None                      # (h, w) of a full-resolution frame; the half-resolution grid is (hs, ws)
        self.small_grid = None
        self.tem_x = self.tem_weights = self.tem_timestamp = None     # CSM: [n_tem * hs * ws, D], [n_tem], [n_tem]
        self.n_tem = 0
        self.spa_x = self.spa_positions = None                        # DAM: [n_spa, h * w, D], int64 [n_spa]
        self.video_embeds = None
        self.tem_members = None
        self._readback = None                 # pinned int32 [8]: n_unique, info[4], flags
        self._pending = None                  # what complete() needs of an enqueued clip ({} when nothing is read back)
        self.fast_steps = self.redone_steps = 0
        self.steps = 0                        # clips whose step completed (a clip that raises is not counted)
        self.encoded = RowBank()              # lazy_full_res: device uint8 [n_frames], 1 once a frame's bank slots are filled
        #                                       (no full_res_bank: 1 once encoded, 2 when its rows are in the base bank)
        self.pixels: Optional[PixelStore] = None   # lazy_full_res: the frames' full-resolution pixel rows
        self.n_encoded = 0                    # lazy_full_res: frames the full-resolution tower has encoded (no
        #                                       full_res_bank: every encode, re-encodes included)
        self.re_encodes = None                # no full_res_bank: device int64 [1], encodes of frames encoded before
        self._fresh = None                    # no full_res_bank: (plan, n, x rows, merged rows) of this step's encodes
        self.tower = None                     # lazy_full_res: callable(pixel rows, grids) -> full-resolution features
        self._in_round = False                # lazy_full_res: the outputs of this step wait for multistream.encode_picked
        self._lazy_ctx = None                 # lazy_full_res: the retrieval context those outputs are made from
        self._plan = None                     # lazy_full_res: device int64, the last pick plan

    # ------------------------------------------------------------------------------------------------ one clip
    def step(self, x_new: torch.Tensor, small_new: torch.Tensor, t: int, grid, small_grid, start_idx: int,
             draws: Optional[dict] = None, merged: Optional[torch.Tensor] = None, tower=None, pixel_table=None):
        """x_new [t * h * w, D] / small_new [t * hs * ws, D]: the tower's two-resolution features of the clip (device);
        grid = (h, w), small_grid = (hs, ws) host integers; merged: the PatchMerger rows of x_new, when the caller has
        merged them already (None: merged here).  Updates the state.  enqueue(), one host wait, complete().
        With lazy_full_res, x_new is the clip's full-resolution pixel rows [t * h * w, 1176] (device) and `tower`
        (callable(rows, grids)) encodes the frames the DAM picks for the first time: the one-stream round of
        multistream.encode_picked, still one host wait.  With compact_pixels, x_new is the clip's codes and
        `pixel_table` their value table (kept for later steps)."""
        if self.lazy_full_res:
            from .multistream import encode_picked
            if tower is not None:
                self.tower = tower
            if pixel_table is not None:
                self.pixel_table = pixel_table
            if self._readback is None:
                self._readback = torch.empty(8, dtype=torch.int32).pin_memory()
            self._in_round = True
            try:
                banks = self.enqueue(x_new, small_new, t, grid, small_grid, start_idx, draws, merged)
            finally:
                if self._lazy_ctx is not None:
                    encode_picked([self], self._readback.view(1, 8))
                self._in_round = False
            self.complete()
            return banks
        banks = self.enqueue(x_new, small_new, t, grid, small_grid, start_idx, draws, merged)
        if self._pending:
            done = torch.cuda.Event()
            done.record()
            done.synchronize()
        self.complete()
        return banks

    def enqueue(self, x_new: torch.Tensor, small_new: torch.Tensor, t: int, grid, small_grid, start_idx: int,
                draws: Optional[dict] = None, merged: Optional[torch.Tensor] = None):
        """The first half of step(): the clip's work up to and including the copy of its 32-byte read-back, enqueued on
        the current stream.  The caller waits until that copy has landed (an event recorded after it), then calls
        complete().  = enqueue_input(), then enqueue_csm() of its request alone (QwenStreamPool enqueues the inputs of
        many states and then one enqueue_csm() for all of them, before one wait)."""
        banks, req = self.enqueue_input(x_new, small_new, t, grid, small_grid, start_idx, draws, merged)
        if req is not None:
            if self._readback is None:
                self._readback = torch.empty(8, dtype=torch.int32).pin_memory()
            enqueue_csm([(self, req)], self._readback.view(1, 8))
        return banks

    def enqueue_input(self, x_new: torch.Tensor, small_new: torch.Tensor, t: int, grid, small_grid, start_idx: int,
                      draws: Optional[dict] = None, merged: Optional[torch.Tensor] = None):
        """The clip up to the CSM k-means: banks, candidates and the k-means draws, taken from this state's draw source
        in the order step() takes them.  -> ((bank, small_bank), req): req is None when the clip needs no fast-path
        k-means (memory still filling, or a branch the synchronous path runs, which is then already enqueued); otherwise
        the k-means to run (cand [T, P, D], cand_w, init, refill, order), which enqueue_csm() takes."""
        flash = self.flash
        dev, dt, D = small_new.device, small_new.dtype, small_new.shape[-1]
        h, w = grid
        hs, ws = small_grid
        if self.grid is None:
            self.grid, self.small_grid = (h, w), (hs, ws)
        assert self.grid == (h, w) and self.small_grid == (hs, ws), "Tensors are not equal"   # merge_thw of the reference (:551-555)
        T0, S0 = flash.temporal_length, flash.spatial_length
        # ---- banks (and, once per frame, the merged rows of the frame)
        self._prev_dam = self._dam()
        self._append_small(small_new.view(t, hs * ws, D), dev)
        small_bank = self.bank_small.rows() if self.bank_small.n else None
        if self.lazy_full_res:
            if self.compact_pixels and (x_new.dtype != torch.uint8 or self.pixel_table is None):
                raise ValueError(f"compact_pixels: the stream takes uint8 codes and their pixel_table (got {x_new.dtype} "
                                 f"rows, table {'set' if self.pixel_table is not None else 'missing'})")
            self._append_lazy(x_new.view(t, h * w, PATCH_DIM), dt, D, dev)
        else:
            if S0 > 0 and self.merger is not None:
                merged = (self.merger(x_new) if merged is None else merged).view(t, h * w // 4, -1)
            else:
                merged = None
            self._append_frames(x_new.view(t, h * w, D), merged, dev)
        bank = self.bank_x.rows() if self.bank_x.n else None
        self.n_frames += t
        # ---- CSM input: carried centroids followed by the clip's half-resolution frames
        T = self.n_tem + t
        P = hs * ws
        if self.n_tem:
            cand = torch.empty(T, P, D, dtype=dt, device=dev)
            cand[: self.n_tem].copy_(self.tem_x.view(self.n_tem, P, D))
            cand[self.n_tem:].copy_(small_new.view(t, P, D))
            cand_w = torch.empty(T, dtype=torch.float32, device=dev)
            cand_w[: self.n_tem].copy_(self.tem_weights)
            cand_w[self.n_tem:].fill_(1.0)
        else:
            cand = small_new.view(t, P, D)
            cand_w = torch.ones(T, dtype=torch.float32, device=dev)
        d = draws or {}
        fast = T > T0 > 0 and flash.temporal_method in _KMEANS_METHODS
        self._pending = {}
        if not fast:
            self._compress_sync(cand, cand_w, T, d, start_idx, t)
            return (bank, small_bank), None
        snap = None
        init = d.get("init_idx")
        if init is None:
            snap = self.rng.snapshot(dev)
            init_dev = self.rng.randperm(T, dev)[:T0].to(torch.int32)        # randperm(n_unique), assuming n_unique == T
        else:
            init_dev = to_device(np.asarray(init)[:T0], np.int32, dev)
        refill = d.get("refill_idx")
        if refill is None:
            refill_dev, _ = self.rng.refill_candidates(T, CF.MAX_ITER * T0, dev)
        else:
            refill = list(int(v) for v in refill)
            refill_dev = to_device(refill + [0] * (CF.MAX_ITER * T0 - len(refill)), np.int32, dev)
        order = d.get("ts_order")
        order_dev = None if order is None else to_device(order, np.int64, dev)
        req = dict(cand=cand, cand_w=cand_w, T=T, d=d, start_idx=start_idx, t=t, snap=snap, own_refills=refill is None,
                   init=init_dev, refill=refill_dev, order=order_dev)
        return (bank, small_bank), req

    def _set_pending(self, req: dict, readback: torch.Tensor):
        """what complete() needs of the enqueued fast-path clip; readback: the row it reads"""
        keep = ("cand", "cand_w", "T", "d", "start_idx", "t", "snap", "own_refills")
        self._pending = dict({k: req[k] for k in keep}, readback=readback)

    def complete(self):
        """The second half of step(), once the read-back of enqueue() has landed: a valid fast-path clip is final (or raises
        ZeroDivisionError on an empty cluster, as the reference does; the state is then left as that raise leaves it); a
        clip with duplicate rows rewinds this state's draw source and is redone through the synchronous path."""
        p, self._pending = self._pending, None
        if p:
            T0 = self.flash.temporal_length
            T = p["T"]
            n_unique, _, consumed, _, _, empty = (int(v) for v in p.get("readback", self._readback)[:6])
            valid = n_unique >= T0 and (p["snap"] is None or n_unique == T)
            if valid:
                if empty:
                    raise ZeroDivisionError("division by zero")          # sum(indices) / len(indices), compress_functions.py:279
                if p["own_refills"]:
                    self.rng.consume(T, consumed)                          # leave `random` where the reference would
                self.fast_steps += 1
            else:                                                          # duplicates among the rows: the general path
                if p["snap"] is not None:
                    self.rng.rewind(p["snap"])
                self.redone_steps += 1
                self._compress_sync(p["cand"], p["cand_w"], T, p["d"], p["start_idx"], p["t"])
        self._prev_dam = None                 # the old DAM is the readers' now, not ours to keep alive
        self.steps += 1

    # ------------------------------------------------------------------------------------------------ pieces
    def _thw(self, n, small=False):
        g = self.small_grid if small else self.grid
        return torch.tensor([n, g[0], g[1]])                    # host tensor: what the reference's list holds at rest

    def _rest_retrieval(self, tem_x, tem_w, tem_ts, n_tem, members, d):
        """the CSM fields, and the DAM picks or, for a klarge retrieval over a bank wholly in HBM (k <= 64), what it
        needs: ctx["retrieve"] = (centroids [st, PD], heaviest int64 [k], bank [n, PD], metric); picks are then set by
        _rest_stage"""
        flash = self.flash
        D = tem_x.shape[-1]
        n = self.n_frames
        dev = tem_x.device
        self.tem_x, self.tem_weights, self.tem_timestamp, self.n_tem, self.tem_members = tem_x, tem_w, tem_ts, n_tem, members
        ctx = dict(tem_x=tem_x, d=d, picks=None, retrieve=None)
        if flash.spatial_length <= 0:
            ctx["picks"], ctx["n_spa"] = torch.empty(0, dtype=torch.int64, device=dev), 0
            return ctx
        n_spa = min(n, flash.spatial_length)                            # known on the host
        ctx["n_spa"] = n_spa
        tem_pos = torch.round(tem_ts.float()).to(torch.int64)
        klarge = flash.spatial_method in ("klarge_retrieve", "klarge_retrieve_cos")
        if (klarge and n > flash.spatial_length and self.n_small_host == 0 and n_spa <= 64
                and (d or {}).get("weight_order") is None and self.small_tier.dtype in (torch.float16, torch.bfloat16)):
            heaviest = O.argsort_desc(tem_w)[:n_spa]                   # spatial_picks' ranking
            ctx["retrieve"] = (tem_x.reshape(n_tem, -1), heaviest, self.bank_small.rows().view(n, -1),
                               "cosine" if flash.spatial_method == "klarge_retrieve_cos" else "euclidean")
        else:
            ctx["picks"] = flash.spatial_picks(self._small_bank(D, dev), n, tem_x, self._thw(n_tem, small=True), tem_w,
                                               tem_pos, draws=d)
        return ctx

    def _rest_outputs(self, ctx):
        """the DAM and video_embeds tensors for the picks of ctx -> (keyword arguments of the dam_gather that fills them,
        or None; (CSM rows, the slice of video_embeds their merged rows go to), or None)"""
        h, w = self.grid
        tem_x, picks, n_spa = ctx["tem_x"], ctx["picks"], ctx["n_spa"]
        D = tem_x.shape[-1]
        dt, dev = self.small_tier.dtype, tem_x.device
        # memory still filling: the DAM is the whole bank, a view of it (a state without a bank gathers it)
        whole = n_spa == self.n_frames and self.n_host == 0 and self.full_res_bank
        spa_x = self.bank_x.rows() if whole else torch.empty(n_spa, h * w, D, dtype=dt, device=dev)
        self.spa_x, self.spa_positions = spa_x, picks
        pm = h * w // 4                                               # merged tokens of a retrieved frame
        out = None
        if self.merger is not None:
            out = torch.empty(n_spa * pm + tem_x.shape[0] // 4, self.merger.dim, dtype=tem_x.dtype, device=tem_x.device)
        # one launch writes the retrieved frames and their merged rows (fresh tensors: readers may hold the old ones)
        gather_x = n_spa > 0 and not whole
        gather_m = n_spa > 0 and out is not None
        gather = None
        if gather_x or gather_m:
            gather = self._gather_args(picks, spa_x if gather_x else None,
                                       out[: n_spa * pm].view(n_spa, pm, -1) if gather_m else None, self._prev_dam)
        merge = (tem_x, out[n_spa * pm:]) if out is not None and out.shape[0] > n_spa * pm else None
        self.video_embeds = out
        return gather, merge

    # ------------------------------------------------------------------------------------------------ two-tier bank
    def _dam(self):
        """the current DAM as a previous-step source for fvs_qwen_dam_gather_multi: (picks, spa_x, DAM rows of
        video_embeds)"""
        if self.spa_positions is None or self.spa_positions.numel() == 0 or not self.spa_x.is_cuda:
            return None
        m = self.spa_positions.numel()
        ve = self.video_embeds
        return self.spa_positions, self.spa_x, None if ve is None else ve[: m * self.spa_x.shape[1] // 4]

    @property
    def n_host(self) -> int:
        """frames of the full-resolution (and merged) bank in its host tier"""
        return self.bank_tier.n

    @property
    def n_small_host(self) -> int:
        """frames of the half-resolution bank in its host tier"""
        return self.small_tier.n

    @property
    def host_chunks(self) -> list:
        """the pinned chunks of the full-resolution (and merged) bank's host tier"""
        return self.bank_tier.chunks

    @property
    def small_chunks(self) -> list:
        """the pinned chunks of the half-resolution bank's host tier"""
        return self.small_tier.chunks

    def _banks(self):
        """the device tier of the full-resolution bank: one RowBank per part of bank_tier (x rows, merged rows)"""
        return [self.bank_x, self.bank_merged][:len(self.bank_tier.shapes)]

    def _append_frames(self, x3, m3, dev):
        """frames x3 [t, h*w, D] (merged rows m3 [t, h*w/4, merger_dim] or None), on the device or the host, appended to
        the two-tier bank, which keeps merged rows when its first frames came with them"""
        parts = [x3] if m3 is None else [x3, m3]
        if self.bank_tier.dtype is None:
            self.bank_tier.lay_out(x3.dtype, [r.shape[1:] for r in parts], self.CHUNK_BYTES)
        _append_tiered(self._banks(), self.bank_tier, self.device_frames, x3.shape[0], parts, dev)

    def _append_lazy(self, pix3, dt, D, dev):
        """lazy_full_res: the clip's pixel rows pix3 [t, h*w, 1176] appended to the pixel store (asynchronous copies to its
        pinned chunks), and t bank slots (zero rows in HBM, chunk rows on the host; none without full_res_bank) with clear
        mask bytes"""
        t, hw = pix3.shape[0], pix3.shape[1]
        if self.bank_tier.dtype is None:
            merged = self.flash.spatial_length > 0 and self.merger is not None
            self.bank_tier.lay_out(dt, [(hw, D)] + ([(hw // 4, int(self.merger.dim))] if merged else []), self.CHUNK_BYTES)
        if self.pixels is None:
            self.pixels = self._pixel_store(hw, self.n_frames, pix3.dtype)
        self.pixels.append(pix3.reshape(t, -1), dev)
        if self.full_res_bank:
            _append_tiered(self._banks(), self.bank_tier, self.device_frames, t, None, dev)
        self.encoded.append(torch.zeros(t, dtype=torch.uint8, device=dev))

    def _pixel_store(self, hw: int, base: int, dtype) -> "PixelStore":
        """an empty pixel store from frame `base` on: uint8 codes with their table that decode to the bank dtype
        (compact_pixels), or rows of `dtype`"""
        if self.compact_pixels:
            return PixelStore(torch.uint8, hw * PATCH_DIM, base, self.CHUNK_BYTES, values=self.pixel_table,
                              out_dtype=self.bank_tier.dtype)
        return PixelStore(dtype, hw * PATCH_DIM, base, self.CHUNK_BYTES)

    def _bank_args(self, dev) -> dict:
        """this state's two-tier bank as the gather and scatter jobs on `dev` read it; n_base: its frames (without
        full_res_bank, those of the base bank, which may be fewer than the stream's)"""
        tier = self.bank_tier
        return dict(n_base=self.bank_x.n + tier.n, dev_x=self.bank_x.buf if self.bank_x.n else None,
                    dev_merged=self.bank_merged.buf if self.bank_merged.n else None, n_dev=self.bank_x.n,
                    chunks=tier.table(dev), chunk_frames=tier.per_chunk, x_frame_elems=tier.shapes[0].numel(),
                    merged_frame_elems=tier.shapes[1].numel() if len(tier.shapes) > 1 else 0)

    def _scatter_args(self, n: int, x_rows, merged_rows) -> dict:
        """the job of Q.bank_scatter_multi that writes the n frames of this state's last pick plan into its banks"""
        bank = self._bank_args(self._plan.device)
        return dict(bank, plan=self._plan, n=n, n_frames=bank["n_base"], x_rows=x_rows,
                    merged_rows=merged_rows if bank["merged_frame_elems"] else None)

    def _append_small(self, s3, dev):
        """half-resolution frames s3 [t, hs*ws, D], on the device or the host, appended to the two-tier half-resolution
        bank"""
        if self.small_tier.dtype is None:
            self.small_tier.lay_out(s3.dtype, [s3.shape[1:]], self.CHUNK_BYTES)
        _append_tiered([self.bank_small], self.small_tier, self.small_device_frames, s3.shape[0], [s3], dev)

    def _small_bank(self, D, dev):
        """the half-resolution bank as the retrieval reads it: the HBM rows [n * hs*ws, D] while every frame is there, a
        qwen.ops.TieredBank once frames have spilled"""
        rb, tier = self.bank_small, self.small_tier
        if tier.n == 0:
            return rb.rows().view(-1, D)
        return Q.TieredBank(rb.rows().view(rb.n, -1) if rb.n else None, rb.n, tier.ptrs(), tier.per_chunk, rb.n + tier.n,
                            tier.dtype, dev)

    def _gather_args(self, picks, spa_x, merged, prev) -> dict:
        """the Q.dam_gather_multi job that writes spa_x / merged for `picks` from the previous DAM `prev`, this step's
        fresh rows (without full_res_bank) and this state's bank"""
        if self.host_fetches is None:
            self.host_fetches = torch.zeros(1, dtype=torch.int64, device=picks.device)
        return dict(self._bank_args(picks.device), picks=picks, n_frames=self.n_frames, prev=prev, fresh=self._fresh,
                    spa_x_out=spa_x, merged_out=merged, host_fetches=self.host_fetches)

    def host_fetch_count(self) -> int:
        """retrieved frames read from the host chunks since the stream started here (synchronises; tests and timing)"""
        return 0 if self.host_fetches is None else int(self.host_fetches.item())

    def re_encode_count(self) -> int:
        """without full_res_bank: full-resolution encodes of frames the tower had encoded before, since the stream
        started here (a clip redone by complete() counts its encodes again; synchronises; tests and timing)"""
        return 0 if self.re_encodes is None else int(self.re_encodes.item())

    def pinned_bytes(self) -> int:
        """bytes of pinned host memory the state holds: bank chunks, half-resolution chunks and pixel chunks"""
        return self.bank_tier.nbytes() + self.small_tier.nbytes() + (0 if self.pixels is None else self.pixels.tier.nbytes())

    def _compress_sync(self, cand, cand_w, T, d, start_idx, t):
        """every other branch of temporal_compress (:149-183): pass-through while the memory is filling, temporal_length 0,
        alternate methods, and the duplicate-rows replay — through the mirror's own (synchronous) method"""
        flash = self.flash
        P, D = cand.shape[1], cand.shape[2]
        ts_in = torch.arange(T, device=cand.device, dtype=torch.float32)      # accepted and ignored by the reference (:279)
        tem_x, tem_thw, tem_w, tem_ts, members = flash.temporal_compress(
            cand.reshape(T * P, D), self._thw(T, small=True), flash.temporal_length, cand_w, ts_in, draws={**d, "source": self.rng})
        _rest_stage([(self, self._rest_retrieval(tem_x, tem_w, tem_ts, int(tem_thw[0]), members, d))])

    # ------------------------------------------------------------------------------------------------ checkpoint / restore
    # What a step reads: the three banks, the CSM (tem_x, weights; n_tem), n_frames and the grids; what as_list() and a
    # publication read besides: timestamps, spa_positions, spa_x and video_embeds.  spa_x is bank_x[spa_positions], so it
    # is rebuilt by a bit-exact gather; the member lists are read by no step (only by spatial_enhance of the step that
    # made them), so a restored state has none, like a reset one.
    def _config(self, dim, dtype):
        cfg = {"flash": dict(self.flash.config), "grid": None if self.grid is None else list(self.grid),
               "small_grid": None if self.small_grid is None else list(self.small_grid), "dtype": dtype, "dim": dim,
               "merger_dim": None if self.merger is None else int(self.merger.dim)}
        if self.compact_pixels:
            cfg["compact_pixels"] = True
        return cfg

    def checkpoint(self):
        """The state as a checkpoint.StreamCheckpoint in pinned host memory (filled rows only; returns once the copies
        have landed).  Call it between steps, from the writer."""
        from .. import checkpoint as CK
        n = self.n_frames
        counters = {"n_frames": n, "steps": self.steps, "n_tem": self.n_tem,
                    "n_spa": 0 if self.spa_positions is None else int(self.spa_positions.numel()),
                    "fast_steps": self.fast_steps, "redone_steps": self.redone_steps,
                    "merged": int(n > 0 and len(self.bank_tier.shapes) > 1),
                    "tem_weights_dtype": None if self.tem_weights is None else CK.dtype_name(self.tem_weights.dtype),
                    "tem_timestamp_dtype": "float32" if n == 0 else CK.dtype_name(self.tem_timestamp.dtype)}
        if self.lazy_full_res and n:          # eager checkpoints carry neither the counter nor the tensors below
            stored = 2 if not self.full_res_bank else 1           # the mask byte of a frame whose rows are stored
            todo = torch.nonzero(self.encoded.rows().cpu() != stored).flatten().tolist()   # frames with pixel rows only
            counters["pix_frames"] = len(todo)
            if not self.full_res_bank:        # the stored (base) bank's frames; the DAM's rows travel as spa_x
                counters["bank_frames"] = self.bank_x.n + self.n_host
        if n == 0:
            return CK.qwen(self._config(0, "float16"), counters, {})
        tensors = {"tem_x": self.tem_x, "tem_timestamp": self.tem_timestamp, "spa_positions": self.spa_positions}
        if self.tem_weights is not None:          # temporal_method 'sample' keeps no weights
            tensors["tem_weights"] = self.tem_weights
        if self.merger is not None:
            tensors["video_embeds"] = self.video_embeds
        with torch.cuda.device(self.tem_x.device):
            owned = {}                            # spilled banks: assembled in pinned memory here, taken as they are
            if self.lazy_full_res:                # the mask, and the pixel rows of the frames not yet encoded, in order
                tensors["encoded"] = self.encoded.rows()
                if self.compact_pixels:           # as codes, with the table they decode through
                    owned["pix_codes"] = self.pixels.rows_of(todo)
                    tensors["pixel_table"] = self.pixels.values
                else:
                    owned["pixels"] = self.pixels.rows_of(todo).view(len(todo), self.bank_tier.shapes[0][0], PATCH_DIM)
            if not self.full_res_bank:
                tensors["spa_x"] = self.spa_x
            if self.n_small_host:
                owned["bank_small"] = self.small_tier.to_host(self.bank_small.rows() if self.bank_small.n else None)
            else:
                tensors["bank_small"] = self.bank_small.rows()
            tier = self.bank_tier
            for part, (name, rb) in enumerate((("bank_x", self.bank_x), ("bank_merged", self.bank_merged))):
                if part and not counters["merged"]:
                    continue
                if tier.n:
                    owned[name] = tier.to_host(rb.rows() if rb.n else None, part)
                elif rb.n:
                    tensors[name] = rb.rows()
                else:                             # no full_res_bank and no base bank: zero frames
                    tensors[name] = torch.empty((0,) + tuple(tier.shapes[part]), dtype=tier.dtype)
            small = self.small_tier
            ck = CK.qwen(self._config(int(small.shapes[0][-1]), CK.dtype_name(small.dtype)), counters, tensors, owned=owned)
            torch.cuda.current_stream().synchronize()
        return ck

    @classmethod
    def restore(cls, ckpt, flash, merger, device, device_frames=None, small_device_frames=None,
                lazy_full_res=False, full_res_bank=True, compact_pixels=False, pixel_table=None) -> "QwenStreamState":
        """A state on `device` that continues `ckpt` bit for bit; `flash` / `merger` must have the configuration the
        checkpoint was taken with (ValueError naming the field otherwise).  The banks' frames are placed by this state's
        `device_frames` and `small_device_frames`, whatever the caps of the state that took the checkpoint.  An eager
        checkpoint (every frame encoded) restores into a lazy_full_res state; a lazy one restores into an eager state
        only once every frame is encoded (NotImplementedError naming the knob otherwise).  Into a state without
        full_res_bank, an eager or lazy checkpoint's stored rows become a frozen base bank (placed by `device_frames`)
        and later frames keep pixel rows only; a checkpoint of such a state restores into a lazy_full_res state (its
        frames without stored rows "not yet encoded"), and into an eager one only when it has no such frame.
        A compact_pixels checkpoint (codes and their table) restores into a compact_pixels state whose `pixel_table`
        (None: the checkpoint's) equals its table (ValueError naming pixel_table otherwise), and into a lazy_full_res
        state without compact_pixels with its codes decoded, bit for bit.  A lazy_full_res checkpoint without codes
        does not restore into a compact_pixels state (NotImplementedError naming compact_pixels): its rows need not
        be codes of any table."""
        from .. import checkpoint as CK
        if ckpt.family != CK.QWEN:
            raise ValueError(f"QwenStreamState.restore: a {ckpt.family!r} checkpoint is not a Qwen2-VL stream's")
        c, n = ckpt.config, ckpt.counters
        if c["flash"] != dict(flash.config):
            bad = next(k for k in set(c["flash"]) | set(flash.config) if c["flash"].get(k) != flash.config.get(k))
            raise ValueError(f"QwenStreamState.restore: config.flash.{bad} of the checkpoint ({c['flash'].get(bad)}) "
                             f"differs from the FlashMemory's ({flash.config.get(bad)})")
        md = None if merger is None else int(merger.dim)
        if n["n_frames"] and c["merger_dim"] != md:
            raise ValueError(f"QwenStreamState.restore: config.merger_dim of the checkpoint ({c['merger_dim']}) differs "
                             f"from the merger's ({md})")
        st = cls(flash, merger, device_frames, small_device_frames, lazy_full_res=lazy_full_res,
                 full_res_bank=full_res_bank, compact_pixels=compact_pixels)
        compact_ck = bool(c.get("compact_pixels")) and "pix_frames" in n
        if compact_pixels and "pix_frames" in n and not compact_ck:
            raise NotImplementedError("QwenStreamState.restore: the checkpoint keeps its pixel rows in the tower dtype, "
                                      "which need not be codes of any table: restore it with compact_pixels=False")
        if compact_pixels and compact_ck and pixel_table is not None and not torch.equal(
                ckpt.tensor("pixel_table"), pixel_table.detach().cpu().float()):
            raise ValueError("QwenStreamState.restore: the checkpoint's pixel_table differs from the stream's: its codes "
                             "would decode to other rows")
        if compact_pixels:
            st.pixel_table = pixel_table if pixel_table is not None or not compact_ck else ckpt.tensor("pixel_table")
            if st.pixel_table is None and n["n_frames"] and lazy_full_res:
                raise ValueError("QwenStreamState.restore: compact_pixels=True needs pixel_table=, the table the "
                                 "stream's codes decode through")
            if st.pixel_table is not None:
                st.pixel_table = st.pixel_table.to(device).float().contiguous()
        if n["n_frames"] == 0:
            return st
        N = n["n_frames"]
        lazy_ck, bankless_ck = "pix_frames" in n, "bank_frames" in n
        stored = torch.ones(N, dtype=torch.bool)  # frames whose rows the checkpoint's bank holds (an eager one: all)
        todo = []
        if lazy_ck:                               # the frames with pixel rows only, which the checkpoint holds
            enc = ckpt.tensor("encoded")
            stored = enc == (2 if bankless_ck else 1)
            if bankless_ck and bool(stored[n["bank_frames"]:].any()):
                raise ValueError(f"QwenStreamState.restore: the mask marks frames past counters.bank_frames "
                                 f"({n['bank_frames']}) as stored")
            todo = torch.nonzero(~stored).flatten().tolist()
            if len(todo) != n["pix_frames"]:
                raise ValueError(f"QwenStreamState.restore: counters.pix_frames ({n['pix_frames']}) is not the number of "
                                 f"frames the mask leaves unencoded ({len(todo)})")
        if todo and not lazy_full_res:
            if bankless_ck:
                raise NotImplementedError("QwenStreamState.restore: the checkpoint is of a stream without a "
                                          "full-resolution bank (full_res_bank=False): restore it with lazy_full_res=True")
            raise NotImplementedError("QwenStreamState.restore: the checkpoint is of a lazy_full_res stream with frames "
                                      "not yet encoded at full resolution: restore it with lazy_full_res=True")
        dev = torch.device(device)
        with torch.cuda.device(dev):
            get = lambda k: ckpt.tensor(k).to(dev, non_blocking=True)
            st._append_frames(ckpt.tensor("bank_x"), ckpt.tensor("bank_merged") if n["merged"] else None, dev)
            st._append_small(ckpt.tensor("bank_small"), dev)
            if lazy_full_res:
                hw = int(c["grid"][0]) * int(c["grid"][1])
                # the pixel store starts at the first frame with pixel rows only; frames without a stored row get them
                base = todo[0] if todo else N
                st.pixels = st._pixel_store(hw, base, st.bank_tier.dtype)
                if todo:
                    st.pixels.append(None, dev, t=N - base)
                    if compact_ck and not compact_pixels:     # decoded here into the rows the tower reads
                        rows = Q.pixel_decode(get("pix_codes").view(-1, PATCH_DIM), get("pixel_table"), st.bank_tier.dtype)
                        st.pixels.put(todo, rows.view(len(todo), -1).cpu())
                    else:
                        st.pixels.put(todo, ckpt.tensor("pix_codes" if compact_ck else "pixels").view(len(todo), -1))
                st.n_encoded = N - len(todo)
                if full_res_bank:                 # frames past the checkpoint's bank get zero slots, "not yet encoded"
                    _append_tiered(st._banks(), st.bank_tier, st.device_frames, N - (st.bank_x.n + st.n_host), None, dev)
                    st.encoded.append(stored.to(torch.uint8).to(dev))
                elif bankless_ck:                 # the base bank and the "encoded before" bytes carry over as they are
                    st.encoded.append(get("encoded"))
                else:                             # the checkpoint's stored rows become the frozen base bank
                    st.encoded.append((stored.to(torch.uint8) * 2).to(dev))
            st.n_frames, st.steps = n["n_frames"], n["steps"]
            st.fast_steps, st.redone_steps = n["fast_steps"], n["redone_steps"]
            st.grid, st.small_grid = tuple(c["grid"]), tuple(c["small_grid"])
            st.tem_x, st.tem_timestamp = get("tem_x"), get("tem_timestamp")
            st.tem_weights = get("tem_weights") if "tem_weights" in ckpt.tensors else None
            st.n_tem = n["n_tem"]
            st.spa_positions = get("spa_positions")
            h, w = st.grid
            if "spa_x" in ckpt.tensors:           # a stream without a bank: the DAM's rows as they were
                st.spa_x = get("spa_x")
            else:
                st.spa_x = torch.empty(n["n_spa"], h * w, int(c["dim"]), dtype=st.bank_tier.dtype, device=dev)
                if n["n_spa"]:
                    Q.dam_gather_multi([st._gather_args(st.spa_positions, st.spa_x, None, None)])
            st.video_embeds = get("video_embeds") if "video_embeds" in ckpt.tensors else None
            torch.cuda.current_stream().synchronize()     # the pinned sources may be freed as soon as this returns
        return st

    # ------------------------------------------------------------------------------------------------ the reference's list
    def as_list(self):
        """the 13 items of `video_embedding_memory` (:620-624); the thw entries are host tensors, everything else lives in HBM.
        Once frames have spilled to the host chunks, or with lazy_full_res, item 7 (the full-resolution bank, which no
        reader of the list uses) is the zero-row stand-in x[:0]; its thw (item 8) stays exact.  Likewise item 9 (the half-resolution bank) once its
        frames have spilled; item 10 stays exact."""
        n, h, w = self.n_frames, *self.grid
        n_spa = 0 if self.spa_positions is None else int(self.spa_positions.numel())
        ve = self.video_embeds
        D = self.tem_x.shape[-1]
        # the stand-ins are zero-row device views of the banks' dtype (tem_x's when no half-resolution frame is in HBM)
        rows = self.bank_small.rows().view(-1, D) if self.bank_small.n else self.tem_x.reshape(-1, D)
        small = rows if self.n_small_host == 0 else rows[:0]
        x = self.bank_x.rows().view(n * h * w, -1) if self.n_host == 0 and not self.lazy_full_res else rows[:0]
        return [self.tem_x, self._thw(self.n_tem, small=True), self.tem_weights, self.tem_timestamp,
                self.spa_x, self._thw(n_spa), self.spa_positions,
                x, self._thw(n), small, self._thw(n, small=True), ve, None if ve is None else ve.shape]


def enqueue_csm(items, readbacks: torch.Tensor):
    """The CSM half of the memory step of every (state, req) in `items`, req as QwenStreamState.enqueue_input returns
    it, enqueued on the current stream: the ordered k-means as one job table per kernel, the DAM retrieval and the merged
    memory (_rest_stage), then ONE copy of every read-back into rows [0, n) of `readbacks` (pinned int32 [>= n, 8]); the
    complete() of items[i] reads row i.  The states share one FlashMemory config and one merger.  A stream stepped alone
    is the one-item call (DESIGN.md §3.17)."""
    T0 = items[0][0].flash.temporal_length
    kms, rb = CF.ordered_kmeans_enqueue_multi([(r["cand"], r["cand_w"], r["init"], r["refill"], r["order"])
                                               for _, r in items], T0)
    ctxs = []
    for i, ((state, req), km) in enumerate(zip(items, kms)):
        P, D = req["cand"].shape[1], req["cand"].shape[2]
        ctxs.append((state, state._rest_retrieval(km["feat"].view(T0 * P, D), km["weights"], km["timestamps"], T0,
                                                  km["members"], req["d"])))
        state._set_pending(req, readbacks[i])
    _rest_stage(ctxs)
    readbacks[: len(items)].copy_(rb, non_blocking=True)


def _rest_stage(ctxs):
    """DAM retrieval and merged memory of every (state, ctx of its _rest_retrieval) in `ctxs`, for CSMs already (being)
    computed; no host round trip for the default spatial methods.  One klarge retrieval table per (metric, dtype) for
    the contexts that ask for one (a bank with host rows has retrieved on its own), _rest_outputs, one DAM gather table
    per dtype, and one PatchMerger call over every CSM slice: the merger is row-wise (§3.5), so each row gets its bits."""
    groups = {}
    for _, c in ctxs:
        if c["retrieve"] is not None:
            groups.setdefault((c["retrieve"][3], c["retrieve"][2].dtype), []).append(c)
    for (metric, _), cs in groups.items():
        for c, picks in zip(cs, Q.klarge_retrieve_multi([c["retrieve"][:3] for c in cs], metric)):
            c["picks"] = picks
    lazy = []                        # lazy_full_res: the outputs wait until the picked frames are encoded
    for state, c in ctxs:
        if state.lazy_full_res:
            state._lazy_ctx = c
            if not state._in_round:   # a clip redone by complete(), outside its round: encoded here, synchronously
                lazy.append(state)
    if lazy:
        from .multistream import encode_picked
        for state in lazy:
            if state._readback is None:
                state._readback = torch.empty(8, dtype=torch.int32).pin_memory()
            encode_picked([state], state._readback.view(1, 8))
    _rest_finish([(s, c) for s, c in ctxs if not s.lazy_full_res])


def _rest_finish(ctxs):
    """the second half of _rest_stage, once the retrieved frames are in the banks (or, without full_res_bank, in the
    fresh rows): _rest_outputs, one DAM gather table per dtype, and one PatchMerger call over every CSM slice"""
    if not ctxs:
        return
    gathers, merges = {}, []
    for state, c in ctxs:
        g, m = state._rest_outputs(c)
        if g is not None:
            out = g["spa_x_out"] if g["spa_x_out"] is not None else g["merged_out"]
            gathers.setdefault(out.dtype, []).append(g)
        if m is not None:
            merges.append(m)
    for calls in gathers.values():
        Q.dam_gather_multi(calls)
    merger = ctxs[0][0].merger
    if len(merges) == 1:
        merger(merges[0][0], out=merges[0][1])
    elif merges:
        y = merger(torch.cat([x for x, _ in merges]))
        r = 0
        for x, out in merges:
            out.copy_(y[r: r + out.shape[0]])
            r += out.shape[0]


def check_lazy_full_res(v, flash, who: str = "lazy_full_res") -> bool:
    """a bool; NotImplementedError when on with a temporal pool size other than 2 (with pool size 1 the half-resolution
    bank is the full-resolution one, so there is nothing to defer)"""
    if not isinstance(v, bool):
        raise ValueError(f"{who} must be True or False, got {v!r}")
    if v and flash.temporal_poolsize != 2:
        raise NotImplementedError(f"{who}=True needs flash_memory_temporal_poolsize=2 (got {flash.temporal_poolsize}): "
                                  f"with pool size 1 the full-resolution bank is the half-resolution one")
    return v


def check_compact_pixels(v, lazy: bool, who: str = "compact_pixels", lazy_who: str = "lazy_full_res") -> bool:
    """a bool; True needs lazy_full_res (ValueError otherwise: only a lazy_full_res stream keeps pixel rows)"""
    if not isinstance(v, bool):
        raise ValueError(f"{who} must be True or False, got {v!r}")
    if v and not lazy:
        raise ValueError(f"{who}=True needs {lazy_who}=True: the codes stand in for the pixel rows only a "
                         f"lazy_full_res stream keeps")
    return v


def check_full_res_bank(v, lazy: bool, who: str = "full_res_bank", lazy_who: str = "lazy_full_res") -> bool:
    """a bool; False needs lazy_full_res (ValueError otherwise: an eager stream's bank is where its features go)"""
    if not isinstance(v, bool):
        raise ValueError(f"{who} must be True or False, got {v!r}")
    if not v and not lazy:
        raise ValueError(f"{who}=False needs {lazy_who}=True: a stream without a full-resolution bank re-encodes its "
                         f"frames from their pixel rows, which only a lazy_full_res stream keeps")
    return v


class PixelStore:
    """lazy_full_res: the full-resolution pixel rows of frames [base, n) of a stream in pinned host chunks of
    chunk_frames frames each (`tier`, a HostChunks with no device tier: frame f is its frame f - base), with a device
    table of the chunks' mapped pointers that fvs_qwen_pixel_gather_multi reads them through.  Frames below `base`
    (encoded before the stream came here from a checkpoint) have no pixel rows; a restored stream's encoded frames above
    it have unwritten slots.  dtype: the rows' element type, the tower dtype or uint8 codes (compact_pixels); a store of
    codes holds `values`, the float32 [3, 256] device table the gather decodes them through into `out_dtype`."""

    def __init__(self, dtype, frame_elems: int, base: int, chunk_bytes: int = CHUNK_BYTES, values=None, out_dtype=None):
        self.dtype, self.frame_elems, self.base = dtype, int(frame_elems), int(base)
        if (dtype == torch.uint8) != (values is not None and out_dtype is not None):
            raise ValueError("PixelStore: uint8 codes go with their value table and the dtype they decode to")
        self.values, self.out_dtype = values, dtype if out_dtype is None else out_dtype
        self.tier = HostChunks().lay_out(dtype, [(self.frame_elems,)], chunk_bytes)
        self.table = None

    chunk_frames = property(lambda self: self.tier.per_chunk)
    chunks = property(lambda self: self.tier.chunks)
    n = property(lambda self: self.base + self.tier.n)

    def append(self, rows: Optional[torch.Tensor], dev, t: Optional[int] = None):
        """rows [t, frame_elems] (device or host): asynchronous copies on the current stream; rows None: t slots left
        unwritten (frames whose rows are put() later or never read)"""
        self.tier.write(self.tier.n, None if rows is None else [rows], t)
        self.table = self.tier.table(dev)

    def _row(self, f: int) -> torch.Tensor:
        c, r = divmod(f - self.base, self.chunk_frames)
        return self.tier.view(c)[r]

    def rows_of(self, frames) -> torch.Tensor:
        """the rows of `frames` (each in [base, n)) as one pinned tensor [len(frames), frame_elems], once the pending
        copies have landed"""
        out = torch.empty(len(frames), self.frame_elems, dtype=self.dtype, pin_memory=True)
        torch.cuda.current_stream().synchronize()
        for i, f in enumerate(frames):
            out[i].copy_(self._row(int(f)))
        return out

    def put(self, frames, rows: torch.Tensor):
        """rows [len(frames), frame_elems] (host, the store's dtype) into the slots of `frames`"""
        if rows.dtype != self.dtype:
            raise ValueError(f"PixelStore.put: {rows.dtype} rows into a store of {self.dtype}")
        for i, f in enumerate(frames):
            self._row(int(f)).copy_(rows[i])


def _append_tiered(banks, tier: HostChunks, cap: Optional[int], t: int, parts, dev):
    """t frames appended to a two-tier bank: to `banks` (its device tier, one RowBank per part of `tier`) while fewer
    than `cap` frames (None: no cap) are there, then to `tier`.  parts: the frames' rows per part [t, ...], on the device
    or the host, or None for t zero slots (zero rows in HBM, unwritten host rows).  Copies are asynchronous on the
    current stream, ordered before any later kernel that reads them."""
    n0 = banks[0].n + tier.n
    k = t if cap is None else max(0, min(t, cap - n0))
    if k:
        for p, rb in enumerate(banks):
            rb.append(torch.zeros((k,) + tier.shapes[p], dtype=tier.dtype, device=dev) if parts is None
                      else parts[p][:k].to(dev, non_blocking=True))
    if k < t:
        tier.write(tier.n, None if parts is None else [r[k:] for r in parts], t - k)
