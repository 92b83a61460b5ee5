"""The memory-manager side of the Qwen2-VL realtime serve loop, and readers of its memory that need no Manager server.

Reference topology (Flash-VStream-Qwen/cli_server_2gpu.py:197-402): the main process builds the model and hangs a
`Manager().list()` on `model.video_embedding_memory`; `frame_memory_manager(model, ...)` runs in a spawned process that calls
`torch.cuda.set_device(1); model = model.cuda()` and `embed_new_video_clip` per clip, which pickles all 13 items of the
memory through the Manager server; the LLM on cuda:0 reads them back with `get_video_embedding_memory_cuda_list()` /
`prepare_realtime_inference` (vstream_qwen2vl_realtime.py:531-540, 632-640).  That topology works unchanged here: a Manager
list receives host copies, like the reference's (see RealtimeStreamingMixin._publish).

What the LLM needs is `video_embeds` plus the CSM timestamps and DAM positions that AM-RoPE needs.  A *publication* holds
just those in one device allocation that the writer updates with one launch per clip under a sequence counter
(fvs_qwen_publish, include/fvs_b200.h), and a reader copies them out consistently on its own device (fvs_qwen_snapshot):
  * same process (reader thread):          QwenMemoryReader(*export_qwen_memory(host)).read()
  * other process, same or other GPU:      ship `export_qwen_memory(host)` ONCE through a torch.multiprocessing queue (a CUDA
                                           IPC handle; peer access for another GPU), then QwenMemoryReader(...).read() per query.
Publication is opt-in: a host that was never exported runs exactly the launches it ran before."""
from __future__ import annotations

import ctypes as C
import time
from typing import Optional

import torch

from .. import _lib as L
from ..ops import _chk_cuda
from ..serve import MetricMeter, serve_pool

HEADER_FIELDS = ("seq", "epoch", "clips", "n_frames", "n_tem", "n_spa", "rows", "grid")
STATUS_FIELDS = ("seq0", "seq1") + HEADER_FIELDS[1:]


def pub_layout(tem_len: int, spa_len: int, grid, small_grid, dim: int) -> dict:
    """fvs_qwen_pub_layout: {rows_cap, ts_off, pos_off, emb_off, bytes} of the publication of a FlashMemory with
    temporal_length / spatial_length frames over full-resolution `grid` = (h, w) and CSM `small_grid` = (hs, ws)."""
    out = (C.c_int64 * 5)()
    L.check(L.load().fvs_qwen_pub_layout(int(tem_len), int(spa_len), *map(int, grid), *map(int, small_grid), int(dim), out),
            "fvs_qwen_pub_layout")
    return dict(zip(("rows_cap", "ts_off", "pos_off", "emb_off", "bytes"), (int(v) for v in out)))


def pack_grid(grid, small_grid) -> int:
    (h, w), (hs, ws) = grid, small_grid
    return int(h) | int(w) << 16 | int(hs) << 32 | int(ws) << 48


def unpack_grid(v: int):
    """-> ((h, w), (hs, ws)); all zero before the first publish"""
    v = int(v) & (2 ** 64 - 1)
    return (v & 0xFFFF, (v >> 16) & 0xFFFF), ((v >> 32) & 0xFFFF, (v >> 48) & 0xFFFF)


def decode_status(words) -> dict:
    """the 9 words a snapshot writes {seq0, seq1, epoch, clips, n_frames, n_tem, n_spa, rows, grid} -> a dict; `valid` is
    the seqlock's acceptance test (both sequence numbers equal and even)"""
    d = dict(zip(STATUS_FIELDS, (int(v) for v in words)))
    d["grid"], d["small_grid"] = unpack_grid(d["grid"])
    d["valid"] = d["seq0"] == d["seq1"] and d["seq0"] % 2 == 0
    return d


class QwenPublication:
    """The device allocation a host publishes its memory into (owned by the host, not by a QwenStreamState: it outlives a
    stream restart, which bumps `epoch` and never resets the sequence number)."""

    def __init__(self, tem_len: int, spa_len: int, grid, small_grid, dim: int, dtype: torch.dtype, device):
        self.tem_len, self.spa_len, self.dim, self.dtype = int(tem_len), int(spa_len), int(dim), dtype
        self.grid, self.small_grid = tuple(grid), tuple(small_grid)
        self.layout = pub_layout(tem_len, spa_len, grid, small_grid, dim)
        self.device = torch.device(device)
        self.buf = torch.zeros(self.layout["bytes"], dtype=torch.uint8, device=self.device)   # header zero: seq 0, clips 0
        self.epoch = 0

    def export(self):
        """(buf, tem_len, spa_len, rows_cap, dim, dtype): what QwenMemoryReader takes; `buf` is an ordinary CUDA tensor,
        so a torch.multiprocessing queue ships it as a CUDA IPC handle (send it once)"""
        return self.buf, self.tem_len, self.spa_len, self.layout["rows_cap"], self.dim, self.dtype

    def new_stream(self):
        self.epoch += 1

    def publish(self, state):
        """one launch on the current stream: the state's video_embeds, tem_timestamp and spa_positions, under the seqlock"""
        if state.grid != self.grid or state.small_grid != self.small_grid:
            raise ValueError(f"the stream's grid {state.grid} / {state.small_grid} is not the exported one "
                             f"{self.grid} / {self.small_grid}")
        ve = state.video_embeds
        assert ve.dtype == self.dtype and ve.shape[1] == self.dim and ve.is_contiguous()
        ts = state.tem_timestamp
        ts = ts if ts.dtype == torch.float32 and ts.is_contiguous() else ts.float().contiguous()
        pos = state.spa_positions.contiguous()
        n_tem, n_spa = int(ts.numel()), int(pos.numel())
        _chk_cuda(ve, ts, pos)
        with torch.cuda.device(self.device):
            L.check(L.load().fvs_qwen_publish(
                L.ptr(self.buf), self.buf.numel(), self.tem_len, self.spa_len, self.layout["rows_cap"], self.dim, L.ptr(ve),
                ve.shape[0], L.ptr(ts), n_tem, L.ptr(pos), n_spa, *self.grid, *self.small_grid, self.epoch, state.steps,
                state.n_frames, L.cur_stream()), "fvs_qwen_publish")


def export_qwen_memory(host, grid=None):
    """Create (once) `host`'s publication and return what a reader needs: (buf, tem_len, spa_len, rows_cap, dim, dtype).
    Before the first clip the grid is not known yet: pass grid=(h, w) (the half-resolution CSM grid follows from
    temporal_poolsize).  Until the first publish a reader gets an empty memory (clips == 0).  From then on every clip
    publishes once it is final; a clip that raises publishes nothing."""
    visual = host.visual
    merger, flash = visual.merger, visual.flash_memory
    if merger is None:
        raise NotImplementedError("a host without a PatchMerger has no video_embeds to publish")
    pub = host.__dict__.get("_qwen_publication")
    state = host.__dict__.get("stream_state")
    started = state is not None and state.grid is not None
    if grid is not None:
        g = tuple(int(v) for v in grid)
        sg = (g[0] // 2, g[1] // 2) if flash.temporal_poolsize > 1 else g
        if started and (state.grid, state.small_grid) != (g, sg):
            raise ValueError(f"grid {g} differs from the stream's grid {state.grid}")
    elif started:
        g, sg = state.grid, state.small_grid
    elif pub is None:
        raise ValueError("export_qwen_memory before the first clip needs grid=(h, w)")
    if pub is not None:
        if grid is not None and (pub.grid, pub.small_grid) != (g, sg):
            raise ValueError(f"grid {g} differs from the exported grid {pub.grid}")
        return pub.export()
    pub = QwenPublication(flash.temporal_length, flash.spatial_length, g, sg, merger.dim, merger.ln_w.dtype,
                          merger.ln_w.device)
    if started:                                   # exported mid-stream: readers see the current memory right away
        pub.new_stream()
        pub.publish(state)
    host._qwen_publication = pub
    return pub.export()


class QwenMemoryReader:
    """Reader of a (possibly remote) publication: read() returns a consistent copy of video_embeds [rows, dim] on `device`
    and its metadata, from one small device->host copy (the status words) per read — per QUERY, not per clip."""

    def __init__(self, buf: torch.Tensor, tem_len: int, spa_len: int, rows_cap: int, dim: int, dtype: torch.dtype,
                 device=None):
        self.buf, self.tem_len, self.spa_len, self.rows_cap, self.dim, self.dtype = buf, tem_len, spa_len, rows_cap, dim, dtype
        self.device = torch.device(device) if device is not None else buf.device
        if self.device.index is None:
            self.device = torch.device("cuda", torch.cuda.current_device())
        with torch.cuda.device(self.device):
            self.embeds = torch.empty(rows_cap, dim, dtype=dtype, device=self.device)
            self.ts = torch.empty(max(tem_len, 1), dtype=torch.float32, device=self.device)
            self.pos = torch.empty(max(spa_len, 1), dtype=torch.int64, device=self.device)
            self.status = torch.zeros(9, dtype=torch.int64, device=self.device)
        self.retries = 0
        self._flash = None

    def read(self, max_tries: int = 1000):
        """-> (video_embeds [rows, dim], meta).  meta: tem_thw / spa_thw (host int64 triples, as in the writer's list),
        tem_timestamp fp32 [n_tem] and spa_positions int64 [n_spa] (device), n_frames, clips, epoch, seq.  The tensors are
        views of this reader's buffers: the next read() overwrites them."""
        with torch.cuda.device(self.device):
            for _ in range(max_tries):
                L.check(L.load().fvs_qwen_snapshot(
                    L.ptr(self.buf), self.buf.numel(), self.tem_len, self.spa_len, self.rows_cap, self.dim, L.ptr(self.embeds),
                    self.embeds.shape[0], L.ptr(self.ts), self.ts.numel(), L.ptr(self.pos), self.pos.numel(),
                    L.ptr(self.status), L.cur_stream()), "fvs_qwen_snapshot")
                st = decode_status(self.status.tolist())
                if st["valid"]:
                    (h, w), (hs, ws) = st["grid"], st["small_grid"]
                    meta = {"tem_thw": torch.tensor([st["n_tem"], hs, ws]), "tem_timestamp": self.ts[:st["n_tem"]],
                            "spa_thw": torch.tensor([st["n_spa"], h, w]), "spa_positions": self.pos[:st["n_spa"]],
                            "n_frames": st["n_frames"], "clips": st["clips"], "epoch": st["epoch"], "seq": st["seq0"]}
                    return self.embeds[:st["rows"]], meta
                self.retries += 1            # a publish was writing while we copied
        raise RuntimeError("QwenMemoryReader.read: no consistent snapshot (is a writer stuck mid-publish?)")

    def prepare_realtime_inference(self, position_ids, visual_position_ids):
        """RealtimeStreamingMixin.prepare_realtime_inference (vstream_qwen2vl_realtime.py:632-640) on a snapshot: returns
        (video_embeds, new position ids) for the memory as of the last published clip."""
        video_embeds, m = self.read()
        if self._flash is None:
            from .vstream_qwen2vl_realtime import FlashMemory
            self._flash = FlashMemory()               # calc_am_rope reads no configuration
        tem_positions = torch.round(m["tem_timestamp"].float()).to(torch.int64)
        new_position_id = self._flash.calc_am_rope(position_ids[:, 0], visual_position_ids[0], m["tem_thw"], tem_positions,
                                                   m["spa_thw"], m["spa_positions"])
        return video_embeds, new_position_id.unsqueeze(1)


def _clip_frames(video_clip) -> int:
    if isinstance(video_clip, dict):
        return int(torch.as_tensor(video_clip["video_grid_thw"]).reshape(-1, 3)[0, 0])
    return len(video_clip)


def frame_memory_manager(model, frame_queue, *, preprocess=None, time_meter: Optional[MetricMeter] = None, device=None,
                         on_clip=None, meter_device_time: bool = True):
    """The loop of the reference's memory-manager process (cli_server_2gpu.py:197-239).  With `device`, the loop first
    does `torch.cuda.set_device(device); model = model.cuda()` like the reference (:198-199).  Clips come off `frame_queue`
    (None ends the stream) and go through `preprocess`, which returns the `video_inputs` dict of embed_new_video_clip
    (pixel_values_videos, video_grid_thw; the CLI's image processor — without it, queue items are that dict already);
    start_idx is the running frame count (the clip's length, or its grid's t for a dict).  The reference's five buckets
    are metered from the returned time list with its formulas (first clip not logged).  The reference's call returns after
    its `.cpu()` copies, i.e. when the memory IS updated; with meter_device_time the loop waits on an event (no data leaves
    the GPU) before stopping the clock.  Returns the number of frames embedded."""
    if device is not None:
        torch.cuda.set_device(device)
        model = model.cuda()
    meter = time_meter if time_meter is not None else MetricMeter()
    frame_cnt = 0
    while True:
        video_clip = frame_queue.get()
        if video_clip is None:
            break
        video_inputs = preprocess(video_clip) if preprocess is not None else video_clip
        start_time = time.perf_counter()
        with torch.inference_mode():
            time_list = model.embed_new_video_clip(**video_inputs, start_idx=frame_cnt)
        if meter_device_time:
            ev = torch.cuda.Event()
            ev.record()
            ev.synchronize()
        end_time = time.perf_counter()
        if frame_cnt > 0:
            meter.add('memory_latency', end_time - start_time)
            meter.add('memory_latency_encoder', time_list[2] - time_list[1] + time_list[6] - time_list[5])
            meter.add('memory_latency_readwrite', time_list[3] - time_list[2] + time_list[7] - time_list[6])
            meter.add('memory_latency_cluster', time_list[4] - time_list[3])
            meter.add('memory_latency_retrieve', time_list[5] - time_list[4])
        frame_cnt += _clip_frames(video_clip)
        if on_clip is not None:
            on_clip(frame_cnt)
    return frame_cnt


def pool_memory_manager(pool, queues, *, time_meter: Optional[dict] = None, on_round=None, meter_device_time: bool = True):
    """frame_memory_manager for many streams of one QwenStreamPool.  `queues` maps the sid of each stream (opened in
    `pool` with its own seed) to its frame queue; None on a queue ends that stream only, its publication keeps the last
    memory, and the loop returns {sid: frames embedded} once every queue has ended.  Each round takes at most one clip
    from every queue that has one (later clips wait, in order, for later rounds), blocks for the next clip when none has
    one, and runs ONE pool.step: uint8 frames [T, H, W, 3] when the pool has a preprocessor (one pre-processing call per
    round), else the video_inputs dicts of embed_new_video_clip.  Frames are counted as frame_memory_manager counts them.
    'memory_latency' is metered per stream into time_meter[sid] (a MetricMeter; a stream's first clip not logged),
    waiting on an event with meter_device_time.  Readers attach at any time, before the first frame too:
    QwenMemoryReader(*export_qwen_memory(pool.stream(sid), grid=(h, w))).  on_round({sid: frames}) runs after each
    round.  Each queue is read by one thread that holds at most one of its clips, so a bounded queue still holds its
    producer back; the threads end with their queue's None, or when the loop raises, and the exception's `unconsumed`
    then gives back, per stream, the clips taken from its queue that were not embedded."""
    def step(clips):
        pool.step({k: (c["pixel_values_videos"], c["video_grid_thw"]) if isinstance(c, dict) else c for k, c in clips.items()})
    return serve_pool(queues, step, _clip_frames, time_meter=time_meter, on_round=on_round,
                      meter_device_time=meter_device_time)
