"""The memory-manager side of the reference's realtime serve loop without host round trips (SURVEY.md §8f-2).

Reference topology (Flash-VStream-LLaVA/flash_vstream/serve/cli_video_stream.py:169-256): the main process loads the model,
hangs a `Manager().list()` on `model.video_embedding_memory`, and starts `frame_memory_manager(model, ...)` in a spawned
process; every step the writer pickles `[cur, long, Turing, frame buffer]` (CPU tensors) through the Manager server and the
reader (prepare_inputs_labels_for_multimodal_streaming, vstream_arch.py:476-485) unpickles them under a lock and copies
them back to the GPU.

Here the state never leaves the GPU.  The writer owns an ops.StreamBank; what a reader needs is TWO tensors — the prefix
buffer (already laid out [Turing | long | key | current], the order the reader concatenates in) and the 64-byte header —
and a consistent snapshot of them (fvs_bank_snapshot: the step kernel brackets its write-back with a sequence counter):
  * same process (reader thread):     MemoryReader(*export_bank(bank)).read()
  * other process, same or other GPU: ship `export_bank(bank)` ONCE through a torch.multiprocessing queue (CUDA IPC handles;
    NVLink peer access for another GPU), then MemoryReader(...).read() per query — no pickling of tensors per frame, no
    host copy, no lock shared between processes.
The Manager-list protocol of the unmodified CLI keeps working too: embed_video_streaming publishes CPU copies when
`video_embedding_memory` is a Manager proxy (see VStreamMetaForCausalLM._publish), which is the reference's own cost model.

MetricMeter mirrors the reference's meter (cli_video_stream.py:33-99) with the same bucket names
('memory_latency' in the memory manager, :194-196).

pool_memory_manager is the same loop for many streams of one multistream.StreamPool: one frame queue per stream, one
pool step per round (DESIGN.md §3.9)."""
from __future__ import annotations

import queue as _queue
import threading
import time
from typing import Optional

import torch

from . import ops


class _Metric:
    def __init__(self):
        self.val, self._sum, self.max, self._count = None, 0.0, 0.0, 0

    @property
    def avg(self):
        return float('nan') if self._count == 0 else self._sum / self._count

    def add(self, value):
        self.val = value
        self._sum += value
        self._count += 1
        self.max = max(self.max, value)

    def __str__(self):
        latest = f"{self.val:.6f}" if self.val is not None else "None"
        return f"{latest} ({self.avg:.6f}, {self.max:.6f})"


class MetricMeter:
    """cli_video_stream.py:66-99: add(key, seconds); meter[key] -> 'latest (avg, max)'"""

    def __init__(self):
        self._metrics = {}

    def add(self, key, value):
        self._metrics.setdefault(key, _Metric()).add(value)

    def _get(self, key):
        m = self._metrics.get(key)
        if m is None or m.val is None:
            raise ValueError(f"No values have been added for key '{key}'.")
        return m

    def val(self, key):
        return self._get(key).val

    def avg(self, key):
        return self._get(key).avg

    def max(self, key):
        return self._get(key).max

    def __getitem__(self, key):
        m = self._metrics.get(key)
        if m is None:
            raise KeyError(f"The key '{key}' does not exist.")
        return str(m)


def export_bank(bank: ops.StreamBank):
    """(prefix_buf, header, cur_size, long_size): everything a reader needs.  Both tensors are ordinary CUDA tensors, so a
    torch.multiprocessing Queue/Pipe ships them as CUDA IPC handles (send them once; they stay valid while the writer keeps
    the bank alive)."""
    return bank.prefix_buf, bank.header, bank.cfg.cur_size, bank.cfg.long_size


class MemoryReader:
    """Reader of a (possibly remote) bank: read() returns a consistent copy of the current visual prefix [rows, D] on
    `device` and the writer's counters.  One small device->host copy (the 56-byte status) per read — per QUERY, not per frame."""

    def __init__(self, prefix_buf: torch.Tensor, header: torch.Tensor, cur_size: int, long_size: int, device=None):
        self.prefix_buf, self.header, self.cur_size, self.long_size = prefix_buf, header, cur_size, long_size
        self.device = torch.device(device) if device is not None else prefix_buf.device
        self.out = torch.empty(prefix_buf.shape, dtype=prefix_buf.dtype, device=self.device)
        self.status = torch.zeros(8, dtype=torch.int64, device=self.device)
        self.retries = 0

    def read(self, max_tries: int = 1000):
        with torch.cuda.device(self.device):
            for _ in range(max_tries):
                ops.bank_snapshot(self.prefix_buf, self.header, self.cur_size, self.long_size, out=self.out, status=self.status)
                seq0, seq1, n_tur, n_long, n_cur, n_frames, step = self.status[:7].tolist()
                if seq0 == seq1 and seq0 % 2 == 0:
                    rows = n_tur + n_long * self.long_size ** 2 + n_cur * self.cur_size ** 2
                    return self.out[:rows], {"step": step, "n_frames": n_frames, "n_tur": n_tur, "n_long": n_long,
                                             "n_cur": n_cur, "seq": seq0}
                self.retries += 1            # a step was writing the prefix while we copied it
        raise RuntimeError("MemoryReader.read: no consistent snapshot (is a writer stuck mid-step?)")


def frame_memory_manager(model, frame_queue, *, preprocess=None, time_meter: Optional[MetricMeter] = None, on_step=None,
                         meter_device_time: bool = True):
    """The loop of the reference's memory-manager process (cli_video_stream.py:169-204): clips come off `frame_queue`
    (None ends the stream), go through `preprocess` (the CLI's image_processor.preprocess + .half(); identity by default) and
    into model.embed_video_streaming; 'memory_latency' is metered like the reference (first clip not logged, :193-197).
    The reference's call returns after its `.cpu()` copies, i.e. when the memory IS updated; ours only enqueues, so with
    meter_device_time the loop waits on an event (no data leaves the GPU) before stopping the clock — set it to False to
    let the host run ahead of the GPU.  Returns the number of frames embedded."""
    meter = time_meter if time_meter is not None else MetricMeter()
    frame_cnt = 0
    while True:
        video_clip = frame_queue.get()
        start_time = time.perf_counter()
        if video_clip is None:
            break
        image = preprocess(video_clip) if preprocess is not None else video_clip
        image_tensor = image.unsqueeze(0).to(model.get_vision_tower().device, dtype=torch.float16, non_blocking=True)
        with torch.inference_mode():
            model.embed_video_streaming(image_tensor)
        if meter_device_time:
            ev = torch.cuda.Event()
            ev.record()
            ev.synchronize()
        if frame_cnt > 0:
            meter.add('memory_latency', time.perf_counter() - start_time)
        frame_cnt += video_clip.shape[0]
        if on_step is not None:
            on_step(frame_cnt)
    return frame_cnt


# ---- many streams: one pool, one queue per stream ---------------------------------------------------------------------
def form_round(keys, ready, ended):
    """The next round of a pool serve loop, from which streams have a clip at the head of their queue (`ready`) and which
    have ended (`ended`: their None was taken).  -> (take, done): take = the live streams with a clip ready, in `keys`
    order, one clip each; done = every stream has ended.  take == [] and not done: wait for the next clip."""
    take = [k for k in keys if k in ready and k not in ended]
    return take, all(k in ended for k in keys)


class _Inbox:
    """One thread per queue hands the loop that queue's next item, and holds at most one item at a time: the others stay
    in the caller's queue, so a bounded queue (the reference's Queue(maxsize=10)) still holds its producer back.  After
    the loop takes a stream's item, that stream's thread looks at its queue without blocking ("fetching"), and the loop
    forms its next round only once every such look is done, so a round has every stream whose queue has a clip.  The
    loop waits on a condition for whichever thread delivers next.  A thread ends after handing over its queue's None, or
    at close(); it waits in q.get with a timeout only so that close() is seen, and an item is handed over as soon as it
    is put."""
    STOP_CHECK_S = 0.05

    def __init__(self, queues):
        self.cv = threading.Condition()
        self.held = {}                                    # key -> the item taken from its queue, not yet given out
        self.fetching = set(queues)                       # keys whose thread has not looked at its queue yet
        self.stop = False
        self.threads = [threading.Thread(target=self._forward, args=(k, q), name=f"pool-queue-{k}", daemon=True)
                        for k, q in queues.items()]
        for t in self.threads:
            t.start()

    def _get(self, key, q):
        """the queue's next item, or _STOP once close() was called"""
        try:
            return q.get_nowait()
        except _queue.Empty:
            pass
        with self.cv:
            self.fetching.discard(key)                    # looked: empty for now
            self.cv.notify_all()
        while True:
            try:
                return q.get(timeout=self.STOP_CHECK_S)
            except _queue.Empty:
                with self.cv:
                    if self.stop:
                        return _STOP

    def _forward(self, key, q):
        while True:
            with self.cv:
                while key in self.held and not self.stop:
                    self.cv.wait()
                if self.stop:
                    return
            item = self._get(key, q)
            if item is _STOP:
                return
            with self.cv:                                 # kept even after close(): close() returns it
                self.held[key] = item
                self.fetching.discard(key)
                self.cv.notify_all()
            if item is None:
                return

    def ready(self, block: bool) -> set:
        """the keys whose next item is held, once every thread has looked at its queue; with `block`, wait until there
        is one"""
        with self.cv:
            while self.fetching or (block and not self.held):
                self.cv.wait()
            return set(self.held)

    def take(self, key):
        with self.cv:
            item = self.held.pop(key)
            if item is not None:                          # the thread of an ended stream has returned
                self.fetching.add(key)
            self.cv.notify_all()
            return item

    def close(self) -> dict:
        """stop and join every thread; -> the items taken from the queues and not given out"""
        with self.cv:
            self.stop = True
            self.cv.notify_all()
        for t in self.threads:
            t.join()
        return self.held


_STOP = object()


def serve_pool(queues, step, frames_of, *, time_meter=None, on_round=None, meter_device_time: bool = True):
    """The loop of both families' pool_memory_manager: rounds from form_round, one `step({key: clip})` per round.  If the
    loop raises, its queue threads are stopped first, and the exception's `unconsumed` maps each stream to the items
    taken from its queue that no completed round embedded, in queue order (the failed round's clip, then the one item
    held for the next round; a None among them is the stream's end)."""
    keys = list(queues)
    inbox = _Inbox(queues)
    meters = time_meter if time_meter is not None else {}
    ended, counts, wait, clips = set(), {k: 0 for k in keys}, False, {}
    try:
        while True:
            ready = inbox.ready(block=wait)
            for k in ready:                               # None at the head of a queue ends that stream only
                if k not in ended and inbox.held[k] is None:
                    inbox.take(k)
                    ended.add(k)
            take, done = form_round(keys, ready - ended, ended)
            if done:
                return counts
            wait = not take
            if wait:
                continue
            clips = {k: inbox.take(k) for k in take}
            start_time = time.perf_counter()
            with torch.no_grad():
                step(clips)
            if meter_device_time:
                ev = torch.cuda.Event()
                ev.record()
                ev.synchronize()
            latency = time.perf_counter() - start_time
            for k in take:
                if counts[k] > 0:                         # a stream's first clip is not logged (cli_video_stream.py:193)
                    meters.setdefault(k, MetricMeter()).add('memory_latency', latency)
                counts[k] += frames_of(clips[k])
            clips = {}
            if on_round is not None:
                on_round(dict(counts))
    except BaseException as e:
        held = inbox.close()
        e.unconsumed = {k: [c for c in ((clips[k],) if k in clips else ()) + ((held[k],) if k in held else ())]
                        for k in keys if k in clips or k in held}
        raise
    finally:
        inbox.close()


def pool_memory_manager(pool, queues, *, time_meter: Optional[dict] = None, on_round=None, meter_device_time: bool = True):
    """frame_memory_manager for many streams of one multistream.StreamPool.  `queues` maps the sid of each stream (opened
    in `pool` with its own seed) to its frame queue; None on a queue ends that stream only, its bank keeps the last
    memory, and the loop returns {sid: frames embedded} once every queue has ended.  Each round takes at most one clip
    from every queue that has one (later clips wait, in order, for later rounds), blocks for the next clip when none has
    one, and runs ONE pool.step: uint8 frames [t, H, W, 3] when the pool has a preprocessor (one pre-processing call per
    round), else pixels [t, 3, S, S].  'memory_latency' is metered per stream into time_meter[sid] (a MetricMeter; a
    stream's first clip not logged), waiting on an event with meter_device_time like frame_memory_manager.  Readers
    attach at any time, before the first frame too: MemoryReader(*export_bank(pool.bank(sid))).  on_round({sid: frames})
    runs after each round.  Each queue is read by one thread that holds at most one of its clips, so a bounded queue
    still holds its producer back; the threads end with their queue's None, or when the loop raises, and the
    exception's `unconsumed` then gives back, per stream, the clips taken from its queue that were not embedded."""
    return serve_pool(queues, pool.step, lambda clip: int(clip.shape[0]), time_meter=time_meter, on_round=on_round,
                      meter_device_time=meter_device_time)
