"""Many video streams on one GPU: a pool of persistent banks stepped together (fvs_stream_step_multi, include/fvs_b200.h).

One `StreamPool.step` encodes the clips of every listed stream in the ViT's micro-batches (weights read once per
micro-batch instead of once per stream) and consolidates all their banks in as few cooperative launches as fit on the
device.  Each stream's result is bit-identical to running it alone through the single-stream path
(`FlashVStreamB200.embed_video_streaming` / `consolidate_streaming`) with the same draws.

RNG: each stream owns a `draws.DrawSource` seeded by `open(seed)` (contract in draws.py), so a stream draws what the
single-stream path draws after `torch.manual_seed(seed); random.seed(seed)` and never touches the global generators.
"""
from __future__ import annotations

import os
from typing import Optional

import numpy as np
import torch

from . import ops
from .compress_functions import kmeans_draws
from .draws import DrawSource

REFERENCE_GRID = 24   # ViT-L/14 at 336 px: the patch grid of finished features when the model has no tower of its own


class _Stream:
    def __init__(self, bank: ops.StreamBank, rng: DrawSource):
        self.bank, self.rng = bank, rng


class StreamPool:
    """A pool of streams sharing one model's tower, abstract-memory weights and STAR config.

    `open(seed)` -> sid; `step({sid: clip, ...})` advances the listed streams in one batched step (clips: pixels
    [t,3,S,S] or [1,t,3,S,S] for a model with a ViT engine, or finished features [t, grid*grid, D] f16; t <= chunk_cap);
    `prefix(sid)` / `state(sid)` are views of the stream's bank; `bank(sid)` is the ops.StreamBank itself (hand it to
    serve.export_bank / MemoryReader).  `close(sid)` resets the bank and keeps it for the next `open`.  Configs the
    fused streaming step does not cover raise NotImplementedError: stream them through the model's single-stream path.
    `device_frames` (ops.StreamBank): every bank of the pool keeps only that many frames of its frame buffer in HBM, the
    later ones in pinned host memory, so a stream's HBM stays what it was when the bank was made.
    `preprocess` (a preprocess.CLIPFramePreprocessor whose crop is the tower's image size): `step` also takes decoded
    uint8 frames [t, H, W, 3] per stream (any mix of sizes, host or device); the round's clips go through ONE
    `preprocess.many` call, whose contiguous output the step reads as it is (no concatenation)."""

    def __init__(self, model, *, chunk_cap: int = 1, max_streams: Optional[int] = None,
                 device_frames: Optional[int] = None, preprocess=None):
        host = model.get_model()
        ntm = host.attention_model
        D = ntm.q_proj.weight.shape[1]
        tower = host.get_vision_tower()
        engine = getattr(tower, "engine", None) if tower is not None else None
        if engine is not None and (engine.dtype != torch.float16 or engine.keep_cls):
            engine = None          # the pooled encoder tail needs an f16 tower with select_feature 'patch'
        self.vit = engine
        grid = engine.grid if engine is not None else REFERENCE_GRID
        s = model._star_cfg()
        knob = model._fused_reject(s, grid, D, torch.float16)
        if knob is not None:
            raise NotImplementedError(f"StreamPool: {knob} is outside what the batched streaming step covers; stream this "
                                      f"config through the model's single-stream path")
        self.cfg = model._fused_cfg(s, grid, D, torch.float16)
        self.ntm = (ntm.q_proj.weight, ntm.q_proj.bias, ntm.k_proj.weight, ntm.k_proj.bias)
        self.device = ntm.q_proj.weight.device
        if self.device.type != "cuda":
            raise ops.L.FvsError("StreamPool needs the model on a CUDA device (no CPU fallback)")
        self.chunk_cap = int(chunk_cap)
        self.device_frames = ops.device_window(self.cfg, self.chunk_cap, device_frames)
        self.max_streams = max_streams
        self.preprocess = preprocess
        self._streams: dict[int, _Stream] = {}
        self._free: list[ops.StreamBank] = []
        self._next = 0

    # ---- streams -------------------------------------------------------------------------------------------------------
    def open(self, seed: Optional[int] = None, *, checkpoint=None) -> int:
        """A new stream -> its sid.  With `checkpoint` (a StreamCheckpoint of `checkpoint(sid)`, from this pool or another,
        on any device), the stream continues where the checkpoint left it: its bank and its draw source's generators.  A
        checkpoint without a draw source (from the single-stream model, whose draws come from the global generators) needs
        `seed=` for the generators the stream draws from from here on."""
        if self.max_streams is not None and len(self._streams) >= self.max_streams:
            raise RuntimeError(f"StreamPool is full ({self.max_streams} streams)")
        if checkpoint is not None and checkpoint.rng is None and seed is None:
            raise ValueError("StreamPool.open: this checkpoint carries no draw source (single-stream model): pass seed=")
        bank = self._free.pop() if self._free else ops.StreamBank(self.cfg, self.ntm, chunk_cap=self.chunk_cap, device=self.device,
                                                                  device_frames=self.device_frames)
        if checkpoint is None:
            bank.reset()
        else:
            try:
                bank.restore(checkpoint)
            except BaseException:
                self._free.append(bank)
                raise
        if seed is None and checkpoint is None:
            seed = int.from_bytes(os.urandom(8), "little") >> 1
        rng = DrawSource(int(seed) if seed is not None else 0, self.device)
        if checkpoint is not None and checkpoint.rng is not None:
            r = checkpoint.rng
            rng.cpu = r["cpu"].clone()
            rng.cuda = r["cuda"].clone() if rng.cuda is not None and r["cuda"] is not None else rng.cuda
            rng.py.setstate(r["py"])
        sid = self._next
        self._next += 1
        self._streams[sid] = _Stream(bank, rng)
        return sid

    def checkpoint(self, sid: int):
        """The stream's state as a StreamCheckpoint in pinned host memory: its bank and its draw source (settled first:
        this blocks on the source's pending refill read-backs, so no consumed count is lost or applied twice).  Suspend =
        checkpoint(sid) then close(sid); resume = open(checkpoint=...)."""
        from . import checkpoint as CK
        st = self._streams[sid]
        st.rng.settle()
        return st.bank.checkpoint(rng=CK.rng_state(st.rng))

    def close(self, sid: int):
        st = self._streams.pop(sid)
        st.bank.reset()
        self._free.append(st.bank)

    def __len__(self):
        return len(self._streams)

    def bank(self, sid: int) -> ops.StreamBank:
        return self._streams[sid].bank

    def prefix(self, sid: int) -> torch.Tensor:
        """[Turing | long | key | current] of the stream: a view of its bank (vstream_arch.py:483)"""
        return self._streams[sid].bank.prefix()

    def state(self, sid: int):
        """(cur, long, Turing, frame buffer) views, as StreamBank.state()"""
        return self._streams[sid].bank.state()

    # ---- one batched step ----------------------------------------------------------------------------------------------
    def step(self, clips: dict, draws: Optional[dict] = None, *, max_blocks: int = 0):
        """One step of every stream in `clips` ({sid: clip}); the others do not move.  draws={sid: (init_idx, refill_idx)}
        bypasses a stream's generators.  If any stream's step is refused, no stream moves and no generator advances.
        With `preprocess`, a round of uint8 frames is pre-processed in one call first; a round mixing them with pixels or
        features is refused."""
        draws = draws or {}
        sids = list(clips)
        streams = [self._streams[sid] for sid in sids]
        frames = {_is_frames(clips[sid]) for sid in sids}
        if len(frames) > 1:
            raise ValueError("one step takes uint8 frames, pixels or features for every stream, not a mix")
        packed = None
        if frames == {True}:
            if self.preprocess is None:
                raise ValueError("uint8 frames need a pool made with preprocess=CLIPFramePreprocessor(...)")
            packed, inputs = self.preprocess.many([clips[sid] for sid in sids])
            if packed.dim() != 4:
                raise ValueError("the preprocessor made crops of different sizes for this round")
        else:
            inputs = []
            for sid in sids:
                x = clips[sid]
                if x.ndim == 5:
                    assert x.shape[0] == 1, "one clip per stream"
                    x = x[0]
                inputs.append(x)
        pixels = {x.ndim == 4 and x.shape[1] == 3 for x in inputs}
        if len(pixels) != 1:
            raise ValueError("one step takes either pixels or features for every stream")
        vit = None
        if pixels.pop():
            if self.vit is None:
                raise NotImplementedError("pixels need the model's ViT engine (an f16 tower with select_feature 'patch')")
            vit = self.vit
        snaps = [st.rng.snapshot() for st in streams]
        dr, refills = [], []
        try:
            for sid, st, x in zip(sids, streams, inputs):
                t, r = x.shape[0], None
                d = draws.get(sid)
                if d is None and st.bank.needs_draws(t):
                    *d, r = kmeans_draws(st.rng, st.bank.working_rows(t), st.bank.cfg.long_len, self.device)
                dr.append(d)
                refills.append(r)
            ops.stream_step_many([st.bank for st in streams], inputs, vit=vit, draws=dr, max_blocks=max_blocks,
                                 _packed=packed)
        except BaseException:
            for st, snap in zip(streams, snaps):
                st.rng.rewind(snap)
            raise
        for st, r in zip(streams, refills):
            if r is not None:          # learn (asynchronously) how many refill candidates the device consumed
                r.consumed_from(st.bank.info()[1])


def _is_frames(clip) -> bool:
    """decoded frames (uint8 [t, H, W, 3], tensor or array), as opposed to pixels or features"""
    return clip.dtype == (torch.uint8 if isinstance(clip, torch.Tensor) else np.uint8)
