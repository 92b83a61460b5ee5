"""Drop-in mirror of the streaming Flash Memory of Flash-VStream-Qwen/models/vstream_qwen2vl_realtime.py on the sm_90a
kernels: class FlashMemory (:83-329; differs from the offline class only in temporal_compress carrying cluster weights,
:149-183) and the per-clip state update FlashVStreamQwen2VLModel.{embed_new_video_clip, prepare_realtime_inference,
get_video_embedding_memory_cuda_list} (:531-640) as a mixin with the same method names, arguments, state layout (the
13-item `video_embedding_memory` list) and return values.

Differences from the reference (behaviour-preserving):
  * the state is a device-resident object (stream_state.QwenStreamState) updated by one enqueue pass per clip with a single
    32-byte read-back at its end; the reference moves all 13 items to the CPU after every clip and back before the next one
    (its "readwrite" bucket, :582-584/:622-627) and drives the k-means bookkeeping from the host.  The published list holds
    CUDA tensors (on which the reference's own `.cuda()` calls are no-ops) and host thw triples;
  * the feature banks `x` / `small_x` grow in place in capacity-doubling buffers instead of being re-concatenated (a full
    copy of the bank per clip in the reference, :589-591), and every bank frame is merged by the PatchMerger once;
  * the vision tower is injected: `visual.forward_simple_not_merge` (:392-426) runs temporal_pool on the device (row a10)
    and hands the two-resolution patch rows to `visual.encode_patches` — the Qwen2-VL ViT blocks (SURVEY row a11).
"""
from __future__ import annotations

import time
from typing import Callable, Optional

import torch
import torch.nn as nn

from .. import _lib as L
from ..draws import GLOBAL
from ..vstream_arch import _is_manager_proxy
from . import offline as _offline_pass
from . import vstream_qwen2vl_model as _offline
from .compress_functions import weighted_kmeans_ordered_feature
from .patch_merger import PatchMerger
from .stream_state import QwenStreamState, check_device_frames, check_full_res_bank, check_lazy_full_res


class FlashMemory(_offline.FlashMemory):
    """vstream_qwen2vl_realtime.py:83-329"""

    def temporal_compress(self, x, thw, temporal_length, temporal_weights, temporal_indices, draws: Optional[dict] = None):
        """:149-183.  temporal_weights are the carried cluster weights; temporal_indices (timestamps) are accepted and —
        exactly like the reference's weighted_kmeans_ordered_feature, which overwrites them with the mean member row index
        (compress_functions.py:279) — do not influence the result.  draws["source"] (a draws.DrawSource, default the global
        generators) is where the draws not given in `draws` come from."""
        t, h, w = _offline._thw(thw)
        if t <= temporal_length:
            return (x, thw, torch.ones(t, device=x.device), torch.arange(t, device=x.device, dtype=torch.int32),
                    [[i] for i in range(t)])
        assert h % 2 == 0
        assert w % 2 == 0
        x = x.reshape(t, h // 2 * w // 2 * 2 * 2, x.shape[-1])
        if temporal_length == 0:
            x = x[:0, ...]
            tem_thw = thw.clone()
            tem_thw[0] = 0
            return (x.reshape(-1, x.shape[-1]), tem_thw, torch.ones(0, device=x.device),
                    torch.arange(0, device=x.device, dtype=torch.int32), [])
        if self.temporal_method != 'kmeans_ordered':
            # same dispatch table as the offline class; the alternates raise NotImplementedError / ValueError there
            return super().temporal_compress(x.reshape(-1, x.shape[-1]), thw, temporal_length, draws=draws)
        d = draws or {}
        x, weights, timestamps, indices = weighted_kmeans_ordered_feature(
            x, temporal_length, temporal_weights, temporal_indices, init_idx=d.get("init_idx"),
            refill_idx=d.get("refill_idx"), order=d.get("ts_order"), source=d.get("source", GLOBAL))
        tem_thw = thw.clone()
        tem_thw[0] = x.shape[0]
        return x.reshape(-1, x.shape[-1]), tem_thw, weights, timestamps, indices


class VisualB200(nn.Module):
    """The `self.visual` object of the streaming model for this path: flash_memory + merger + the injected ViT blocks.
    `forward` is the offline pass of the same object (qwen/offline.py); offline_max_rows bounds the tower rows of one of
    its calls (whole temporal patches per call, DESIGN.md §3.16)."""

    def __init__(self, flash_memory: FlashMemory, merger: PatchMerger, encode_patches: Optional[Callable] = None,
                 dtype=torch.bfloat16, device="cuda", offline_max_rows: int = _offline_pass.DEFAULT_MAX_ROWS):
        super().__init__()
        self.flash_memory, self.merger, self.encode_patches = flash_memory, merger, encode_patches
        self._dtype, self._device = dtype, torch.device(device)
        self.offline_max_rows = _offline_pass.check_max_rows(offline_max_rows)

    @classmethod
    def from_reference(cls, visual, *, dtype=None, device="cuda", offline_max_rows: int = _offline_pass.DEFAULT_MAX_ROWS,
                       **tower_kw):
        """From the reference's FlashVStreamQwen2VisionTransformerPretrainedModel: its blocks (QwenVisionBlocksB200),
        the mirror FlashMemory of its flash_memory.config and its merger, in `dtype` (default: the module's)."""
        from .vision_tower import QwenVisionBlocksB200
        dtype = dtype or next(visual.parameters()).dtype
        tower = QwenVisionBlocksB200.from_module(visual, dtype=dtype, device=device, **tower_kw)
        m = visual.merger
        merger = PatchMerger.from_weights({k: v.detach().to(dtype) for k, v in (
            ("ln_w", m.ln_q.weight), ("ln_b", m.ln_q.bias), ("fc1_w", m.mlp[0].weight), ("fc1_b", m.mlp[0].bias),
            ("fc2_w", m.mlp[2].weight), ("fc2_b", m.mlp[2].bias))}, device=device)
        return cls(FlashMemory(**visual.flash_memory.config), merger, encode_patches=tower, dtype=dtype, device=device,
                   offline_max_rows=offline_max_rows)

    def forward(self, hidden_states, grid_thw, position_ids, visual_position_ids, draws: Optional[list] = None):
        """vstream_qwen2vl_model.py:388-428: (video_embeds, position_ids).  The full-resolution tower runs only on the
        frames the memory keeps, in chunks of at most offline_max_rows rows; the bits are the unpruned pass's."""
        return _offline_pass.forward(self, hidden_states, grid_thw, position_ids, visual_position_ids, draws=draws,
                                     max_rows=self.offline_max_rows)

    def _apply(self, fn, recurse=True):
        """.cuda() / .to(device) of this module or of its host also move the injected tower (QwenVisionBlocksB200.to), so
        `torch.cuda.set_device(1); model.cuda()` in the reference's memory-manager process puts the whole vision side on
        cuda:1 (cli_server_2gpu.py:198-199)."""
        super()._apply(fn, recurse)
        dev = fn(torch.empty(0, device=self._device)).device
        if dev != self._device:
            self._device = dev
            if hasattr(self.encode_patches, "to"):
                self.encode_patches = self.encode_patches.to(dev)
        return self

    def get_dtype(self):
        return self._dtype

    def get_device(self):
        return self._device

    def forward_simple_not_merge(self, hidden_states, grid_thw):
        """:392-426: build the half-resolution pathway with temporal_pool, run the ViT blocks on both resolutions."""
        hidden_states = hidden_states.view(-1, 3 * 2 * 14 * 14)
        if self.flash_memory.temporal_poolsize > 1:
            small, small_thw, st = [], [], 0
            for i in range(grid_thw.shape[0]):
                ed = st + int(grid_thw[i].prod())
                new_x, new_thw = self.flash_memory.temporal_pool(hidden_states[st:ed], grid_thw[i])
                small.append(new_x)
                small_thw.append(new_thw)
                st = ed
            small_grid_thw = torch.stack(small_thw, dim=0)
            hidden_states = torch.cat([hidden_states] + small, dim=0)
            total_grid_thw = torch.cat([grid_thw, small_grid_thw], dim=0)
        else:
            small_grid_thw, total_grid_thw = None, grid_thw
        if self.encode_patches is None:
            raise NotImplementedError("no vision tower attached: pass encode_patches=QwenVisionBlocksB200(...) (the sm_90a "
                                      "blocks of vstream_qwen2vl_realtime.py:414-423) or any callable(patch_rows, total_grid_thw)")
        return self.encode_patches(hidden_states, total_grid_thw), grid_thw, small_grid_thw


class RealtimeStreamingMixin:
    """embed_new_video_clip / prepare_realtime_inference / get_video_embedding_memory_cuda_list of
    FlashVStreamQwen2VLModel (:531-640) over a device-resident QwenStreamState (stream_state.py).  The host provides
    `self.visual` (VisualB200-like: flash_memory, merger, forward_simple_not_merge, get_dtype, get_device).

    fvs_bank_device_frames: None (default: every bank frame in HBM) or an integer >= 0 — how many frames of the
    full-resolution and merged feature banks stay in HBM; later frames go to pinned host memory and a step reads back only
    the frames it retrieves (DESIGN.md §3.13).  Results are bit-identical either way.  It applies from the next stream
    (and to load_video_stream); changing it in the middle of a stream raises ValueError.

    fvs_bank_small_device_frames: the same for the half-resolution bank, whose later frames the retrieval sweeps in place
    over PCIe every step (DESIGN.md §3.13).  With both caps set, a stream's HBM no longer grows with its length.

    fvs_lazy_full_res: False (default) or True — keep each clip's full-resolution pixel rows and run the full-resolution
    tower on a frame only the first time the DAM picks it (DESIGN.md §3.18); item 7 of the list is then the zero-row
    stand-in.  Needs flash_memory_temporal_poolsize=2.  Like the caps, it applies from the next stream (and to
    load_video_stream); changing it in the middle of a stream raises ValueError.

    fvs_full_res_bank: True (default) or False — with fvs_lazy_full_res, keep no full-resolution or merged row beyond
    the DAM, and re-encode from its pixel rows a pick the previous DAM does not hold (DESIGN.md §3.19).  False without
    fvs_lazy_full_res raises ValueError; it applies, and refuses a change mid-stream, like the knobs above."""

    fvs_bank_device_frames = None
    fvs_bank_small_device_frames = None
    fvs_lazy_full_res = False
    fvs_full_res_bank = True

    def _bank_device_frames(self):
        return self._cap("fvs_bank_device_frames", "device_frames")

    def _bank_small_device_frames(self):
        return self._cap("fvs_bank_small_device_frames", "small_device_frames")

    def _lazy_full_res(self):
        return self._cap("fvs_lazy_full_res", "lazy_full_res",
                         lambda v, k: check_lazy_full_res(v, self.visual.flash_memory, k))

    def _full_res_bank(self, lazy: bool):
        return self._cap("fvs_full_res_bank", "full_res_bank",
                         lambda v, k: check_full_res_bank(v, lazy, k, "fvs_lazy_full_res"))

    def _cap(self, knob, attr, check=check_device_frames):
        """the validated value of the cap attribute `knob`, which the stream in progress (its state's `attr`) must share"""
        cap = check(getattr(self, knob), knob)
        st = self.__dict__.get("stream_state")
        if st is not None and st.n_frames > 0 and self.video_embedding_memory and getattr(st, attr) != cap:
            raise ValueError(f"{knob} changed from {getattr(st, attr)} to {cap} in the middle of a stream: "
                             f"it takes effect with the next stream (init_streaming())")
        return cap

    def init_streaming(self):
        self.use_video_streaming_mode = True
        self.video_embedding_memory = []
        from torch.multiprocessing import Lock      # what the reference hangs there (vstream_qwen2vl_realtime.py:43,529):
        self.video_embedding_mem_lock = Lock()      # shared with a spawned memory-manager process when the model is passed to it
        self.stream_state = None

    def __getstate__(self):
        """The reference's CLI pickles the whole model into its memory-manager process (cli_server_2gpu.py:301-304).  The
        streaming state is not transferred, so a host with a stream in progress refuses; a publication stays with the
        process that exported it."""
        state = self.__dict__.get("stream_state")
        if state is not None and state.n_frames > 0:
            raise L.FvsError("a Qwen2-VL host with a stream in progress cannot be pickled: init_streaming() first, or hand "
                             "the reader its tensors (flash_vstream_b200.qwen.serve.export_qwen_memory)")
        d = dict(super().__getstate__())
        d.pop("_qwen_publication", None)
        return d

    def get_video_embedding_memory_cuda_list(self):
        with self.video_embedding_mem_lock:
            return [item.cuda() if hasattr(item, 'cuda') else item for item in self.video_embedding_memory]

    def embed_new_video_clip(self, pixel_values_videos, video_grid_thw, start_idx, draws: Optional[dict] = None):
        """:548-630.  One clip: tower, then QwenStreamState.step (one enqueue pass, one 32-byte read-back), then the
        13-item list is republished under the lock.  Returns the reference's list of 8 host-clock timestamps; the buckets
        keep their names, but since nothing blocks between them the device time of a clip shows up in the bucket that ends
        with the read-back ("temporal_compress" .. "merger" of the reference's meter are one bucket here: time_3..time_6)."""
        time_0 = time.perf_counter()
        assert self.use_video_streaming_mode
        cap, small_cap, lazy = self._bank_device_frames(), self._bank_small_device_frames(), self._lazy_full_res()
        bank = self._full_res_bank(lazy)
        grid_host = video_grid_thw.cpu()          # the grid stays on the host: every shape below comes from it (a CUDA grid
        t, h, w = (int(v) for v in grid_host.reshape(-1, 3)[0].tolist())   # costs one sync here, a host grid none)
        pixel_values_videos = pixel_values_videos.type(self.visual.get_dtype()).to(self.visual.get_device(), non_blocking=True)
        time_1 = time.perf_counter()
        if lazy:                                  # only the half-resolution rows now; the picked frames' full rows later
            small, small_grid = self.visual.flash_memory.temporal_pool(pixel_values_videos.view(-1, 3 * 2 * 14 * 14),
                                                                       grid_host.reshape(-1, 3)[0])
            if self.visual.encode_patches is None:
                raise NotImplementedError("fvs_lazy_full_res: no vision tower attached (visual.encode_patches)")
            feats = self.visual.encode_patches(small, small_grid.view(1, 3))
        else:
            feats, _, small_grid_thw = self.visual.forward_simple_not_merge(pixel_values_videos, grid_host)
        time_2 = time.perf_counter()
        if lazy:
            hs, ws = h // 2, w // 2
            x_new, small_new = pixel_values_videos.view(-1, 3 * 2 * 14 * 14), feats
        elif small_grid_thw is not None:
            hs, ws = h // 2, w // 2
            x_new, small_new = feats[: t * h * w], feats[t * h * w: t * h * w + t * hs * ws]
        else:
            hs, ws = h, w
            x_new = small_new = feats
        pub = self.__dict__.get("_qwen_publication")              # set by qwen.serve.export_qwen_memory (opt-in)
        if self.stream_state is None or not self.video_embedding_memory:
            self.stream_state = QwenStreamState(self.visual.flash_memory, self.visual.merger, device_frames=cap,
                                                small_device_frames=small_cap, lazy_full_res=lazy, full_res_bank=bank)
            if pub is not None:
                pub.new_stream()
        time_3 = time.perf_counter()
        self.stream_state.step(x_new, small_new, t, (h, w), (hs, ws), start_idx, draws=draws,
                               tower=self.visual.encode_patches if lazy else None)
        time_6 = time.perf_counter()
        if pub is not None:
            pub.publish(self.stream_state)                         # the clip is final: one launch, under the seqlock
        self._publish(self.stream_state.as_list())
        time_7 = time.perf_counter()
        return [time_0, time_1, time_2, time_3, time_6, time_6, time_6, time_7]

    # ---- suspend / resume (DESIGN.md §3.12) ---------------------------------------------------------------------------
    def save_video_stream(self):
        """The stream in progress as a checkpoint.StreamCheckpoint (pinned host memory) that load_video_stream continues
        bit for bit, here, in another process or on another GPU.  Draws come from the global generators (draws.GLOBAL):
        settled first, neither stored nor set — a resumed stream continues from the resuming process's generators."""
        from ..draws import GLOBAL
        state = self.__dict__.get("stream_state")
        if state is None or state.n_frames == 0 or not self.video_embedding_memory:
            raise ValueError("save_video_stream: no stream in progress")
        GLOBAL.settle()
        return state.checkpoint()

    def load_video_stream(self, ckpt):
        """Continue the stream of `ckpt` in this host: `stream_state` is restored on the vision side's device and the
        13-item list republished.  An exported host (qwen.serve.export_qwen_memory) must have the checkpoint's grid; its
        readers see the resumed memory under a new epoch."""
        from .. import checkpoint as CK
        if ckpt.family != CK.QWEN:
            raise ValueError(f"load_video_stream: a {ckpt.family!r} checkpoint is not a Qwen2-VL stream's")
        pub = self.__dict__.get("_qwen_publication")
        if pub is not None and ckpt.counters["n_frames"] and \
                (tuple(ckpt.config["grid"]), tuple(ckpt.config["small_grid"])) != (pub.grid, pub.small_grid):
            raise ValueError(f"load_video_stream: config.grid {ckpt.config['grid']} / {ckpt.config['small_grid']} is not "
                             f"the exported grid {pub.grid} / {pub.small_grid}")
        cap = check_device_frames(self.fvs_bank_device_frames, "fvs_bank_device_frames")
        small_cap = check_device_frames(self.fvs_bank_small_device_frames, "fvs_bank_small_device_frames")
        lazy = check_lazy_full_res(self.fvs_lazy_full_res, self.visual.flash_memory, "fvs_lazy_full_res")
        bank = check_full_res_bank(self.fvs_full_res_bank, lazy, "fvs_full_res_bank", "fvs_lazy_full_res")
        state = QwenStreamState.restore(ckpt, self.visual.flash_memory, self.visual.merger, self.visual.get_device(),
                                        device_frames=cap, small_device_frames=small_cap, lazy_full_res=lazy,
                                        full_res_bank=bank)
        state.tower = self.visual.encode_patches if lazy else None
        if state.n_frames == 0:
            self.stream_state = None
            self._publish([])
            return
        self.stream_state = state
        if pub is not None:
            pub.new_stream()
            pub.publish(state)
        self._publish(state.as_list())

    def _publish(self, new_list):
        """`self.video_embedding_memory[:] = [...]` under the lock (:620-624).  The reference's CLI hangs a Manager().list()
        there and reads it from another process (cli_server_2gpu.py:301, :632-640): a Manager server cannot forward CUDA IPC
        handles, so the items travel as host copies, the reference's own cost.  The two feature banks (items 7 and 9) are
        read by nobody on the LLM side (prepare_realtime_inference unpacks and drops them) nor by this writer (the stream
        state owns them), so empty stand-ins travel instead of the whole O(n) banks; the thw items stay exact."""
        mem = self.video_embedding_memory
        if _is_manager_proxy(mem):
            new_list = [v[:0].cpu() if i in (7, 9) else v.cpu() if torch.is_tensor(v) else v for i, v in enumerate(new_list)]
        with self.video_embedding_mem_lock:
            mem[:] = new_list

    def prepare_realtime_inference(self, position_ids, visual_position_ids):
        """:632-640"""
        assert self.use_video_streaming_mode
        (tem_x, tem_thw, tem_weights, tem_timestamp, spa_x, spa_thw, spa_positions, x, thw, small_x, small_thw, video_embeds,
         video_embeds_shape) = self.get_video_embedding_memory_cuda_list()
        tem_positions = torch.round(tem_timestamp.float()).to(torch.int64)       # np.round of the reference: half to even
        new_position_id = self.visual.flash_memory.calc_am_rope(position_ids[:, 0], visual_position_ids[0], tem_thw,
                                                                tem_positions, spa_thw, spa_positions)
        return video_embeds, new_position_id.unsqueeze(1)


class FlashVStreamQwen2VLRealtimeB200(RealtimeStreamingMixin, nn.Module):
    """Minimal host of the mixin for this path (vision side only; the Qwen2 language model is outside §8)."""

    def __init__(self, visual: VisualB200):
        super().__init__()
        self.visual = visual
        self.init_streaming()
