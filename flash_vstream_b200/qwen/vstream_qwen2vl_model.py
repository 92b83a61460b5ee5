"""Drop-in mirror of the Flash Memory of Flash-VStream-Qwen/models/vstream_qwen2vl_model.py (class FlashMemory :78-330 and
the grid helpers :43-75) on the sm_90a kernels: same class name, constructor arguments, method names, argument meaning,
return tuples and error behaviour, so a caller (the reference's FlashVStreamQwen2VLModel, :478) can swap the import.

Data layout (as in the reference): a clip is `t` frames of `h*w` ViT tokens, rows ordered (t, h/2, w/2, 2, 2) so that every
4 consecutive rows are one 2x2 merge block; one "frame" for clustering / retrieval is the flattened [h*w * xdim] row.
CSM = the temporal_length cluster centroids of the half-resolution clip; DAM = the spatial_length full-resolution frames
nearest (Euclidean, 16-bit GEMM form) to the heaviest centroids.

No CPU path: tensors must be CUDA tensors; every arithmetic step runs in libfvs_b200.so (torch only allocates, slices,
concatenates and scatters).
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch
import torch.nn as nn

from .. import ops as O
from ..draws import GLOBAL
from . import compress_functions as CF
from . import ops as Q
from .compress_functions import weighted_kmeans_ordered_feature

_CFG_KEYS = ("flash_memory_temporal_length", "flash_memory_temporal_method", "flash_memory_temporal_poolsize",
             "flash_memory_temporal_pca_dim", "flash_memory_spatial_length", "flash_memory_spatial_method")
# temporal methods the reference dispatches on (vstream_qwen2vl_model.py:160-172) -> the callables of compress_functions
_ALTERNATE_TEMPORAL = dict(merge="merge_feature", drop="drop_feature", kmeans="weighted_kmeans_feature",
                           pca_kmeans_ordered="pca_weighted_kmeans_ordered_feature",
                           torchpca_kmeans_ordered="torchpca_weighted_kmeans_ordered_feature",
                           fast_kmeans_ordered="fast_weighted_kmeans_ordered_feature", dbscan="dbscan_feature",
                           gmm="gmm_feature", attention="attention_feature")
_TEMPORAL_METHODS = ("sample", "merge", "drop", "kmeans", "kmeans_ordered", "pca_kmeans_ordered", "torchpca_kmeans_ordered",
                     "fast_kmeans_ordered", "dbscan", "gmm", "attention")
_SPATIAL_METHODS = ['sample', 'nearest', 'klarge_retrieve', 'klarge_retrieve_cos']


def _ints(thw):
    return tuple(int(v) for v in (thw.tolist() if isinstance(thw, torch.Tensor) else thw))


_thw = _ints   # used by the streaming subclass


def _like(thw, values):
    return torch.tensor(list(values), dtype=thw.dtype, device=thw.device)


def _with_t(thw, t):
    out = thw.clone()
    out[0] = t
    return out


def get_real_grid_thw(thw, flash_memory_config):
    """vstream_qwen2vl_model.py:43-60: grid of one clip after memory compression (host integer logic): at most
    temporal_length/2 frames; with temporal pooling the side lengths are halved and rounded up to even."""
    if flash_memory_config is None:
        return thw
    pool = flash_memory_config['flash_memory_temporal_poolsize']
    if pool > 2:
        raise NotImplementedError(f"Only support t_pool=2 or t_pool=1, t_pool={pool}")
    t, h, w = _ints(thw)
    if pool == 2:
        h, w = (h // 2 + 1) // 2 * 2, (w // 2 + 1) // 2 * 2
    return _like(thw, (min(t, flash_memory_config['flash_memory_temporal_length'] // 2), h, w))


def get_real_grid_thws(grid_thw, flash_memory_config):
    """vstream_qwen2vl_model.py:62-67"""
    return torch.stack([get_real_grid_thw(row, flash_memory_config) for row in grid_thw], dim=0)


def get_spatial_real_grid_thw(thw, flash_memory_config):
    """vstream_qwen2vl_model.py:69-75: the DAM side keeps at most spatial_length/2 frames (a None config is dereferenced
    there too, so it raises TypeError like the reference)."""
    t, h, w = _ints(thw)
    cap = flash_memory_config['flash_memory_spatial_length'] // 2
    return _like(thw, (min(t, cap), h, w))


class FlashMemory(nn.Module):
    """vstream_qwen2vl_model.py:78-330.  `draws` (forward / temporal_compress / spatial_enhance) optionally replays the RNG
    draws and unstable-sort permutations recorded from a reference run: dict(init_idx=, refill_idx=, ts_order=,
    weight_order=, source=); by default the same generators as the reference are consumed (source: a draws.DrawSource
    to draw from instead) and ties sort stably."""

    def __init__(self, flash_memory_temporal_length=120, flash_memory_temporal_method='kmeans_ordered',
                 flash_memory_temporal_poolsize=2, flash_memory_temporal_pca_dim=32, flash_memory_spatial_length=60,
                 flash_memory_spatial_method='klarge_retrieve'):
        super().__init__()
        given = locals()
        self.config = {k: given[k] for k in _CFG_KEYS}
        for k in ("flash_memory_temporal_length", "flash_memory_spatial_length"):
            short = k.replace("flash_memory_", "")
            # the reference's message for the spatial check prints the temporal value (:104); kept for message parity
            assert given[k] % 2 == 0, f"In FlashMemory, {short} should be even, {short}={flash_memory_temporal_length}"
        # lengths count LLM tokens of 2 temporal patches each -> frames kept = length / 2
        self.temporal_length, self.spatial_length = flash_memory_temporal_length // 2, flash_memory_spatial_length // 2
        self.temporal_method, self.spatial_method = flash_memory_temporal_method, flash_memory_spatial_method
        self.temporal_poolsize, self.temporal_pca_dim = flash_memory_temporal_poolsize, flash_memory_temporal_pca_dim

    # ------------------------------------------------------------------------------------------------ :113-142
    def temporal_pool(self, x, thw):
        t, h, w = _ints(thw)
        assert self.temporal_poolsize == 2
        assert x.shape[-1] == 3 * 2 * 14 * 14
        for name, side in (("pad_h", h), ("pad_w", w)):
            if (side // 2) % 2:
                raise NotImplementedError(f"Performing temporal pool, {name} > 0, {name}={(side // 2) % 2}")
        pooled = Q.temporal_pool(x, t, h, w)
        new_thw = thw.clone() if isinstance(thw, torch.Tensor) else torch.tensor([t, h, w])
        new_thw[1], new_thw[2] = h // 2, w // 2
        return pooled, new_thw

    # ------------------------------------------------------------------------------------------------ :145-180
    def _compress_frames(self, frames, keep, weights=None, times=None, draws: Optional[dict] = None):
        """[t, tokens, xdim] -> (frames', weights, timestamps, member lists) by the configured temporal method"""
        method = self.temporal_method
        if method not in _TEMPORAL_METHODS:
            raise ValueError(f"temporal_method should be one of {_TEMPORAL_METHODS}")
        t = frames.shape[0]
        if method == 'sample':
            picks = torch.linspace(0, t - 1, keep)
            return O.gather_rows(frames, picks.long().to(frames.device)), None, picks.to(frames.device).long(), None
        if method in ('kmeans_ordered', 'fast_kmeans_ordered'):      # same arithmetic (see CF.fast_weighted_kmeans_ordered_feature)
            d = draws or {}
            return weighted_kmeans_ordered_feature(frames, keep, weights, times, init_idx=d.get("init_idx"),
                                                   refill_idx=d.get("refill_idx"), order=d.get("ts_order"),
                                                   source=d.get("source", GLOBAL))
        return getattr(CF, _ALTERNATE_TEMPORAL[method])(frames, keep)      # raises NotImplementedError (not built)

    def temporal_compress(self, x, thw, temporal_length, draws: Optional[dict] = None):
        """CSM memory from temporal clustering.  Returns (x [T1*h*w, xdim], tem_thw, weights, timestamps, indices)."""
        t, h, w = _ints(thw)
        dev = x.device
        if t <= temporal_length:        # nothing to compress: unit weights, timestamps 0..t-1
            return x, thw, torch.ones(t, device=dev), torch.arange(t, device=dev, dtype=torch.int32), [[i] for i in range(t)]
        assert h % 2 == 0
        assert w % 2 == 0
        xdim = x.shape[-1]
        if temporal_length == 0:
            return (x.new_empty(0, xdim), _with_t(thw, 0), torch.ones(0, device=dev),
                    torch.arange(0, device=dev, dtype=torch.int32), [])
        kept, weights, timestamps, indices = self._compress_frames(x.reshape(t, h * w, xdim), temporal_length, draws=draws)
        return kept.reshape(-1, xdim), _with_t(thw, kept.shape[0]), weights, timestamps, indices

    # ------------------------------------------------------------------------------------------------ :183-244
    def spatial_enhance(self, x, small_x, thw, tem_x, tem_thw, tem_weights, tem_positions, tem_indices,
                        draws: Optional[dict] = None):
        """Given tem_x (CSM memory), retrieve spa_x (DAM memory) from x (feature bank)."""
        t, h, w = _ints(thw)
        xdim = x.shape[-1]
        bank = x.reshape(t, h * w, xdim)
        picks = self.spatial_picks(small_x, t, tem_x, tem_thw, tem_weights, tem_positions, draws=draws)
        if t <= self.spatial_length:    # the whole bank fits
            return bank, _with_t(thw, t), picks
        return O.gather_rows(bank, picks), _with_t(thw, self.spatial_length), picks

    def spatial_picks(self, small_x, t, tem_x, tem_thw, tem_weights, tem_positions, draws: Optional[dict] = None):
        """The frame indices spatial_enhance retrieves from a bank of t frames (int64 [min(t, spatial_length)], on
        small_x's device) without touching the full-resolution bank: a caller that keeps that bank elsewhere gathers
        the frames itself (stream_state.QwenStreamState).  small_x may be a qwen.ops.TieredBank of the t frames."""
        dev = small_x.device
        if t <= self.spatial_length:
            return torch.arange(t, device=dev).long()
        if self.spatial_method not in _SPATIAL_METHODS:
            raise ValueError(f"spatial_method should be one of {_SPATIAL_METHODS}")
        n = self.spatial_length
        if self.spatial_method == 'sample':
            return torch.linspace(0, t - 1, n).round().long().to(dev)
        order = (draws or {}).get("weight_order")            # torch.argsort(tem_weights, descending=True) of the reference
        ranked = O.argsort_desc(tem_weights) if order is None else torch.as_tensor(order).to(device=dev, dtype=torch.int64)
        heaviest = ranked[:n]
        if self.spatial_method == 'nearest':
            return tem_positions[heaviest]                    # index plumbing only
        # 'klarge_retrieve' (Euclidean distance) / 'klarge_retrieve_cos' (argmin of the cosine similarity, :208-215)
        bank = small_x if isinstance(small_x, Q.TieredBank) else small_x.reshape(t, -1)
        return self._klarge_retrieve(tem_x.reshape(_ints(tem_thw)[0], -1), heaviest, bank,
                                     "cosine" if self.spatial_method == 'klarge_retrieve_cos' else "euclidean")

    def _klarge_retrieve(self, centroids, klarge_indices, bank, metric="euclidean"):
        """efficient_euclidean_distance / cosine_similarity + argmin (:197-215, :231-238) in the 16-bit dtype of the
        features: one fvs_qwen_klarge_retrieve call (centroid gather, norms, c.b, distance / similarity tail, argmin)."""
        if bank.dtype not in (torch.float16, torch.bfloat16):
            raise NotImplementedError(f"klarge_retrieve on {bank.dtype} features: the Qwen2-VL vision tower emits 16-bit "
                                      f"features")
        return Q.klarge_retrieve(centroids, klarge_indices, bank, metric=metric)

    # ------------------------------------------------------------------------------------------------ :246-251
    def cat_spa_tem(self, spa_x, tem_x):
        """DAM rows first, then CSM rows (whole 2x2 merge groups stay together)"""
        width = spa_x.shape[-1]
        return torch.cat([spa_x.reshape(-1, width), tem_x.reshape(-1, width)], dim=0).contiguous()

    # ------------------------------------------------------------------------------------------------ :254-277
    def calc_am_rope(self, position_id, visual_position_id, tem_thw, tem_positions, spa_thw, spa_positions):
        """AM-RoPE: 3-D position ids of the memory tokens from the CSM / DAM temporal positions (batch size 1, in place)."""
        is_visual = visual_position_id >= 0
        where = torch.nonzero(is_visual, as_tuple=False)
        first, last = int(where[0]), int(where[-1])
        start = position_id[:, first]
        assert start[0] == start[1] and start[1] == start[2]
        (dam_t, dam_h, dam_w), (csm_t, csm_h, csm_w) = _ints(spa_thw), _ints(tem_thw)
        for name, pos, frames in (("spa", spa_positions, dam_t), ("tem", tem_positions, csm_t)):
            assert pos.shape[0] == frames, f"t_positions.shape={pos.shape} should be equal to llm_grid_t={frames}"
        n_dam, n_csm = dam_t * dam_h * dam_w // 4, csm_t * csm_h * csm_w // 4
        assert n_dam + n_csm == last - first + 1, \
            f"sth went wrong! check: spa_size={n_dam}, tem_size={n_csm}, visual_end_pos={last}, visual_start_pos={first}"
        ids = Q.am_rope(spa_positions.long(), (dam_t, dam_h // 2, dam_w // 2), tem_positions.long(),
                        (csm_t, csm_h // 2, csm_w // 2), int(start[0]), position_id.device)
        position_id[:, is_visual] = ids.to(position_id.dtype)
        return position_id

    # ------------------------------------------------------------------------------------------------ :279-330
    def _streams(self, x, grid_thw, small_grid_thw):
        """per-sample (full-resolution rows, grid, half-resolution rows, grid); without a second resolution the
        full-resolution rows serve as both (:285-296)"""
        if small_grid_thw is None:
            parts = torch.split(x, grid_thw.prod(dim=1).tolist())
            return [(p, g, p, g) for p, g in zip(parts, grid_thw)]
        parts = torch.split(x, torch.cat([grid_thw, small_grid_thw], dim=0).prod(dim=1).tolist())
        assert len(parts) % 2 == 0
        n = len(parts) // 2
        return [(parts[i], grid_thw[i], parts[n + i], small_grid_thw[i]) for i in range(n)]

    def forward(self, x, grid_thw, small_grid_thw, position_ids, visual_position_ids, draws: Optional[list] = None):
        memories, positions = [], []
        per_sample = zip(self._streams(x, grid_thw, small_grid_thw), torch.unbind(position_ids, dim=1), visual_position_ids)
        for b, ((full, thw, small, small_thw), position_id, visual_position_id) in enumerate(per_sample):
            d = None if draws is None else draws[b]
            tem_x, tem_thw, tem_weights, tem_timestamp, tem_indices = self.temporal_compress(small, small_thw,
                                                                                            self.temporal_length, draws=d)
            # timestamps are means of at most t integers: round-half-even on the host equals torch.round on fp32
            tem_positions = torch.from_numpy(np.round(tem_timestamp.float().cpu().numpy()).astype(np.int64)).to(full.device)
            if self.spatial_length > 0:
                spa_x, spa_thw, spa_positions = self.spatial_enhance(full, small, thw, tem_x, tem_thw, tem_weights,
                                                                     tem_positions, tem_indices, draws=d)
            else:
                spa_x, spa_thw, spa_positions = full[0:0], _with_t(thw, 0), torch.zeros(0, dtype=torch.long, device=full.device)
            memories.append(self.cat_spa_tem(spa_x=spa_x, tem_x=tem_x))
            positions.append(self.calc_am_rope(position_id, visual_position_id, tem_thw, tem_positions, spa_thw, spa_positions))
        return torch.stack(memories, dim=0), torch.stack(positions, dim=1)
