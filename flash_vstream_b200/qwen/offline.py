"""The offline vision pass of the Qwen2-VL family on sm_90a: FlashVStreamQwen2VisionTransformerPretrainedModel.forward
(Flash-VStream-Qwen/models/vstream_qwen2vl_model.py:388-428), the call FlashVStreamQwen2VLModel.forward makes with
pixel_values_videos (:528-530) and that the evaluation drivers go through.  VisualB200.forward delegates here.

Same inputs, outputs and draws as the reference (temporal_pool, the tower, FlashMemory.forward, the PatchMerger), with two
differences that change no bit (DESIGN.md §3.16):
  * the tower runs per sample and per resolution in chunks of whole temporal patches of at most `max_rows` rows, so its
    workspace and activations are bounded by the row budget and not by the video length;
  * the full-resolution tower runs only on the frames the Flash Memory keeps.  The DAM picks come from the half-resolution
    bank and the CSM alone, so they are known before any full-resolution frame is encoded; the tower's attention never
    crosses a temporal patch, so a frame encoded alone has the bits it has inside the whole video.  For 384 temporal
    patches at 32x32 with spatial_length 60 that is 129,024 tower rows instead of 491,520.
"""
from __future__ import annotations

from typing import Callable, List, Optional, Sequence, Tuple

import numpy as np
import torch

from .. import ops as O
from . import compress_functions as CF
from . import ops as Q
from . import vstream_qwen2vl_model as _offline

PATCH_DIM = 3 * 2 * 14 * 14
# 32,768 tower rows per call: fvs_qwen_vit_workspace_bytes is 16*E + 2*mlp + 4 bytes a row (plus 256-byte alignment of
# its seven buffers), 30,724 B at the Qwen2-VL width (E 1280, mlp 5120), so one call's workspace is 0.94 GiB; the output
# and the pooled pixels of the chunk add 4,912 B a row.  That is 32 full-resolution temporal patches at 32x32.
DEFAULT_MAX_ROWS = 32768


def check_max_rows(max_rows) -> int:
    """the validated row budget: an int >= 1"""
    if isinstance(max_rows, bool) or not isinstance(max_rows, (int, np.integer)):
        raise TypeError(f"offline_max_rows must be an int, got {type(max_rows).__name__}")
    if max_rows < 1:
        raise ValueError(f"offline_max_rows must be >= 1, got {max_rows}")
    return int(max_rows)


def plan_chunks(t: int, rows_per_patch: int, max_rows: int) -> List[Tuple[int, int]]:
    """(first temporal patch, patches) of each tower call over t patches of rows_per_patch rows: whole patches only,
    in order, at most max_rows rows a call"""
    if rows_per_patch > max_rows:
        raise ValueError(f"offline_max_rows={max_rows} is smaller than one temporal patch ({rows_per_patch} rows): "
                         f"the tower never splits a temporal patch")
    per = max_rows // rows_per_patch
    return [(p, min(per, t - p)) for p in range(0, t, per)]


def _refuse(fm, grids: Sequence[Tuple[int, int, int]], rows: int, encode, max_rows: int):
    """Every refusal of the reference's forward, in the order it would reach them, plus the row budget — raised before
    anything is enqueued or drawn."""
    if rows != sum(t * h * w for t, h, w in grids):
        raise ValueError(f"pixel rows {rows} do not match grid_thw {list(grids)}")
    pool = fm.temporal_poolsize
    if pool > 1:
        for t, h, w in grids:                                    # FlashMemory.temporal_pool (:113-142)
            assert pool == 2
            for name, side in (("pad_h", h), ("pad_w", w)):
                if (side // 2) % 2:
                    raise NotImplementedError(f"Performing temporal pool, {name} > 0, {name}={(side // 2) % 2}")
    if encode is None:
        raise NotImplementedError("no vision tower attached: pass encode_patches=QwenVisionBlocksB200(...) (the sm_90a "
                                  "blocks of vstream_qwen2vl_model.py:416-425)")
    for t, h, w in grids:
        sh, sw = (h // 2, w // 2) if pool > 1 else (h, w)
        plan_chunks(t, sh * sw, max_rows)
        if pool > 1 and fm.spatial_length > 0:                   # the full-resolution pass runs too
            plan_chunks(min(t, fm.spatial_length), h * w, max_rows)
        if t > fm.temporal_length:                               # FlashMemory.temporal_compress (:145-179)
            assert sh % 2 == 0
            assert sw % 2 == 0
            if fm.temporal_length > 0:
                method = fm.temporal_method
                if method not in _offline._TEMPORAL_METHODS:
                    raise ValueError(f"temporal_method should be one of {_offline._TEMPORAL_METHODS}")
                if method not in ("sample", "kmeans_ordered", "fast_kmeans_ordered"):
                    getattr(CF, _offline._ALTERNATE_TEMPORAL[method])()      # raises the alternate's NotImplementedError
        if 0 < fm.spatial_length < t and fm.spatial_method not in _offline._SPATIAL_METHODS:
            raise ValueError(f"spatial_method should be one of {_offline._SPATIAL_METHODS}")


def encode_chunked(encode: Callable, rows_of: Callable, t: int, h: int, w: int, max_rows: int) -> torch.Tensor:
    """[t*h*w, E]: the tower over t temporal patches of (h, w), one call per plan_chunks chunk; rows_of(p, n) gives the
    patch rows of temporal patches [p, p + n)"""
    chunks = plan_chunks(t, h * w, max_rows)
    out = None
    for p, n in chunks:
        y = encode(rows_of(p, n), [(n, h, w)])
        if len(chunks) == 1:
            return y
        if out is None:
            out = y.new_empty(t * h * w, y.shape[-1])
        out[p * h * w: (p + n) * h * w].copy_(y)
    return out


def forward(visual, hidden_states: torch.Tensor, grid_thw: torch.Tensor, position_ids: torch.Tensor,
            visual_position_ids: torch.Tensor, draws: Optional[list] = None, max_rows: int = DEFAULT_MAX_ROWS):
    """(video_embeds [sum of merged memory rows, hidden], position_ids) of `visual` (a VisualB200) — the reference's
    return value.  draws: None (the global generators, like the reference) or one FlashMemory draws dict per sample."""
    fm, encode = visual.flash_memory, visual.encode_patches
    grids = [tuple(int(v) for v in g) for g in grid_thw.tolist()]
    x = hidden_states.view(-1, PATCH_DIM)
    _refuse(fm, grids, x.shape[0], encode, max_rows)
    memories, positions, st = [], [], 0
    per_sample = zip(grids, grid_thw, torch.unbind(position_ids, dim=1), visual_position_ids)
    for b, ((t, h, w), thw, position_id, visual_position_id) in enumerate(per_sample):
        hw = h * w
        px = x[st: st + t * hw]
        st += t * hw
        d = None if draws is None else draws[b]
        # half-resolution bank (or, without a second resolution, the full-resolution bank that serves as both)
        if fm.temporal_poolsize > 1:
            small_thw = _offline._like(thw, (t, h // 2, w // 2))
            small = encode_chunked(encode, lambda p, n: Q.temporal_pool(px[p * hw: (p + n) * hw], n, h, w),
                                   t, h // 2, w // 2, max_rows)
        else:
            small_thw = thw
            small = encode_chunked(encode, lambda p, n: px[p * hw: (p + n) * hw], t, h, w, max_rows)
        # the offline temporal_compress (a realtime FlashMemory overrides it with the carried-weights form)
        tem_x, tem_thw, tem_weights, tem_timestamp, tem_indices = _offline.FlashMemory.temporal_compress(
            fm, small, small_thw, fm.temporal_length, draws=d)
        tem_positions = torch.from_numpy(np.round(tem_timestamp.float().cpu().numpy()).astype(np.int64)).to(small.device)
        if fm.spatial_length == 0:
            spa_x, spa_thw = small[0:0], _offline._with_t(thw, 0)
            spa_positions = torch.zeros(0, dtype=torch.long, device=small.device)
        elif fm.temporal_poolsize == 1:
            spa_x, spa_thw, spa_positions = fm.spatial_enhance(small, small, thw, tem_x, tem_thw, tem_weights,
                                                               tem_positions, tem_indices, draws=d)
        else:
            spa_positions = fm.spatial_picks(small, t, tem_x, tem_thw, tem_weights, tem_positions, draws=d)
            if t <= fm.spatial_length:                           # the whole bank is the DAM memory
                spa_x = encode_chunked(encode, lambda p, n: px[p * hw: (p + n) * hw], t, h, w, max_rows)
            else:                                                # only the picked frames, in pick order, repeats included
                frames = px.view(t, hw * PATCH_DIM)
                spa_x = encode_chunked(encode, lambda p, n: O.gather_rows(frames, spa_positions[p: p + n]).view(-1, PATCH_DIM),
                                       fm.spatial_length, h, w, max_rows)
            spa_thw = _offline._with_t(thw, min(t, fm.spatial_length))
        memories.append(fm.cat_spa_tem(spa_x=spa_x, tem_x=tem_x))
        positions.append(fm.calc_am_rope(position_id, visual_position_id, tem_thw, tem_positions, spa_thw, spa_positions))
    return visual.merger(torch.stack(memories, dim=0)), torch.stack(positions, dim=1)
