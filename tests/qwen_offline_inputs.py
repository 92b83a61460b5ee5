"""Seeded inputs of the offline Qwen2-VL vision pass (visual.forward): a small tower, a merger, scene-structured pixel
clips and the LLM-side position ids.  Shared by tests/golden/make_golden_qwen_offline.py and the tests."""
from __future__ import annotations

import torch

from tests import qwen_vit_inputs as VI
from tests.golden_inputs import _gen, checksum  # noqa: F401
from tests.qwen_inputs import DT

TOWER = dict(depth=2, embed=1280, heads=16, seed=97)
MERGER_OUT = 256                       # PatchMerger(dim=256, context_dim=1280): dims fvs_linear admits
# the golden's memory: 4 CSM centroids, 2 DAM frames (lengths count LLM tokens of two temporal patches each)
GOLDEN_FM = dict(flash_memory_temporal_length=8, flash_memory_temporal_method='kmeans_ordered',
                 flash_memory_temporal_poolsize=2, flash_memory_temporal_pca_dim=32, flash_memory_spatial_length=4,
                 flash_memory_spatial_method='klarge_retrieve')
# name -> (grid, scene lengths) of every video of one call.  t=3: DAM retrieval without k-means; t=7: both; a 12x8 grid;
# a batch of two lengths whose memories have the same size (the reference stacks them).  The scenes keep two-member
# clusters out of the DAM's heaviest centroids: a centroid of two frames is equidistant from both, an exact tie.
GOLDEN_CASES = {
    "t3": [((3, 8, 8), (1, 1, 1))],
    "t7": [((7, 8, 8), (4, 1, 1, 1))],
    "t8_12x8": [((8, 12, 8), (3, 1, 3, 1))],
    "batch_t6_t9": [((6, 8, 8), (3, 1, 1, 1)), ((9, 8, 8), (3, 1, 3, 2))],
}
GOLDEN_ROWS = slice(None, None, 3)     # the golden keeps every third row of video_embeds
PREFIX, SUFFIX = 5, 3


def tower_state_dict(dtype="bf16"):
    return VI.state_dict(TOWER, dtype)


def merger_weights(dtype="bf16", seed=98, out=MERGER_OUT, context=1280):
    """ln_q / mlp[0] / mlp[2] of a transformers PatchMerger, rounded to `dtype`"""
    g = _gen(seed)
    dt, hid = DT[dtype], 4 * context
    rn = lambda *s, scale=1.0: (torch.randn(*s, generator=g) * scale).to(dt)
    return {"ln_q.weight": (1 + 0.1 * torch.randn(context, generator=g)).to(dt), "ln_q.bias": rn(context, scale=0.05),
            "mlp.0.weight": rn(hid, hid, scale=hid ** -0.5), "mlp.0.bias": rn(hid, scale=0.05),
            "mlp.2.weight": rn(out, hid, scale=hid ** -0.5), "mlp.2.bias": rn(out, scale=0.05)}


def clip_pixels(t, h, w, seed, dtype="bf16", scenes=None):
    """[t*h*w, 1176] patch rows of a clip of consecutive scenes of the given lengths (default: t random scenes).  The
    j-th temporal patch of a scene is the scene plus noise of amplitude 0.05 + 0.1 j, so the members of a cluster sit at
    clearly different distances from its centroid: the k-means and the retrieval have margins far above the tower's
    16-bit rounding, and a 16-bit run picks what the fp32 run picks."""
    g = _gen(seed)
    scenes = scenes or (1,) * t
    assert sum(scenes) == t
    base = torch.randn(len(scenes), h * w, 1176, generator=g) * 1.2
    which = torch.repeat_interleave(torch.arange(len(scenes)), torch.tensor(scenes))
    amp = torch.cat([0.05 + 0.1 * torch.arange(n) for n in scenes])
    x = base[which] + amp.view(t, 1, 1) * torch.randn(t, h * w, 1176, generator=g)
    return x.reshape(-1, 1176).to(DT[dtype])


def pixels(videos, seed, dtype="bf16"):
    """the patch rows of one call: videos is [(grid, scene lengths | None)]"""
    return torch.cat([clip_pixels(*grid, seed + 17 * i, dtype, scenes) for i, (grid, scenes) in enumerate(videos)])


def n_visual(grid, temporal_length, spatial_length, pool=2):
    """LLM tokens of one video's memory: DAM frames at full resolution, CSM frames at the pooled one, 4 rows a token"""
    t, h, w = grid
    hs, ws = (h // 2, w // 2) if pool > 1 else (h, w)
    return (min(t, spatial_length) * h * w + min(t, temporal_length) * hs * ws) // 4


def positions(n_vis, prefix=PREFIX, suffix=SUFFIX):
    """(position_ids [3, B, L], visual_position_ids [B, L]) of B sequences with n_vis visual tokens each (one length)"""
    assert len(set(n_vis)) == 1, "the reference stacks the memories: one visual length per call"
    B, n = len(n_vis), n_vis[0]
    L = prefix + n + suffix
    pos = torch.arange(L).view(1, 1, L).expand(3, B, L).clone()
    vis = torch.full((B, L), -1, dtype=torch.long)
    vis[:, prefix: prefix + n] = torch.arange(n)
    return pos, vis
