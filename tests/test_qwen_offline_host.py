"""CPU: the offline Qwen2-VL vision pass (VisualB200.forward, qwen/offline.py) — its chunk plan, its row budget, the
refusals it raises before touching a device, and the self-consistency of tests/golden/qwen_offline.npz (the reference's
own visual.forward, recorded by tests/golden/make_golden_qwen_offline.py)."""
import os

import numpy as np
import pytest
import torch

from flash_vstream_b200._lib import FvsError
from flash_vstream_b200.qwen import offline as OF
from flash_vstream_b200.qwen import vstream_qwen2vl_model as M
from flash_vstream_b200.qwen import vstream_qwen2vl_realtime as rt
from tests import qwen_offline_inputs as OI

G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "qwen_offline.npz")


# ------------------------------------------------------------------------------------------------ the chunk plan
@pytest.mark.parametrize("t,rows,budget", [(1, 64, 64), (7, 64, 64), (7, 64, 127), (7, 64, 128), (384, 256, 32768),
                                           (384, 1024, 32768), (30, 4784, 32768), (5, 16, 10 ** 6)])
def test_plan_covers_whole_patches_within_the_budget(t, rows, budget):
    plan = OF.plan_chunks(t, rows, budget)
    assert [p for p, _ in plan] == [sum(n for _, n in plan[:i]) for i in range(len(plan))]     # in order, no gap
    assert sum(n for _, n in plan) == t and all(n >= 1 for _, n in plan)
    assert all(n * rows <= budget for _, n in plan)
    assert all(n == budget // rows for _, n in plan[:-1])                                        # full chunks but the last
    if budget < 2 * rows:
        assert plan == [(p, 1) for p in range(t)]                                                # one patch a chunk


def test_plan_refuses_a_budget_below_one_patch():
    with pytest.raises(ValueError, match="smaller than one temporal patch"):
        OF.plan_chunks(3, 1024, 1023)


def test_default_budget_is_the_stated_workspace():
    """DESIGN.md §3.16: fvs_qwen_vit_workspace_bytes at the Qwen2-VL width is 16 E + 2 mlp + 4 bytes a row (seven
    buffers, each rounded up to 256 bytes); 32,768 rows stay under 1 GiB and hold 32 temporal patches at 32x32"""
    E, mlp, rows = 1280, 5120, OF.DEFAULT_MAX_ROWS
    per_row = 16 * E + 2 * mlp + 4
    assert per_row == 30724 and per_row * rows < 2 ** 30
    assert OF.plan_chunks(384, 1024, rows) == [(p, min(32, 384 - p)) for p in range(0, 384, 32)]


# ------------------------------------------------------------------------------------------------ the knob
@pytest.mark.parametrize("bad,exc", [(0, ValueError), (-4, ValueError), (True, TypeError), (1.5, TypeError),
                                     ("4096", TypeError), (None, TypeError)])
def test_max_rows_knob_is_validated(bad, exc):
    with pytest.raises(exc, match="offline_max_rows"):
        rt.VisualB200(rt.FlashMemory(), None, offline_max_rows=bad)


def test_max_rows_knob_default_and_value():
    assert rt.VisualB200(rt.FlashMemory(), None).offline_max_rows == OF.DEFAULT_MAX_ROWS
    assert rt.VisualB200(rt.FlashMemory(), None, offline_max_rows=np.int64(576)).offline_max_rows == 576


# ------------------------------------------------------------------------------------------------ refusals
def _never(*a, **k):
    raise AssertionError("the tower ran on a refused call")


def _call(fm_kw, grids, max_rows=OF.DEFAULT_MAX_ROWS, encode=_never):
    fm = M.FlashMemory(**fm_kw)
    visual = rt.VisualB200(fm, None, encode_patches=encode, offline_max_rows=max_rows)
    rows = sum(t * h * w for t, h, w in grids)
    pos, vis = torch.zeros(3, len(grids), 8, dtype=torch.long), torch.zeros(len(grids), 8, dtype=torch.long)
    return visual(torch.zeros(rows, 1176), torch.tensor(grids), pos, vis)


@pytest.mark.parametrize("fm_kw,grids,exc,match", [
    ({}, [(2, 6, 8)], NotImplementedError, "Performing temporal pool, pad_h > 0, pad_h=1"),
    ({}, [(2, 8, 8), (2, 8, 10)], NotImplementedError, "Performing temporal pool, pad_w > 0, pad_w=1"),
    (dict(flash_memory_temporal_poolsize=3), [(2, 8, 8)], AssertionError, ""),
    (dict(flash_memory_temporal_method="nope", flash_memory_temporal_length=2), [(2, 8, 8)], ValueError,
     "temporal_method should be one of"),
    (dict(flash_memory_temporal_method="merge", flash_memory_temporal_length=2), [(2, 8, 8)], NotImplementedError,
     "merge_feature"),
    (dict(flash_memory_spatial_method="nope", flash_memory_spatial_length=2), [(2, 8, 8)], ValueError,
     "spatial_method should be one of"),
])
def test_reference_refusals_before_the_tower(fm_kw, grids, exc, match):
    with pytest.raises(exc, match=match):
        _call(fm_kw, grids)


def test_unknown_methods_refused_only_where_the_reference_reaches_them():
    """the reference dispatches on the method only when the clip exceeds the memory: a short clip never reaches it"""
    with pytest.raises(FvsError, match="no CPU path"):             # past every check, at the first kernel
        _call(dict(flash_memory_temporal_method="nope", flash_memory_spatial_method="nope"), [(2, 8, 8)])


def test_budget_refusals():
    with pytest.raises(ValueError, match="smaller than one temporal patch"):
        _call({}, [(2, 8, 8)], max_rows=63)                        # the full-resolution pass needs 64 rows a patch
    with pytest.raises(FvsError, match="no CPU path"):             # no full-resolution pass: 16 rows a patch suffice
        _call(dict(flash_memory_spatial_length=0), [(2, 8, 8)], max_rows=16)
    with pytest.raises(ValueError, match="do not match grid_thw"):
        visual = rt.VisualB200(rt.FlashMemory(), None, encode_patches=_never)
        visual(torch.zeros(65, 1176), torch.tensor([[1, 8, 8]]), torch.zeros(3, 1, 8), torch.zeros(1, 8))


def test_no_tower_refused():
    with pytest.raises(NotImplementedError, match="no vision tower attached"):
        _call({}, [(2, 8, 8)], encode=None)


def test_image_branch_raises_like_the_reference():
    """FlashVStreamQwen2VLModel's image branch calls self.visual(pixel_values, grid_thw=...) without positions"""
    visual = rt.VisualB200(rt.FlashMemory(), None, encode_patches=_never)
    with pytest.raises(TypeError, match="missing 2 required positional arguments: 'position_ids' and 'visual_position_ids'"):
        visual(torch.zeros(64, 1176), grid_thw=torch.tensor([[1, 8, 8]]))


# ------------------------------------------------------------------------------------------------ the golden
@pytest.mark.parametrize("name", list(OI.GOLDEN_CASES))
def test_golden_is_self_consistent(name):
    g = np.load(G)
    videos = OI.GOLDEN_CASES[name]
    px = OI.pixels(videos, int(g[f"{name}_seed"]))
    assert (OI.checksum(px) == g[f"{name}_chk"]).all(), "seeded input drifted"
    fm = M.FlashMemory(**OI.GOLDEN_FM)
    S, T0 = fm.spatial_length, fm.temporal_length
    pos = g[f"{name}_pos"]
    n_vis = [OI.n_visual(grid, T0, S) for grid, _ in videos]
    assert pos.shape == (3, len(videos), OI.PREFIX + n_vis[0] + OI.SUFFIX)
    rows = 0
    for b, ((t, h, w), _) in enumerate(videos):
        picks, ts = g[f"{name}_v{b}_picks"], g[f"{name}_v{b}_ts"]
        assert len(picks) == min(t, S) and ((0 <= picks) & (picks < t)).all()
        assert len(ts) == min(t, T0) and (np.diff(ts) > 0).all()
        assert len(g[f"{name}_v{b}_init"]) == (T0 if t > T0 else 0)
        p, start = pos[:, b], OI.PREFIX
        n_dam, n_csm = min(t, S) * h * w // 4, min(t, T0) * h * w // 16
        # AM-RoPE: DAM tokens carry their frame's index, CSM tokens the rounded timestamp after the DAM block
        assert (p[0, start: start + n_dam] == start + np.repeat(picks, h * w // 4)).all()
        assert (p[0, start + n_dam: start + n_dam + n_csm] == start + n_dam + np.repeat(np.round(ts), h * w // 16)).all()
        assert (p[:, :start] == np.arange(start)).all()
        rows += (n_dam + n_csm)
    assert g[f"{name}_rows"].tolist() == [rows, OI.MERGER_OUT]
    e32 = torch.from_numpy(g[f"{name}_emb32"])
    e16 = torch.from_numpy(g[f"{name}_emb16"].view(np.int16)).view(torch.bfloat16).float()
    assert e32.shape == e16.shape == (len(range(rows)[OI.GOLDEN_ROWS]), OI.MERGER_OUT)
    assert float((e16 - e32).norm() / e32.norm()) < 2e-2          # the reference's bf16 run against its fp32 run
