"""CPU tests of QwenStreamPool's host logic (DESIGN.md §3.15): how a round's clips are laid out over tower calls, rounds
refused before anything is enqueued, and the completion half of a stream's step drawing from the stream's own source."""
import random

import pytest
import torch

from flash_vstream_b200.draws import DrawSource
from flash_vstream_b200.qwen.multistream import MAX_GRIDS, QwenStreamPool, _Stream, plan_tower_calls
from flash_vstream_b200.qwen.stream_state import QwenStreamState
from flash_vstream_b200.qwen.vision_tower import QwenVisionBlocksB200
from flash_vstream_b200.qwen.vstream_qwen2vl_realtime import FlashMemory, VisualB200


def segs(t, h, w):
    return [(t, h, w), (t, h // 2, w // 2)]


def check_plan(clips, plan, max_rows):
    seen = set()
    for grids, places in plan:
        keys = [(h, w) for _, h, w in grids]
        assert len(keys) == len(set(keys)) <= MAX_GRIDS
        rows = sum(t * h * w for t, h, w in grids)
        assert rows <= max_rows or len(places) == 1
        spans = []
        for i, offs in places:
            assert i not in seen
            seen.add(i)
            for (t, h, w), off in zip(clips[i], offs):
                spans.append((off, off + t * h * w, (h, w)))
        spans.sort()
        assert spans[0][0] == 0 and spans[-1][1] == rows                  # the call's rows, tiled without gaps
        assert all(a[1] == b[0] for a, b in zip(spans, spans[1:]))
        r = 0
        for t, h, w in grids:                                            # each grid entry is one contiguous block
            block = [s for s in spans if s[2] == (h, w)]
            assert block[0][0] == r and sum(e - s for s, e, _ in block) == t * h * w
            r += t * h * w
    assert seen == set(range(len(clips)))


def test_same_grid_clips_merge_into_one_entry():
    clips = [segs(1, 24, 24), segs(8, 24, 24), segs(2, 24, 24), segs(1, 24, 36)]
    plan = plan_tower_calls(clips, 1 << 20)
    check_plan(clips, plan, 1 << 20)
    assert len(plan) == 1
    grids, places = plan[0]
    assert sorted(grids) == sorted([(11, 24, 24), (11, 12, 12), (1, 24, 36), (1, 12, 18)])
    offs = dict(places)
    assert offs[0][0] < offs[1][0] < offs[2][0]                          # the clips of a grid entry in round order


def test_at_most_16_grids_per_call():
    clips = [segs(1, 8, 8 * k) for k in range(1, 10)] + [segs(2, 8, 8)]   # 18 distinct (h, w)
    plan = plan_tower_calls(clips, 1 << 20)
    check_plan(clips, plan, 1 << 20)
    assert len(plan) == 2 and all(len(g) <= MAX_GRIDS for g, _ in plan)
    assert sum(len(p) for _, p in plan) == len(clips)


def test_row_budget_splits_calls():
    clips = [segs(t, 24, 24) for t in (1, 2, 8, 1, 1, 8, 3)]
    for budget in (720, 1500, 6000, 10 ** 6):
        plan = plan_tower_calls(clips, budget)
        check_plan(clips, plan, budget)
        if budget == 720:
            assert len(plan) == len(clips)
    big = [segs(8, 24, 24)]
    plan = plan_tower_calls(big, 100)                                   # a clip over the budget goes alone
    assert len(plan) == 1 and plan[0][0] == [(8, 24, 24), (8, 12, 12)]


def test_random_rounds_tile_their_calls():
    r = random.Random(3)
    shapes = [(8, 8), (8, 16), (16, 8), (24, 24), (24, 36), (12, 72), (4, 4), (8, 72)]
    for _ in range(50):
        clips = [segs(r.choice([1, 2, 8]), *r.choice(shapes)) for _ in range(r.randint(1, 40))]
        budget = r.choice([500, 3000, 20000, 1 << 20])
        check_plan(clips, plan_tower_calls(clips, budget), budget)


# ------------------------------------------------------------------------------------------------ the pool on the host
def _tower_stub():
    return QwenVisionBlocksB200.__new__(QwenVisionBlocksB200)          # passes the type check; never called here


class _Host:
    def __init__(self, visual):
        self.visual = visual


def test_refused_configs_name_the_knob():
    with pytest.raises(NotImplementedError, match="encode_patches"):
        QwenStreamPool(_Host(VisualB200(FlashMemory(), None, encode_patches=lambda x, g: x)))
    with pytest.raises(NotImplementedError, match="flash_memory_temporal_method"):
        QwenStreamPool(_Host(VisualB200(FlashMemory(flash_memory_temporal_method="sample"), None,
                                        encode_patches=_tower_stub())))
    with pytest.raises(NotImplementedError, match="flash_memory_temporal_poolsize"):
        QwenStreamPool(_Host(VisualB200(FlashMemory(flash_memory_temporal_poolsize=1), None,
                                        encode_patches=_tower_stub())))
    with pytest.raises(ValueError, match="device_frames"):
        QwenStreamPool(_Host(VisualB200(FlashMemory(), None, encode_patches=_tower_stub(), device="cuda:0")),
                       device_frames=-1)


def _cpu_pool(n_streams):
    """a pool whose tower records its calls, with streams made by hand (open() needs a CUDA device for the generators)"""
    pool = QwenStreamPool.__new__(QwenStreamPool)
    flash = FlashMemory(flash_memory_temporal_length=8, flash_memory_spatial_length=6)
    pool.visual = VisualB200(flash, None, encode_patches=None, device="cpu")
    pool.flash, pool.merger, pool.device = flash, None, torch.device("cuda", 0)
    calls = []
    pool.tower = lambda *a: calls.append(a)
    pool._streams = {}
    for sid in range(n_streams):
        st = QwenStreamState(flash, None)
        st.rng = DrawSource(sid, "cpu")
        pool._streams[sid] = _Stream(pool.visual, st)
    return pool, calls


def _clip(t, h, w):
    return torch.zeros(t * h * w, 1176), torch.tensor([[t, h, w]])


@pytest.mark.parametrize("bad, exc", [
    (_clip(1, 8, 8)[0], ValueError),                                      # pixels of another grid
    ((torch.zeros(1 * 8 * 8, 1176), torch.tensor([[1, 8, 8], [1, 8, 8]])), ValueError),   # two clips for one stream
    (_clip(1, 6, 8), NotImplementedError),                                # h / 2 odd: temporal_pool's padding rule
    (_clip(1, 8, 10), NotImplementedError),                               # w / 2 odd
    (_clip(1, 7, 8), ValueError),                                         # odd grid side
    (_clip(0, 8, 8), ValueError),
])
def test_refused_round_enqueues_nothing(bad, exc):
    pool, calls = _cpu_pool(3)
    if isinstance(bad, torch.Tensor):
        bad = (bad, torch.tensor([[1, 16, 8]]))
    g_torch, g_py = torch.get_rng_state(), random.getstate()
    snaps = {sid: s.stream_state.rng.snapshot() for sid, s in pool._streams.items()}
    with pytest.raises(exc):
        pool.step({0: _clip(2, 8, 8), 1: bad, 2: _clip(1, 8, 8)})
    assert not calls
    for sid, s in pool._streams.items():
        st = s.stream_state
        assert st.n_frames == 0 and st.steps == 0 and st.grid is None and st._pending is None
        a, b = snaps[sid], st.rng.snapshot()
        assert torch.equal(a[0], b[0]) and a[2] == b[2]
    assert torch.equal(torch.get_rng_state(), g_torch) and random.getstate() == g_py


def test_grid_must_match_the_stream_and_sids_must_exist():
    pool, calls = _cpu_pool(2)
    pool._streams[1].stream_state.grid = (16, 16)
    with pytest.raises(ValueError, match="differs from the stream's grid"):
        pool.step({0: _clip(1, 8, 8), 1: _clip(1, 8, 8)})
    with pytest.raises(KeyError):
        pool.step({0: _clip(1, 8, 8), 7: _clip(1, 8, 8)})
    assert not calls


# ------------------------------------------------------------------------------------------------ the completion half
def _enqueued(st, T, n_unique, consumed, empty, own=True):
    """a state as enqueue() leaves it on the fast path, with the read-back as the device would have written it"""
    st._readback = torch.tensor([n_unique, 3, consumed, 1, 0, empty, 0, 0], dtype=torch.int32)
    st._pending = dict(cand=None, cand_w=None, T=T, d={}, start_idx=0, t=1, snap=st.rng.snapshot("cpu"),
                       own_refills=own)


def test_completion_draws_from_the_stream_source_only():
    flash = FlashMemory(flash_memory_temporal_length=8)
    g_torch, g_py = torch.get_rng_state(), random.getstate()
    st = QwenStreamState(flash, None)
    st.rng = DrawSource(11, "cpu")
    twin = random.Random(11)
    _enqueued(st, 6, 6, 5, 0)
    st.complete()
    for _ in range(5):
        twin.randint(0, 5)
    assert st.rng.py.getstate() == twin.getstate() and st.fast_steps == 1 and st.steps == 1
    # duplicates among the rows: this stream's source is rewound, and the clip is redone through the synchronous path
    redo = []
    st._compress_sync = lambda *a: redo.append(a)
    snap = st.rng.snapshot("cpu")
    st.rng.randperm(6, "cpu")                                            # the fast path's randperm(T)
    _enqueued(st, 6, 5, 2, 0)
    st._pending["snap"] = snap
    st.complete()
    assert len(redo) == 1 and st.redone_steps == 1 and st.steps == 2 and torch.equal(st.rng.cpu, snap[0])
    assert st.rng.py.getstate() == twin.getstate()
    assert torch.equal(torch.get_rng_state(), g_torch) and random.getstate() == g_py


def test_empty_cluster_leaves_the_stream_unfinished():
    flash = FlashMemory(flash_memory_temporal_length=8)
    st = QwenStreamState(flash, None)
    st.rng = DrawSource(2, "cpu")
    py = st.rng.py.getstate()
    _enqueued(st, 6, 6, 3, 1)
    with pytest.raises(ZeroDivisionError):
        st.complete()
    assert st.steps == 0 and st.fast_steps == 0 and st.rng.py.getstate() == py and st._pending is None


def test_round_completes_every_stream_then_names_the_failing_ones():
    pool, _ = _cpu_pool(4)
    for sid, s in pool._streams.items():
        _enqueued(s.stream_state, 6, 6, 1, int(sid in (1, 3)))
    with pytest.raises(ZeroDivisionError, match=r"\[1, 3\]") as ei:
        pool._complete([0, 1, 2, 3])
    assert set(ei.value.errors) == {1, 3}
    assert [s.stream_state.steps for s in pool._streams.values()] == [1, 0, 1, 0]
    assert all(s.stream_state._pending is None for s in pool._streams.values())
