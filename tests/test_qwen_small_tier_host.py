"""Half-resolution host tier of the Qwen2-VL streaming state, host side: the small_device_frames knob of the state, the
pool and the realtime host, the row ranges of a tiered klarge sweep, and the refusals of the tiered entry point (returned
before any CUDA call, nothing launched)."""
import ctypes as C
from types import SimpleNamespace

import numpy as np
import pytest
import torch

from flash_vstream_b200 import _lib as L
from flash_vstream_b200.qwen import ops as Q
from flash_vstream_b200.qwen import stream_state as SS
from flash_vstream_b200.qwen import vstream_qwen2vl_realtime as rt
from flash_vstream_b200.qwen.multistream import QwenStreamPool
from flash_vstream_b200.qwen.vision_tower import QwenVisionBlocksB200

A = 0x10000          # a 16-byte aligned stand-in address: the refusals happen before anything is dereferenced


def _host():
    return rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(rt.FlashMemory(), None))


def _pool(**kw):
    tower = QwenVisionBlocksB200.__new__(QwenVisionBlocksB200)          # passes the type check; never called here
    model = SimpleNamespace(visual=rt.VisualB200(rt.FlashMemory(), None, encode_patches=tower, device="cuda:0"))
    return QwenStreamPool(model, **kw)


# ------------------------------------------------------------------------------------------------ the knob
@pytest.mark.parametrize("good", [None, 0, 1, 12, np.int64(7)])
def test_knob_values(good):
    want = None if good is None else int(good)
    st = SS.QwenStreamState(rt.FlashMemory(), None, small_device_frames=good)
    assert st.small_device_frames == want and st.device_frames is None
    assert _pool(small_device_frames=good).small_device_frames == want
    host = _host()
    host.fvs_bank_small_device_frames = good
    assert host._bank_small_device_frames() == want


def test_knob_defaults():
    assert SS.QwenStreamState(rt.FlashMemory(), None).small_device_frames is None
    assert _pool().small_device_frames is None
    assert _host().fvs_bank_small_device_frames is None


@pytest.mark.parametrize("bad", [-1, 1.5, "4", True, False, [3]])
def test_knob_is_validated(bad):
    with pytest.raises(ValueError, match="small_device_frames"):
        SS.QwenStreamState(rt.FlashMemory(), None, small_device_frames=bad)
    with pytest.raises(ValueError, match="small_device_frames"):
        _pool(small_device_frames=bad)
    host = _host()
    host.fvs_bank_small_device_frames = bad
    with pytest.raises(ValueError, match="fvs_bank_small_device_frames"):        # before the tower runs
        host.embed_new_video_clip(torch.zeros(4 * 1176), torch.tensor([[1, 2, 2]]), 0)


def test_knob_change_mid_stream_is_refused():
    """a host with a stream in progress refuses a different half-resolution cap; the same cap, or a new stream, is
    accepted; the two caps are checked independently"""
    host = _host()
    host.stream_state = SimpleNamespace(n_frames=4, device_frames=None, small_device_frames=None)
    host.video_embedding_memory[:] = [0]
    host.fvs_bank_small_device_frames = 8
    with pytest.raises(ValueError, match="fvs_bank_small_device_frames changed from None to 8 in the middle"):
        host._bank_small_device_frames()
    assert host._bank_device_frames() is None
    host.fvs_bank_small_device_frames = None
    assert host._bank_small_device_frames() is None
    host.fvs_bank_small_device_frames = 0
    host.init_streaming()
    assert host._bank_small_device_frames() == 0


# ------------------------------------------------------------------------------------------------ the range plan
@pytest.mark.parametrize("t", [1, 2, 7, 12, 25])
@pytest.mark.parametrize("F", [1, 3, 4, 728])
def test_plan_covers_every_row_once(t, F):
    for n_dev in sorted({0, 1, t - 1, t, t + 1, t + 40}):
        plan = Q.klarge_plan(t, n_dev, F)
        seen = []
        for c, first, rows in plan:
            assert rows > 0
            if c < 0:
                assert first == 0 and rows == min(n_dev, t)
            else:                                   # chunk c holds rows n_dev + c*F + [0, F), read from its start
                assert first == n_dev + c * F and rows <= F
            seen += range(first, first + rows)
        assert seen == list(range(t)), (t, F, n_dev, plan)
        chunks = [c for c, _, _ in plan if c >= 0]
        assert chunks == list(range(len(chunks))) and len(chunks) == -(-max(0, t - n_dev) // F)
        assert sum(1 for c, _, _ in plan if c < 0) == (1 if n_dev > 0 else 0)


def test_plan_cases():
    assert Q.klarge_plan(5, 5, 2) == [(-1, 0, 5)]
    assert Q.klarge_plan(5, 9, 2) == [(-1, 0, 5)]
    assert Q.klarge_plan(5, 0, 2) == [(0, 0, 2), (1, 2, 2), (2, 4, 1)]
    assert Q.klarge_plan(6, 1, 2) == [(-1, 0, 1), (0, 1, 2), (1, 3, 2), (2, 5, 1)]
    assert SS.chunk_frames(144 * 1280 * 2) == 728            # 24x24 half-resolution frames in one 256 MiB chunk


# ------------------------------------------------------------------------------------------------ the C entry point
def test_symbol_exported():
    lib = L.load()
    assert hasattr(lib, "fvs_qwen_klarge_retrieve_tiered") and "fvs_qwen_klarge_retrieve_tiered" in L.SIGNATURES


def _tiered(chunks=(A, A, A), **kw):
    a = dict(tem_x=A, klarge_idx=A, dev_bank=A, n_dev=4, host_chunks=None, chunk_frames=3, k=2, t_total=10, PD=1024,
             dtype=L.BF16, metric=L.KLARGE_EUCLIDEAN, idx_out=A, dist_out=None, workspace=A, workspace_bytes=1 << 30,
             stream=None)
    a.update(kw)
    if "host_chunks" not in kw and chunks is not None:
        a["host_chunks"] = (C.c_void_p * len(chunks))(*chunks)
    return L.load().fvs_qwen_klarge_retrieve_tiered(*a.values())


@pytest.mark.parametrize("kw, msg", [
    (dict(n_dev=11), "n_dev"),
    (dict(n_dev=-1), "n_dev"),
    (dict(chunks=None), "chunk table"),
    (dict(chunk_frames=0), "chunk table"),
    (dict(chunks=(A, None, A)), "host chunk 1"),
    (dict(chunks=(A, A, None), n_dev=1), "host chunk 2"),
    (dict(dev_bank=None), "null pointer"),
    (dict(k=65), "0 < k <= 64"),
    (dict(t_total=0, n_dev=0), "0 < k <= 64"),
    (dict(PD=1000), "multiple of"),
    (dict(dtype=L.F32), "dtype"),
    (dict(metric=7), "metric"),
    (dict(workspace_bytes=16), "workspace"),
])
def test_tiered_refusals_launch_nothing(kw, msg):
    lib = L.load()
    before = lib.fvs_launch_count()
    assert _tiered(**kw) == L.FVS_EINVAL
    err = lib.fvs_last_error().decode()
    assert msg in err and err.startswith("fvs_qwen_klarge_retrieve_tiered"), err
    assert lib.fvs_launch_count() == before


def test_tiered_accepts_what_it_needs():
    """host rows need exactly ceil((t - n_dev) / F) chunk pointers; no device rows need no device pointer; no host rows
    need no chunk table (refused here only by the workspace check, which comes after them)"""
    assert _tiered(chunks=(A, A, A, None), n_dev=1, workspace_bytes=16) == L.FVS_EINVAL
    assert "workspace" in L.load().fvs_last_error().decode()
    assert _tiered(chunks=(A, A, A, A), dev_bank=None, n_dev=0, workspace_bytes=16) == L.FVS_EINVAL
    assert "workspace" in L.load().fvs_last_error().decode()
    assert _tiered(chunks=None, n_dev=10, chunk_frames=0, workspace_bytes=16) == L.FVS_EINVAL
    assert "workspace" in L.load().fvs_last_error().decode()
