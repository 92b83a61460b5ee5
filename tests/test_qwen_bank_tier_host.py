"""Two-tier feature bank of the Qwen2-VL streaming state, host side: the exported gather (a one-job table), its
refusals (returned before any CUDA call, nothing launched), where every frame lands, and the fvs_bank_device_frames
knob."""
import ctypes as C

import pytest
import torch

from flash_vstream_b200 import _lib as L
from flash_vstream_b200.qwen import stream_state as SS
from flash_vstream_b200.qwen import vstream_qwen2vl_realtime as rt

A = 0x10000          # a 16-byte aligned stand-in address: the refusals happen before anything is dereferenced


def test_gather_symbols_exported():
    lib = L.load()
    for name in ("fvs_qwen_dam_gather_multi", "fvs_host_device_ptr"):
        assert hasattr(lib, name) and name in L.SIGNATURES


def _gather(dtype=L.BF16, **kw):
    a = dict(picks=A, n=4, n_frames=10, dev_x=A, dev_merged=A, n_dev=4, host_chunks=A, chunk_frames=3, prev_picks=A, m=2,
             prev_x=A, prev_merged=A, x_frame_elems=64, merged_frame_elems=32, spa_x_out=A, merged_out=A, host_fetches=A,
             n_base=10)
    a.update(kw)
    return L.load().fvs_qwen_dam_gather_multi((L.QwenGatherJob * 1)(L.QwenGatherJob(**a)), 1, dtype, None)


@pytest.mark.parametrize("kw, msg", [
    (dict(picks=None), "null picks"),
    (dict(n=0), "0 < n"),
    (dict(n=70000), "0 < n"),
    (dict(dtype=L.F32), "dtype"),
    (dict(spa_x_out=None, merged_out=None), "no output"),
    (dict(n_dev=11), "n_dev"),
    (dict(n_frames=0, n_dev=0), "n_dev"),
    (dict(n_dev=-1), "n_dev"),
    (dict(x_frame_elems=0), "frame sizes"),
    (dict(x_frame_elems=60), "16 bytes"),
    (dict(merged_frame_elems=0), "merged_out without"),
    (dict(dev_x=None), "device tier"),
    (dict(dev_merged=None), "device tier"),
    (dict(host_chunks=None), "chunk table"),
    (dict(chunk_frames=0), "chunk table"),
    (dict(prev_picks=None), "previous DAM"),
    (dict(prev_merged=None), "previous DAM"),
    (dict(m=-1), "previous DAM"),
    (dict(spa_x_out=A + 8), "aligned"),
    (dict(picks=A + 4), "8-byte"),
])
def test_gather_table_refusals_launch_nothing(kw, msg):
    lib = L.load()
    before = lib.fvs_launch_count()
    assert _gather(**kw) == L.FVS_EINVAL
    assert msg in lib.fvs_last_error().decode()
    assert lib.fvs_launch_count() == before


def test_host_device_ptr_refuses_null():
    out = C.c_void_p()
    assert L.load().fvs_host_device_ptr(None, C.byref(out)) == L.FVS_EINVAL


def _where(frame, cap, F):
    """the reference placement of one frame"""
    if cap is None or frame < cap:
        return (-1, frame)
    return divmod(frame - cap, F)


@pytest.mark.parametrize("cap", [None, 0, 1, 4, 5, 7, 9, 12, 100])
@pytest.mark.parametrize("F", [1, 3, 4])
def test_placement_frame_by_frame(cap, F):
    """clips of 1-3 frames appended in order: every frame lands where the tier rule says, spans are maximal within a chunk
    and cover each clip exactly once (caps inside a clip and at chunk edges included)"""
    n0 = 0
    for t in [1, 3, 2, 3, 1, 2, 3, 3, 1, 2]:
        spans = SS.placement(n0, t, cap, F)
        got = {}
        for c, dst, s, cnt in spans:
            assert cnt > 0 and (c < 0 or dst + cnt <= F)
            for k in range(cnt):
                got[s + k] = (c, dst + k) if c >= 0 else (-1, dst + k)
        assert sorted(got) == list(range(t))
        for s in range(t):
            assert got[s] == _where(n0 + s, cap, F), (n0, t, s)
        assert len(spans) == len({c for c, *_ in spans})         # one span per tier / chunk
        n0 += t


def test_placement_cases():
    assert SS.placement(0, 3, None, 2) == [(-1, 0, 0, 3)]
    assert SS.placement(4, 3, 5, 2) == [(-1, 4, 0, 1), (0, 0, 1, 2)]          # the cap inside a clip
    assert SS.placement(5, 3, 5, 2) == [(0, 0, 0, 2), (1, 0, 2, 1)]           # a clip across a chunk edge
    assert SS.placement(7, 1, 5, 2) == [(1, 0, 0, 1)]                         # the first frame of a chunk
    assert SS.placement(0, 2, 0, 4) == [(0, 0, 0, 2)]


def test_chunk_frames():
    assert SS.chunk_frames(2_506_752) == (1 << 28) // 2_506_752 == 107      # 24x24 x + merged rows in 256 MiB
    assert SS.chunk_frames(10, 25) == 2 and SS.chunk_frames(1 << 30) == 1


@pytest.mark.parametrize("bad", [-1, 1.5, "4", True, [3]])
def test_knob_is_validated(bad):
    with pytest.raises(ValueError, match="device_frames"):
        SS.check_device_frames(bad)
    with pytest.raises(ValueError, match="device_frames"):
        SS.QwenStreamState(rt.FlashMemory(), None, device_frames=bad)
    host = rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(rt.FlashMemory(), None))
    host.fvs_bank_device_frames = bad
    with pytest.raises(ValueError, match="fvs_bank_device_frames"):
        host.embed_new_video_clip(torch.zeros(4 * 1176), torch.tensor([[1, 2, 2]]), 0)


def test_knob_values():
    assert SS.check_device_frames(None) is None and SS.check_device_frames(0) == 0
    import numpy as np
    assert SS.check_device_frames(np.int64(7)) == 7
    assert rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(rt.FlashMemory(), None)).fvs_bank_device_frames is None


def test_knob_change_mid_stream_is_refused_before_the_tower():
    """a host with a stream in progress refuses a different cap before it runs anything; the same cap, or a new stream,
    is accepted"""
    from types import SimpleNamespace
    host = rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(rt.FlashMemory(), None))
    host.stream_state = SimpleNamespace(n_frames=4, device_frames=None)
    host.video_embedding_memory[:] = [0]
    host.fvs_bank_device_frames = 8
    with pytest.raises(ValueError, match="middle of a stream"):
        host._bank_device_frames()
    host.fvs_bank_device_frames = None
    assert host._bank_device_frames() is None
    host.fvs_bank_device_frames = 8
    host.init_streaming()
    assert host._bank_device_frames() == 8
