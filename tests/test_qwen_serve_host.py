"""CPU tests of the Qwen2-VL memory publication (qwen/serve.py, fvs_qwen_* of include/fvs_b200.h): layout arithmetic,
header decoding, the library's validation (refused before any CUDA call, so no device is needed) and the pickling guard."""
import ctypes as C
import pickle
import re
from pathlib import Path
from types import SimpleNamespace

import pytest
import torch

from flash_vstream_b200 import _lib as L
from flash_vstream_b200.qwen import serve as S

ROOT = Path(__file__).resolve().parents[1]


def test_layout_default_config():
    """60 CSM + 30 DAM frames of 24x24 / 12x12 tokens, merger 3584: 30*144 + 60*36 = 6480 rows (the ~46 MB video_embeds)"""
    lay = S.pub_layout(60, 30, (24, 24), (12, 12), 3584)
    assert lay["rows_cap"] == 6480
    assert lay["ts_off"] == 64 and lay["pos_off"] == 64 + 4 * 60 and lay["emb_off"] == 544
    assert lay["bytes"] == 544 + 6480 * 3584 * 2


@pytest.mark.parametrize("tem_len,spa_len,grid,small,dim", [
    (3, 5, (6, 10), (4, 6), 256),      # odd counts: the int64 positions start on an 8-byte boundary after padding
    (7, 0, (4, 4), (2, 2), 64),        # no DAM
    (0, 2, (2, 6), (2, 2), 8),         # no CSM
])
def test_layout_odd_configs(tem_len, spa_len, grid, small, dim):
    lay = S.pub_layout(tem_len, spa_len, grid, small, dim)
    assert lay["rows_cap"] == spa_len * grid[0] * grid[1] // 4 + tem_len * small[0] * small[1] // 4
    assert lay["ts_off"] == 64
    assert lay["pos_off"] % 8 == 0 and lay["pos_off"] >= 64 + 4 * tem_len and lay["pos_off"] - (64 + 4 * tem_len) < 8
    assert lay["emb_off"] % 16 == 0 and lay["emb_off"] >= lay["pos_off"] + 8 * spa_len
    assert lay["emb_off"] - (lay["pos_off"] + 8 * spa_len) < 16
    assert lay["bytes"] == lay["emb_off"] + lay["rows_cap"] * dim * 2


@pytest.mark.parametrize("args", [(2, 2, (3, 3), (2, 2), 64), (2, 2, (4, 4), (2, 2), 60), (-1, 2, (4, 4), (2, 2), 64),
                                  (2, 2, (0, 4), (2, 2), 64), (2, 2, (70000, 4), (2, 2), 64)])
def test_layout_refuses_bad_shapes(args):
    with pytest.raises(ValueError):
        S.pub_layout(*args)


def test_header_decoding():
    grid = S.pack_grid((24, 28), (12, 14))
    assert S.unpack_grid(grid) == ((24, 28), (12, 14))
    assert S.unpack_grid(S.pack_grid((65535, 1), (2, 65535))) == ((65535, 1), (2, 65535))
    st = S.decode_status([6, 6, 2, 17, 34, 8, 4, 624, grid])
    assert st["valid"] and st["epoch"] == 2 and st["clips"] == 17 and st["n_frames"] == 34
    assert st["n_tem"] == 8 and st["n_spa"] == 4 and st["rows"] == 624
    assert st["grid"] == (24, 28) and st["small_grid"] == (12, 14)
    assert not S.decode_status([5, 5, 0, 0, 0, 0, 0, 0, 0])["valid"]         # a publish was in progress
    assert not S.decode_status([6, 8, 0, 0, 0, 0, 0, 0, 0])["valid"]         # one completed while we copied
    empty = S.decode_status([0] * 9)                                          # never published: an empty memory
    assert empty["valid"] and empty["clips"] == 0 and empty["rows"] == 0 and empty["grid"] == (0, 0)
    # torch.int64 status words: a grid with ws >= 32768 comes back negative and must still decode
    big = S.pack_grid((2, 2), (2, 40000))
    assert S.unpack_grid(torch.tensor([big - 2 ** 64 if big >= 2 ** 63 else big]).item()) == ((2, 2), (2, 40000))


def test_new_symbols_are_declared_and_bound():
    header = (ROOT / "include" / "fvs_b200.h").read_text()
    for name in ("fvs_qwen_pub_layout", "fvs_qwen_publish", "fvs_qwen_snapshot"):
        assert re.search(rf"\bint {name}\(", header), name
        assert name in L.SIGNATURES
        assert getattr(L.load(), name) is not None


def _publish(lib, pub=0x1000, pub_bytes=1 << 20, tem_len=4, spa_len=2, rows_cap=None, dim=64, emb=0x2000, rows=None,
             ts=0x3000, n_tem=4, pos=0x4000, n_spa=2, grid=(4, 4), small=(2, 2)):
    rc = spa_len * grid[0] * grid[1] // 4 + tem_len * small[0] * small[1] // 4
    rows_cap = rc if rows_cap is None else rows_cap
    rows = n_spa * grid[0] * grid[1] // 4 + n_tem * small[0] * small[1] // 4 if rows is None else rows
    return lib.fvs_qwen_publish(pub, pub_bytes, tem_len, spa_len, rows_cap, dim, emb, rows, ts, n_tem, pos, n_spa, *grid,
                                *small, 1, 1, 8, None)


def _snapshot(lib, pub=0x1000, pub_bytes=1 << 20, rows_cap=12, out_rows=12, ts_cap=4, pos_cap=2, out=0x2000, status=0x5000):
    return lib.fvs_qwen_snapshot(pub, pub_bytes, 4, 2, rows_cap, 64, out, out_rows, 0x3000, ts_cap, 0x4000, pos_cap, status,
                                 None)


@pytest.mark.parametrize("kw,msg", [
    (dict(pub=None), "null publication"),
    (dict(emb=None), "null source"),
    (dict(ts=None), "null source"),
    (dict(pos=None), "null source"),
    (dict(pub_bytes=63), "bytes"),                      # smaller than the header
    (dict(pub_bytes=64 + 16 + 16 + 12 * 64 * 2 - 1), "bytes"),
    (dict(n_tem=5), "exceed"),
    (dict(rows=11), "rows do not match"),
    (dict(rows_cap=11), "rows do not match"),
    (dict(dim=60), "dim"),
    (dict(grid=(3, 3)), "bad grid"),
    (dict(emb=0x2008), "aligned"),
])
def test_publish_refusals_launch_nothing(kw, msg):
    lib = L.load()
    n0 = lib.fvs_launch_count()
    assert _publish(lib, **kw) == L.FVS_EINVAL
    assert msg in lib.fvs_last_error().decode()
    assert lib.fvs_launch_count() == n0


@pytest.mark.parametrize("kw,msg", [
    (dict(pub=None), "null pointer"),
    (dict(out=None), "null pointer"),
    (dict(status=None), "null pointer"),
    (dict(pub_bytes=100), "bytes"),
    (dict(out_rows=11), "below the publication's capacity"),
    (dict(ts_cap=3), "below the publication's capacity"),
    (dict(pos_cap=1), "below the publication's capacity"),
    (dict(rows_cap=-1), "negative capacity"),
])
def test_snapshot_refusals_launch_nothing(kw, msg):
    lib = L.load()
    n0 = lib.fvs_launch_count()
    assert _snapshot(lib, **kw) == L.FVS_EINVAL
    assert msg in lib.fvs_last_error().decode()
    assert lib.fvs_launch_count() == n0


def _cpu_host():
    import flash_vstream_b200.qwen.vstream_qwen2vl_realtime as rt
    visual = rt.VisualB200(rt.FlashMemory(), None, encode_patches=None, device="cpu")
    return rt.FlashVStreamQwen2VLRealtimeB200(visual)


def test_pickling_refused_mid_stream():
    host = _cpu_host()
    host.stream_state = SimpleNamespace(n_frames=4)
    with pytest.raises(L.FvsError, match="stream in progress"):
        pickle.dumps(host)


def test_lock_is_a_process_lock_and_export_needs_a_merger():
    import multiprocessing.synchronize as ms
    host = _cpu_host()
    assert isinstance(host.video_embedding_mem_lock, ms.Lock)        # torch.multiprocessing.Lock, as the reference
    with pytest.raises(NotImplementedError):
        S.export_qwen_memory(host, grid=(24, 24))
    assert "_qwen_publication" not in host.__dict__


def test_memory_manager_meters_the_reference_buckets():
    """the five buckets with the reference's formulas over the returned time list; the first clip is not logged"""
    import queue

    class Fake:
        def __init__(self):
            self.starts = []

        def embed_new_video_clip(self, pixel_values_videos, video_grid_thw, start_idx):
            self.starts.append(start_idx)
            return [0.0, 1.0, 3.0, 6.0, 10.0, 15.0, 21.0, 28.0]

    q = queue.Queue()
    for _ in range(3):
        q.put({"pixel_values_videos": None, "video_grid_thw": torch.tensor([[2, 4, 4]])})
    q.put(None)
    meter = S.MetricMeter()
    model = Fake()
    assert S.frame_memory_manager(model, q, time_meter=meter, meter_device_time=False) == 6
    assert model.starts == [0, 2, 4]
    assert meter.val("memory_latency_encoder") == (3 - 1) + (21 - 15)
    assert meter.val("memory_latency_readwrite") == (6 - 3) + (28 - 21)
    assert meter.val("memory_latency_cluster") == 4 and meter.val("memory_latency_retrieve") == 5
    assert meter._metrics["memory_latency"]._count == 2
