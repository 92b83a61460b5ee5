"""CPU checks of the pool serve loops and of many-clip pre-processing: round formation (readiness, per-stream order, end of
stream, all ended) through serve_pool with a fake step, the job-table planner fvs_preprocess_plan and its refusals
through the C ABI, and the argument checks of many() that need no device."""
from __future__ import annotations

import ctypes as C
import queue
import threading

import numpy as np
import pytest

from flash_vstream_b200 import _lib
from flash_vstream_b200 import preprocess as P
from flash_vstream_b200.serve import MetricMeter, form_round, serve_pool


# ---- round formation ---------------------------------------------------------------------------------------------------
def test_form_round():
    keys = ["a", "b", "c"]
    assert form_round(keys, {"c", "a"}, set()) == (["a", "c"], False)      # keys order, one clip each
    assert form_round(keys, set(), set()) == ([], False)                    # nothing ready: wait
    assert form_round(keys, {"a", "b"}, {"b"}) == (["a"], False)            # an ended stream takes no part
    assert form_round(keys, set(), {"a", "b"}) == ([], False)
    assert form_round(keys, set(), {"a", "b", "c"}) == ([], True)
    assert form_round([], set(), set()) == ([], True)


def _run(queues, feed=None):
    rounds = []

    def step(clips):
        rounds.append(dict(clips))
    meters = {}
    if feed is not None:
        threading.Thread(target=feed, daemon=True).start()
    counts = serve_pool(queues, step, len, time_meter=meters, meter_device_time=False)
    return counts, rounds, meters


def test_serve_pool_rounds_keep_order_and_end_streams_alone():
    qa, qb, qc = queue.Queue(), queue.Queue(), queue.Queue()
    for i in range(3):
        qa.put([("a", i)] * 2)                     # clips of 2 "frames"
    qa.put(None)
    qb.put([("b", 0)])
    qb.put(None)                                   # b ends after one clip; the others go on
    for i in range(5):
        qc.put([("c", i)])
    qc.put(None)
    counts, rounds, meters = _run({"a": qa, "b": qb, "c": qc})
    assert counts == {"a": 6, "b": 1, "c": 5}
    assert [sorted(r) for r in rounds] == [["a", "b", "c"]] + [["a", "c"]] * 2 + [["c"]] * 2
    for k in "ac":                                 # each stream's clips in its queue's order
        assert [r[k][0][1] for r in rounds if k in r] == list(range(3 if k == "a" else 5))
    assert isinstance(meters["a"], MetricMeter) and "b" not in meters      # first clip of a stream not logged
    assert meters["c"]._get("memory_latency")._count == 4


def test_serve_pool_blocks_until_a_clip_arrives():
    qa, qb = queue.Queue(), queue.Queue()
    go = threading.Event()

    def feed():                                    # b's clips arrive late, one by one, after a's stream ended
        qa.put([1])
        qa.put(None)
        go.wait(5)
        for i in range(3):
            qb.put([i])
        qb.put(None)
    threading.Timer(0.2, go.set).start()
    counts, rounds, _ = _run({"a": qa, "b": qb}, feed)
    assert counts == {"a": 1, "b": 3}
    assert [r.get("b") for r in rounds if "b" in r] == [[0], [1], [2]]


def test_serve_pool_returns_when_every_queue_ended():
    qs = {k: queue.Queue() for k in range(4)}
    for q in qs.values():
        q.put(None)
    counts, rounds, _ = _run(qs)
    assert counts == {k: 0 for k in range(4)} and rounds == []


def _no_queue_threads():
    for t in threading.enumerate():
        if t.name.startswith("pool-queue-"):
            t.join(5)
            assert not t.is_alive(), t.name


def test_serve_pool_keeps_a_bounded_queue_bounded():
    """the loop holds at most one clip per stream: a producer that outruns the steps blocks on its bounded queue"""
    q = queue.Queue(maxsize=3)
    put = []

    def feed():
        for i in range(40):
            q.put([i])
            put.append(i)
        q.put(None)
    behind = []

    def step(clips):
        threading.Event().wait(0.01)              # the GPU is slower than the camera
        behind.append(len(put) - sum(len(r) for r in rounds))
        rounds.append(clips)
    rounds = []
    t = threading.Thread(target=feed)
    t.start()
    counts = serve_pool({"a": q}, step, len, meter_device_time=False)
    t.join()
    assert counts == {"a": 40} and [r["a"] for r in rounds] == [[i] for i in range(40)]
    # put but not yet stepped: the round's clip + one held + 3 in the queue
    assert max(behind) <= 5, behind
    _no_queue_threads()


def test_serve_pool_gives_back_what_it_took_when_the_step_raises():
    qa, qb = queue.Queue(), queue.Queue()
    for i in range(6):
        qa.put(["a", i])
        qb.put(["b", i])
    done = []

    def step(clips):
        if len(done) == 2:
            raise ValueError("refused")
        done.append(clips)
    with pytest.raises(ValueError, match="refused") as err:
        serve_pool({"a": qa, "b": qb}, step, len, meter_device_time=False)
    _no_queue_threads()
    for k, q in (("a", qa), ("b", qb)):
        rest = []
        while not q.empty():
            rest.append(q.get_nowait()[1])
        back = [c[1] for c in err.value.unconsumed[k]]
        assert [r[k][1] for r in done] + back + rest == list(range(6)), (k, back, rest)   # nothing lost, order kept
        assert back[0] == 2 and len(back) <= 2                 # the failed round's clip, at most one held
    qa.put(["a", 9])                                           # no thread of the finished loop takes from the queues
    threading.Event().wait(0.2)
    assert qa.get_nowait() == ["a", 9]


# ---- the job-table planner (no device) ---------------------------------------------------------------------------------
_TABLES = np.zeros(16, np.int64)                   # stands in for device tables: the planner reads only the pointers


def _job(T, H, W, pre, ch=3):
    (oh, fy, cy), (ow, fx, cx), _ = pre._windows(H, W)
    axes = []
    for n_in, n_out, first, count in ((W, ow, fx, cx), (H, oh, fy, cy)):
        ax, _, _ = P.resample_plan(n_in, n_out, first, count)
        ax.bounds = ax.coeffs = _TABLES.ctypes.data
        axes.append(ax)
    return _lib.PreprocessJob(8, T, H, W, ch, *axes)


def _plan(jobs, layout, pool=1):
    n = len(jobs)
    arr, plan, totals = (_lib.PreprocessJob * n)(*jobs), (C.c_int64 * (4 * n))(), (C.c_int64 * 2)()
    r = _lib.load().fvs_preprocess_plan(arr, n, layout, pool, plan, totals)
    return r, np.array(plan[:]).reshape(n, 4), tuple(totals)


class _Clip(P.CLIPFramePreprocessor):
    def __init__(self):                            # the defaults of CLIPImageProcessor: 336 shortest edge and crop
        from tests.test_preprocess_host import _clip_processor
        super().__init__(_clip_processor())


SIZES = [(2, 480, 640), (3, 720, 1280), (1, 1080, 1920), (4, 333, 517), (1, 90, 100)]


@pytest.mark.parametrize("n", [1, 2, 33, 70])
def test_plan_clip_offsets_and_totals(n):
    pre = _Clip()
    sizes = [SIZES[i % len(SIZES)] for i in range(n)]
    r, plan, (out_total, ws_total) = _plan([_job(*s, pre) for s in sizes], _lib.PRE_CLIP)
    assert r == -(-n // 32)                                                 # launch pairs
    rows = col = out = ws = 0
    for i, (T, H, W) in enumerate(sizes):
        (oh, fy, cy), (ow, fx, cx), _ = pre._windows(H, W)
        ax, _, _ = P.resample_plan(W, ow, fx, cx)
        ay, _, _ = P.resample_plan(H, oh, fy, cy)
        if i % 32 == 0:
            rows = col = 0
        assert tuple(plan[i]) == (rows, col, out, ws), i
        rows += ay.span_count * T
        col += ay.count * T
        out += T * 3 * 336 * 336
        ws += int(_lib.load().fvs_preprocess_workspace_bytes(C.byref(ax), C.byref(ay), T))
    assert (out_total, ws_total) == (out, ws)


@pytest.mark.parametrize("pool", [1, 2])
def test_plan_qwen_output_rows(pool):
    pre = P.Qwen2VLFramePreprocessor(additional_pool_size=pool)
    sizes = [(2, 480, 640), (1, 333, 517), (4, 720, 1280)]
    r, plan, (out_total, _) = _plan([_job(*s, pre) for s in sizes], _lib.PRE_QWEN, pool)
    assert r == 1
    rows = [int(np.prod(pre.output_shape(*s))) for s in sizes]
    assert list(plan[:, 2]) == [0, rows[0], rows[0] + rows[1]] and out_total == sum(rows)


def test_plan_refusals_name_the_job():
    clip, qwen = _Clip(), P.Qwen2VLFramePreprocessor()
    good = _job(2, 480, 640, clip)
    stale = _job(2, 480, 640, clip)
    stale.W = 648                                                           # the plan is for 640 columns
    cases = [([good, good, _job(2, 480, 640, clip, ch=4)], _lib.PRE_CLIP, "job 2: 4 channels"),
             ([good, stale], _lib.PRE_CLIP, "job 1: the x-axis plan is for 640"),
             ([_job(2, 56, 56, qwen), _job(3, 56, 56, qwen)], _lib.PRE_QWEN, "job 1: Qwen2-VL clips hold 1 or an even"),
             ([good, _job(0, 480, 640, clip)], _lib.PRE_CLIP, "job 1: empty input"),
             ([good], 7, "job 0: unknown layout")]
    for jobs, layout, msg in cases:
        r, _, _ = _plan(jobs, layout)
        assert r == _lib.FVS_EINVAL
        assert msg in _lib.load().fvs_last_error().decode(), (msg, _lib.load().fvs_last_error())
    nulled = _job(2, 480, 640, clip)
    nulled.frames = None
    assert _plan([good, nulled], _lib.PRE_CLIP)[0] == _lib.FVS_EINVAL
    assert "job 1: null frames" in _lib.load().fvs_last_error().decode()


def test_multi_refuses_before_any_launch_without_a_device():
    """every check of fvs_preprocess_multi runs on the host: refused calls return before any CUDA call"""
    clip = _Clip()
    jobs = (_lib.PreprocessJob * 2)(_job(2, 480, 640, clip), _job(1, 720, 1280, clip, ch=4))
    lib = _lib.load()
    r = lib.fvs_preprocess_multi(jobs, 2, 16, _lib.PRE_CLIP, 1, 16, 16, 1 << 30, None)
    assert r == _lib.FVS_EINVAL and "job 1: 4 channels" in lib.fvs_last_error().decode()
    jobs[1].C = 3
    r = lib.fvs_preprocess_multi(jobs, 2, 16, _lib.PRE_CLIP, 1, 16, 16, 100, None)
    assert r == _lib.FVS_EINVAL and "workspace of 100 bytes" in lib.fvs_last_error().decode()
    assert lib.fvs_preprocess_multi(jobs, 0, 16, _lib.PRE_CLIP, 1, 16, 16, 100, None) == _lib.FVS_EINVAL


# ---- many(): argument checks that need no device -----------------------------------------------------------------------
def test_many_argument_checks():
    pre = P.Qwen2VLFramePreprocessor()
    with pytest.raises(TypeError, match="list"):
        pre.many(np.zeros((2, 56, 56, 3), np.uint8))
    with pytest.raises(ValueError, match="empty"):
        pre.many([])
    with pytest.raises(ValueError, match="clip 1 must be uint8"):
        pre.many([np.zeros((2, 56, 56, 3), np.uint8), np.zeros((2, 56, 56, 3), np.float32)])
    with pytest.raises(ValueError, match="clip 0 must be uint8"):
        pre.many([np.zeros((56, 56, 3), np.uint8)])
    with pytest.raises(TypeError, match="clip 2"):
        _Clip().many([np.zeros((1, 8, 8, 3), np.uint8)] * 2 + ["frame"])
