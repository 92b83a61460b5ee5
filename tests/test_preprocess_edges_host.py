"""CPU checks behind tests/test_preprocess_edges_gpu.py: the guard checker reports what it must (a changed guard, an
output element left at the sentinel, a workspace or frame tail written); the restated fetch_video arithmetic (sizes,
picks) and the processor's grid at the sizes real videos have, against tests/golden/qwen_fetch_sizes.npz, which the
reference's own fetch_video and image processor made; the library's host plan at its limits (a 16384-column row span,
T = 65535), with nothing launched when it refuses."""
from __future__ import annotations

import ctypes as C
import os
import zlib

import numpy as np
import pytest
import torch

from flash_vstream_b200 import _lib
from flash_vstream_b200 import preprocess as P
from tests import preprocess_edges as E
from tests import qwen_fetch_sizes_inputs as QS

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "qwen_fetch_sizes.npz")


@pytest.fixture(scope="module")
def golden():
    return np.load(GOLDEN)


def case(name):
    """(seeded frames, the fetch_video element without its 'video', additional_pool_size)"""
    seed, shape, keys, pool = QS.CASES[name]
    return QS.frames(seed, shape), {"type": "video", **keys}, pool


# ---- the guard checker -----------------------------------------------------------------------------------------------
def _runs(dtype, n=40):
    """two clean runs of a fake call: the same payload inside each run's guarded output, poisoned workspaces of 100
    bytes given, one job's frames of 30 bytes"""
    payload = torch.arange(n).to(dtype)
    outs, wss, fbs = [], [], []
    for run in (0, 1):
        buf, view = E.guarded_output(n, dtype, run, "cpu")
        view.copy_(payload)
        outs.append(buf)
        wss.append(E.poisoned_workspace(100, run, "cpu"))
        fbs.append([E.poisoned_frames(torch.arange(30, dtype=torch.uint8), run)])
    return outs, wss, fbs


@pytest.mark.parametrize("dtype", [torch.uint8, torch.float16, torch.float32])
def test_guard_checker_reports_planted_faults(dtype):
    outs, wss, fbs = _runs(dtype)
    assert E.report("clean", outs, wss, 100, fbs, [30]) == []
    for where in (E.GUARD - 1, E.GUARD + 40):              # the element before the first job, after the last
        outs, wss, fbs = _runs(dtype)
        E.as_int(outs[1])[where] ^= 1                        # a flipped low bit: a NaN guard stays NaN
        probs = E.report("flip", outs, wss, 100, fbs, [30])
        assert len(probs) == 1 and "run 1: 1 output guard elements changed" in probs[0], probs
        assert f"element {-1 if where < E.GUARD else 40}" in probs[0], probs
    outs, wss, fbs = _runs(dtype)
    for run in (0, 1):                           # an element the kernel never wrote keeps each run's sentinel
        E.as_int(outs[run])[E.GUARD + 7] = E.signed(E.SENTINEL[dtype][run], dtype)
    probs = E.report("left", outs, wss, 100, fbs, [30])
    assert len(probs) == 1 and "1 output elements differ between the two poisons, 1 of them still the sentinel" in \
        probs[0] and "first at element 7" in probs[0], probs
    outs, wss, fbs = _runs(dtype)
    wss[0][100] = 3                                         # a byte past the workspace the call was given
    fbs[1][0][30] = 3                                       # a byte past the job's frames
    probs = E.report("tails", outs, wss, 100, fbs, [30])
    assert len(probs) == 2 and "run 0: 1 workspace bytes past the 100 given" in probs[0] and \
        "run 1: the poison past job 0's frames" in probs[1], probs


def test_sentinels_are_two_different_nans_and_bytes():
    for dtype, (a, b) in E.SENTINEL.items():
        assert a != b
        if dtype != torch.uint8:
            ib = E.as_int(torch.empty(0, dtype=dtype)).dtype
            bits = torch.tensor([E.signed(a, dtype), E.signed(b, dtype)], dtype=ib)
            assert bool(torch.isnan(bits.view(dtype)).all()), dtype
    assert E.POISON == (0x00, 0xFF)


# ---- the drivers' chain at real sizes: host arithmetic ---------------------------------------------------------------
@pytest.mark.parametrize("name", list(QS.CASES))
def test_fetch_sizes_picks_and_grids_equal_golden(golden, name):
    f, ele, pool = case(name)
    assert zlib.crc32(f.tobytes()) == int(golden[f"{name}_crc"]), f"seeded frames of {name} changed"
    picks = P.fetch_video_picks(len(f), ele)
    assert picks == golden[f"{name}_picks"].tolist()
    h1, w1 = P.fetch_video_size(*f.shape[1:3], len(f), ele)
    assert (h1, w1) == tuple(golden[f"{name}_size"].tolist())
    pre = P.Qwen2VLFramePreprocessor(QS.PROC_MIN_PIXELS, QS.PROC_MAX_PIXELS, pool)
    assert pre.grid_thw(len(picks), h1, w1) == tuple(golden[f"{name}_grid"].tolist())
    assert 2 <= len(f) <= 16


def test_cases_cover_real_sizes(golden):
    """360p to 1080p, a portrait, 4:3 and ultra-wide frame; a first stage capped by VIDEO_MAX_PIXELS, second stages
    that resize and that do not; the golden holds digests only"""
    sizes = {shape[1:] for _, shape, _, _ in QS.CASES.values()}
    assert {(360, 640), (480, 854), (720, 1280), (1080, 1920), (1920, 1080), (768, 1024), (1080, 2560)} <= sizes
    assert {k for _, _, keys, _ in QS.CASES.values() for k in keys} == {"max_frames", "total_pixels", "max_pixels",
                                                                         "resized_height", "resized_width"}
    resizes = set()
    for name, (_, _, _, pool) in QS.CASES.items():
        h1, w1 = golden[f"{name}_size"].tolist()
        pre = P.Qwen2VLFramePreprocessor(QS.PROC_MIN_PIXELS, QS.PROC_MAX_PIXELS, pool)
        resizes.add(pre.resized(h1, w1) != (h1, w1))
    assert resizes == {False, True}
    assert os.path.getsize(GOLDEN) < 64 * 1024


# ---- the library's host plan at its limits ---------------------------------------------------------------------------
def _axis(in_size, out_size, first=0, count=None):
    ax, _, _ = P.resample_plan(in_size, out_size, first, count)
    ax.bounds = ax.coeffs = 8               # never read: the plan does not touch the device
    return ax


def _plan(jobs, layout=_lib.PRE_RGB8, pool=1):
    n = len(jobs)
    arr, plan, totals = (_lib.PreprocessJob * n)(*jobs), (C.c_int64 * (4 * n))(), (C.c_int64 * 2)()
    return _lib.load().fvs_preprocess_plan(arr, n, layout, pool, plan, totals), list(totals)


def test_plan_limits():
    lib = _lib.load()
    n0 = lib.fvs_launch_count()
    x, y = _axis(16384, 8191), _axis(3, 2)
    assert x.span_count == 16384
    assert _plan([_lib.PreprocessJob(8, 2, 3, 16384, 3, x, y)]) == (1, [2 * 2 * 8191 * 3, 2 * 3 * 3 * 8191])
    wide = _lib.PreprocessJob(8, 1, 3, 16385, 3, _axis(16385, 8192), y)
    assert _plan([wide])[0] == _lib.FVS_EINVAL
    assert "a window reading 16385 source columns" in lib.fvs_last_error().decode()
    two = _lib.PreprocessJob(8, 1, 3, 8192, 3, _axis(8192, 16385), _axis(3, 3), _axis(16385, 100), _axis(3, 3))
    assert _plan([two])[0] == _lib.FVS_EINVAL and "16385 source columns" in lib.fvs_last_error().decode()
    tiny = _axis(3, 5), _axis(2, 3)
    assert _plan([_lib.PreprocessJob(8, 65535, 2, 3, 3, *tiny)]) == (1, [65535 * 3 * 5 * 3, 65535 * 3 * 2 * 5])
    good = [_lib.PreprocessJob(8, 2, 2, 3, 3, *tiny)] * 40
    assert _plan(good + [_lib.PreprocessJob(8, 65536, 2, 3, 3, *tiny)])[0] == _lib.FVS_EINVAL
    assert "job 40: 65536 frames in one call (at most 65535)" in lib.fvs_last_error().decode()
    assert _plan(good)[0] == 2
    assert lib.fvs_launch_count() == n0
