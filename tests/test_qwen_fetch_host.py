"""CPU checks of the Qwen2-VL evaluation drivers' pre-processing chain (preprocess.Qwen2VLVideoFetcher): the restated
fetch_video arithmetic (frame pick, padding, sizes) and the numpy oracle chain (preprocess_oracle.resize twice, then
qwen_pixels) against tests/golden/qwen_fetch.npz, which the reference's own fetch_video and image processor made; the
refusals, raised before any copy; and the library's host plan of two-stage and FVS_PRE_RGB8 jobs."""
from __future__ import annotations

import ctypes as C
import hashlib
import os
import zlib

import numpy as np
import pytest
import torch

from flash_vstream_b200 import _lib
from flash_vstream_b200 import preprocess as P
from tests import preprocess_oracle as O
from tests import qwen_fetch_inputs as QF

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "qwen_fetch.npz")


@pytest.fixture(scope="module")
def g():
    return np.load(GOLDEN)


def golden_stage1(g, name):
    """np.stack(fetch_video(ele)) of a case: the stored images, the last one repeated up to an even count"""
    s = g[f"{name}_stage1"]
    return np.concatenate([s, s[-1:]]) if len(s) % 2 else s


def digest(rows) -> str:
    """SHA-256 of fp32 rows, as the golden stores the reference's pixel_values_videos"""
    return hashlib.sha256(np.ascontiguousarray(np.asarray(rows), np.float32).tobytes()).hexdigest()


def golden_pixels(g, name):
    """the reference's pixel_values_videos of a case: the oracle on the golden's stage-1 bytes, held to the reference's
    digest (the rows are not stored)"""
    pool = QF.CASES[name][3]
    pre = P.Qwen2VLFramePreprocessor(QF.PROC_MIN_PIXELS, QF.PROC_MAX_PIXELS, pool)
    stage1 = golden_stage1(g, name)
    pix, _ = O.qwen_pixels(stage1, pre.resized(*stage1.shape[1:3]), pre.table)
    assert digest(pix) == str(g[f"{name}_pixels_sha256"]), f"{name}: the oracle's rows are not the reference's"
    return pix


def case(name):
    seed, shape, keys, pool = QF.CASES[name]
    return QF.frames(seed, shape), {"type": "video", **keys}, pool


@pytest.mark.parametrize("name", list(QF.CASES))
def test_host_arithmetic_and_oracle_chain_equal_golden(g, name):
    f, ele, pool = case(name)
    assert zlib.crc32(f.tobytes()) == int(g[f"{name}_crc"])
    picks = P.fetch_video_picks(len(f), ele)
    h1, w1 = P.fetch_video_size(*f.shape[1:3], len(f), ele)
    stage1 = golden_stage1(g, name)
    assert (len(picks), h1, w1) == stage1.shape[:3] and tuple(g[f"{name}_size"]) == (h1, w1)
    assert np.array_equal(O.resize(f[picks], h1, w1), stage1)
    pre = P.Qwen2VLFramePreprocessor(QF.PROC_MIN_PIXELS, QF.PROC_MAX_PIXELS, pool)
    pix, grid = O.qwen_pixels(stage1, pre.resized(h1, w1), pre.table)
    assert digest(pix) == str(g[f"{name}_pixels_sha256"])
    assert tuple(grid) == tuple(g[f"{name}_grid"]) == pre.grid_thw(len(picks), h1, w1)


def test_picks_follow_fetch_video():
    assert P.fetch_video_picks(5, {}) == [0, 1, 2, 3, 4, 4]                      # odd count: the last frame repeated
    assert P.fetch_video_picks(12, {"max_frames": 5}) == [0, 4, 7, 11]           # floor(5 / 2) * 2 = 4 picks
    assert P.fetch_video_picks(769, {}) == torch.linspace(0, 768, 768).round().long().unique().tolist()
    # max_pixels comes from the count before padding, and only from the picked count when max_frames cuts it
    assert P._fetch_budget(7, {})[2] == max(min(P.VIDEO_MAX_PIXELS, P.VIDEO_TOTAL_PIXELS / 7 * 2),
                                            P.VIDEO_MIN_PIXELS * 1.05)
    assert P._fetch_budget(7, {"max_pixels": 1234})[2] == 1234
    # resized_height / resized_width: fetch_image's own pixel bounds, not the video's
    assert P.fetch_video_size(10, 10, 3, {"resized_height": 30, "resized_width": 30, "max_pixels": 1}) == (56, 56)


class _NoCopy:
    """fails any host -> device copy or device allocation made while it is active"""

    def __enter__(self):
        self.saved = torch.Tensor.to, torch.Tensor.cuda, torch.empty

        def refuse(*a, **k):
            raise AssertionError("a refused element reached a copy or an allocation")
        torch.Tensor.to = torch.Tensor.cuda = refuse
        torch.empty = refuse
        return self

    def __exit__(self, *exc):
        torch.Tensor.to, torch.Tensor.cuda, torch.empty = self.saved


def test_refusals_raise_before_any_copy(g):
    fetcher = P.Qwen2VLVideoFetcher()
    seed, shape, keys, _ = QF.RATIO_CASE
    ratio = {"video": list(QF.frames(seed, shape)), **keys}
    with _NoCopy():
        with pytest.raises(ValueError) as e:
            fetcher.fetch(ratio)
        assert str(e.value) == str(g["ratio_error"])
        with pytest.raises(ValueError, match="no frame"):
            fetcher(dict(video=list(QF.frames(1, (3, 56, 56))), max_frames=1))
        with pytest.raises(ValueError, match="more than one size"):
            fetcher.many([{"video": [np.zeros((56, 56, 3), np.uint8), np.zeros((56, 84, 3), np.uint8)]}])
        with pytest.raises(ValueError, match="uint8"):
            fetcher.fetch({"video": [np.zeros((56, 56), np.uint8)] * 2})
        with pytest.raises(TypeError):
            fetcher.fetch({"video": "file:///a.mp4"})


def _axis(in_size, out_size, ptr=8):
    ax, _, _ = P.resample_plan(in_size, out_size)
    ax.bounds = ax.coeffs = ptr
    return ax


def _plan(jobs, layout, pool=2):
    n = len(jobs)
    arr, plan, totals = (_lib.PreprocessJob * n)(*jobs), (C.c_int64 * (4 * n))(), (C.c_int64 * 2)()
    r = _lib.load().fvs_preprocess_plan(arr, n, layout, pool, plan, totals)
    return r, list(plan), list(totals)


def test_library_plans_two_stage_and_rgb8_jobs():
    ws = _lib.load().fvs_preprocess_workspace_bytes
    x1, y1, x2, y2 = _axis(420, 196), _axis(300, 140), _axis(196, 224), _axis(140, 112)
    one = _lib.PreprocessJob(8, 2, 300, 420, 3, x1, y1)
    r, _, (out, wsb) = _plan([one], _lib.PRE_RGB8)
    assert r == 1 and out == 2 * 140 * 196 * 3 and wsb == ws(C.byref(x1), C.byref(y1), 2)
    two = _lib.PreprocessJob(8, 2, 300, 420, 3, x1, y1, x2, y2)
    assert _plan([one, two], _lib.PRE_QWEN)[0] == _lib.FVS_EINVAL        # job 0's 140x196 is not a multiple of 56
    r, plan, (out, wsb) = _plan([two, two], _lib.PRE_QWEN)
    scratch = max(ws(C.byref(x1), C.byref(y1), 2), ws(C.byref(x2), C.byref(y2), 2))
    assert r == 1 and out == 2 * (8 * 16 * 1176) and wsb == 2 * (scratch + 2 * 140 * 196 * 3)
    assert plan[4 + 2] == 8 * 16 * 1176 and plan[4 + 3] == scratch + 2 * 140 * 196 * 3
    # refusals: a second stage planned for another size, or only one of its axes set
    bad = _lib.PreprocessJob(8, 2, 300, 420, 3, x1, y1, _axis(200, 224), y2)
    assert _plan([bad], _lib.PRE_QWEN)[0] == _lib.FVS_EINVAL
    assert "second-stage x" in _lib.load().fvs_last_error().decode()
    half = _lib.PreprocessJob(8, 2, 300, 420, 3, x1, y1, x2)
    assert _plan([half], _lib.PRE_QWEN)[0] == _lib.FVS_EINVAL
    assert _plan([one], 4)[0] == _lib.FVS_EINVAL
