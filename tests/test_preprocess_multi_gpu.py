"""GPU tests of many-clip pre-processing (fvs_preprocess_multi / _FramePreprocessor.many): each clip's slice of the one
contiguous output is bit-identical to the preprocessor's single-clip output, at mixed sizes, in both layouts, for 1 to
70 clips (across the 32-job launch boundary), with two launches per 32 clips; a refused call launches nothing, writes
nothing and names the job."""
import ctypes as C

import numpy as np
import pytest
import torch

from flash_vstream_b200 import _lib
from flash_vstream_b200 import preprocess as P
from tests import preprocess_inputs as PI
from tests.test_gpu_parity import fvs  # noqa: F401  (a fixture)
from tests.test_preprocess_host import GOLDEN, _clip_processor

pytestmark = pytest.mark.gpu

SIZES = [(2, 480, 640), (2, 720, 1280), (2, 1080, 1920), (2, 333, 517), (1, 480, 640)]


def _clips(n, seed=0):
    """n seeded uint8 clips cycling through SIZES; every other one on the host (pinned or pageable)"""
    out = []
    for i in range(n):
        f = torch.from_numpy(PI.frames(seed + i, SIZES[i % len(SIZES)]))
        out.append(f.cuda() if i % 2 == 0 else (f.pin_memory() if i % 4 == 1 else f))
    return out


def _processors():
    return {"clip336": P.CLIPFramePreprocessor(_clip_processor()), "qwen_pool1": P.Qwen2VLFramePreprocessor(),
            "qwen_pool2": P.Qwen2VLFramePreprocessor(additional_pool_size=2)}


@pytest.mark.parametrize("n", [1, 2, 5, 33, 70])
@pytest.mark.parametrize("name", ["clip336", "qwen_pool1", "qwen_pool2"])
def test_many_equals_one_clip_at_a_time(fvs, name, n):
    pre = _processors()[name]
    clips = _clips(n, 10 * n)
    lib = _lib.load()
    n0 = lib.fvs_launch_count()
    res = pre.many(clips)
    launches = lib.fvs_launch_count() - n0
    assert launches == 2 * -(-n // 32)
    out, views = res[0], res[1]
    assert out.is_contiguous() and len(views) == n
    r = 0
    for i, (f, v) in enumerate(zip(clips, views)):
        one = pre(f)
        if name == "clip336":
            assert v.shape == one.shape == (f.shape[0], 3, 336, 336)
        else:
            assert torch.equal(res[2][i], one["video_grid_thw"]), i
            one = one["pixel_values_videos"]
        assert torch.equal(v, one), (name, n, i)
        assert v.data_ptr() == out.data_ptr() + r * out.element_size()        # back to back in job order
        r += v.numel()
    assert r == out.numel()


def test_many_into_caller_buffers(fvs):
    pre = P.CLIPFramePreprocessor(_clip_processor())
    clips = _clips(3, 7)
    want, _ = pre.many(clips)
    out = torch.full_like(want, float("nan"))
    ws = torch.empty(sum(pre.workspace_bytes(*f.shape[:3]) for f in clips), dtype=torch.uint8, device="cuda")
    got, views = pre.many(clips, out=out, workspace=ws)
    assert got is out and torch.equal(out, want) and views[1].data_ptr() > out.data_ptr()


def _refused(pre, clips, match, out=None, workspace=None):
    """the call raises, names the job, launches nothing and leaves a sentinel-filled output as it was"""
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.fvs_launch_count()
    with pytest.raises(ValueError, match=match):
        pre.many(clips, out=out, workspace=workspace)
    torch.cuda.synchronize()
    assert lib.fvs_launch_count() == n0


def test_refusals_launch_nothing(fvs):
    qwen = P.Qwen2VLFramePreprocessor()
    clips = [torch.from_numpy(PI.frames(1, s)).cuda() for s in ((2, 56, 56), (3, 56, 56))]     # an odd count > 1
    _refused(qwen, clips, "job 1: Qwen2-VL clips hold 1 or an even number")
    four = [clips[0], clips[0], torch.zeros(2, 56, 56, 4, dtype=torch.uint8, device="cuda")]
    _refused(qwen, four, "job 2: 4 channels")
    host = [np.zeros((2, 56, 56, 3), np.uint8), np.zeros((3, 56, 56, 3), np.uint8)]    # host clips: planned, not copied
    qwen.many(host[:1])                                                                # the plan tables of 56x56 exist
    torch.cuda.synchronize()
    n_alloc = torch.cuda.memory_stats()["allocation.all.allocated"]
    _refused(qwen, host, "job 1: Qwen2-VL clips hold 1 or an even number")
    assert torch.cuda.memory_stats()["allocation.all.allocated"] == n_alloc
    clip = P.CLIPFramePreprocessor(_clip_processor())
    good = _clips(3, 3)
    out = torch.full((6, 3, 336, 336), 7.0, dtype=torch.float16, device="cuda")
    _refused(clip, good, "workspace of 16 bytes", out=out, workspace=torch.empty(16, dtype=torch.uint8, device="cuda"))
    assert bool((out == 7).all())


def test_stale_plan_refused_through_the_abi(fvs):
    """a job whose plan is for another frame size (a stale plan): refused by fvs_preprocess_multi before any launch,
    naming the job, the sentinel output untouched"""
    pre = P.CLIPFramePreprocessor(_clip_processor())
    f = [torch.from_numpy(PI.frames(2, (1, 480, 640))).cuda(), torch.from_numpy(PI.frames(3, (1, 720, 1280))).cuda()]
    jobs = (_lib.PreprocessJob * 2)()
    for i, x in enumerate(f):
        ax, ay, _, _ = pre._plan(x.device, 480, 640)                         # job 1 gets job 0's plan
        jobs[i] = _lib.PreprocessJob(x.data_ptr(), 1, *x.shape[1:], ax, ay)
    out = torch.full((2, 3, 336, 336), 7.0, dtype=torch.float16, device="cuda")
    ws = torch.empty(1 << 24, dtype=torch.uint8, device="cuda")
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.fvs_launch_count()
    r = lib.fvs_preprocess_multi(jobs, 2, pre._table(x.device).data_ptr(), _lib.PRE_CLIP, 1, out.data_ptr(), ws.data_ptr(),
                                 ws.numel(), _lib.cur_stream())
    assert r == _lib.FVS_EINVAL and "job 1: the x-axis plan is for 640" in lib.fvs_last_error().decode()
    torch.cuda.synchronize()
    assert lib.fvs_launch_count() == n0 and bool((out == 7).all())
    plan, totals = (C.c_int64 * 8)(), (C.c_int64 * 2)()
    assert lib.fvs_preprocess_plan(jobs, 2, _lib.PRE_CLIP, 1, plan, totals) == _lib.FVS_EINVAL


def test_single_clip_call_unchanged_goldens(fvs):
    """fvs_preprocess is the one-job case of the job table: the committed goldens through both entry points"""
    g = np.load(GOLDEN)
    for name, (seed, shape, se, crop) in PI.CLIP_CASES.items():
        pre = P.CLIPFramePreprocessor(_clip_processor(se, crop))
        f = torch.from_numpy(PI.frames(seed, shape)).cuda()
        assert torch.equal(pre.many([f])[1][0].cpu(), torch.from_numpy(g[f"clip_{name}"])), name
    for name, (seed, shape, mn, mx, pool) in PI.QWEN_CASES.items():
        f = torch.from_numpy(PI.frames(seed, shape)).cuda()
        _, views, grids = P.Qwen2VLFramePreprocessor(mn, mx, pool).many([f, f])
        for v in views:
            assert torch.equal(v.cpu(), torch.from_numpy(g[f"qwen_{name}"])), name
        assert torch.equal(grids[1], torch.from_numpy(g[f"qwen_{name}_grid"]).reshape(1, 3)), name
