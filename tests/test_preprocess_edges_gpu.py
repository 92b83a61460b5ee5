"""GPU tests of the frame pre-processing kernels (csrc/preprocess_kernels.cu) at their edges, every call under poisoned
neighbours (tests/preprocess_edges.py: frames followed by poison, a poisoned workspace, outputs between guards, each
call run under two poisons):

- the 220 (h, w) -> (H, W) pairs of test_preprocess_host._size_pairs (1-pixel axes, downscales up to 12x, upscales up
  to 8x, odd sizes) in the RGB8 layout, byte for byte against Pillow called here, as one table (7 launch groups) and one
  job per call; the same pairs as two-stage jobs (there and back) against Pillow applied twice;
- the CLIP layout with crop windows at offset 0, the centre and the far edge of each axis, and the Qwen2-VL fp32 rows
  and 8-bit codes at pool 1 and 2 with T = 1, 2 and 4, against the numpy oracle's crop / patchify of Pillow's bytes;
- the limits: a 16384-column row span (16385 refused), T = 65535 (65536 refused), a refused table launches nothing,
  H = 1 and W = 1 in both stages;
- Qwen2VLVideoFetcher at the sizes real videos have (tests/golden/qwen_fetch_sizes.npz, made by the reference's
  fetch_video and image processor): fetch, __call__, codes=True and many against the golden's digests, Pillow for the
  first stage and the oracle for the second."""
import ctypes as C
import hashlib

import numpy as np
import pytest
import torch
from PIL import Image

from flash_vstream_b200 import _lib
from flash_vstream_b200 import preprocess as P
from tests import preprocess_edges as E
from tests import preprocess_inputs as PI
from tests import preprocess_oracle as O
from tests import qwen_fetch_sizes_inputs as QS
from tests.test_preprocess_edges_host import case, golden  # noqa: F401  (golden is a fixture)
from tests.test_preprocess_host import _size_pairs

pytestmark = pytest.mark.gpu

# CLIP's and Qwen2-VL's value table: the library's (P.value_table) is what the kernels are given, the oracle's, built
# from the processors' published constants (tests/preprocess_inputs.py), is what the references look bytes up in
TABLE = P.value_table(1 / 255, P.OPENAI_CLIP_MEAN, P.OPENAI_CLIP_STD)
REF_TABLE = O.value_table(1 / 255, PI.OPENAI_CLIP_MEAN, PI.OPENAI_CLIP_STD)
OUT_DTYPE = {_lib.PRE_CLIP: torch.float16, _lib.PRE_QWEN: torch.float32, _lib.PRE_QWEN_CODES: torch.uint8,
             _lib.PRE_RGB8: torch.uint8}
PAIRS = _size_pairs()
_plans = {}


@pytest.fixture(scope="module")
def dev():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    return {"table": torch.from_numpy(TABLE).cuda()}


def axis(in_size, out_size, first=0, count=None):
    """the library's plan of one axis, its tables on the device (kept for the module)"""
    count = out_size - first if count is None else count
    key = (in_size, out_size, first, count)
    if key not in _plans:
        ax, bounds, coeffs = P.resample_plan(*key)
        b, k = torch.from_numpy(bounds).cuda(), torch.from_numpy(coeffs).cuda()
        ax.bounds, ax.coeffs = b.data_ptr(), k.data_ptr()
        _plans[key] = (ax, b, k)
    return _plans[key][0]


class Job:
    """one clip of a table: device frames [T, H, W, 3] and its plans (x2 / y2 set: a two-stage job)"""

    def __init__(self, frames, x, y, x2=None, y2=None):
        self.frames, self.x, self.y, self.x2, self.y2 = frames, x, y, x2, y2

    def struct(self):
        T, H, W, ch = self.frames.shape
        extra = (self.x2, self.y2) if self.x2 is not None else ()
        return _lib.PreprocessJob(self.frames.data_ptr(), T, H, W, ch, self.x, self.y, *extra)


def call(name, jobs, layout, pool, dev):
    """every job through one fvs_preprocess_multi call under each poison -> (run 0's output on the device, each job's
    output offset, the problems E.report finds); checks the launch count (two per group of 32, two more for a group
    with a two-stage job)"""
    lib = _lib.load()
    n = len(jobs)
    arr = (_lib.PreprocessJob * n)(*[j.struct() for j in jobs])
    plan, totals = (C.c_int64 * (4 * n))(), (C.c_int64 * 2)()
    groups = lib.fvs_preprocess_plan(arr, n, layout, pool, plan, totals)
    assert groups == -(-n // 32), (name, groups, lib.fvs_last_error())
    launches = sum(2 + 2 * any(j.x2 is not None for j in jobs[g:g + 32]) for g in range(0, n, 32))
    n_out, n_ws = int(totals[0]), int(totals[1])
    outs, wss, fbufs = [], [], []
    for run in (0, 1):
        fb = [E.poisoned_frames(j.frames, run) for j in jobs]
        for i, b in enumerate(fb):
            arr[i].frames = b.data_ptr()
        ws = E.poisoned_workspace(n_ws, run, "cuda")
        buf, view = E.guarded_output(n_out, OUT_DTYPE[layout], run, "cuda")
        n0 = lib.fvs_launch_count()
        r = lib.fvs_preprocess_multi(arr, n, dev["table"].data_ptr(), layout, pool, view.data_ptr(), ws.data_ptr(),
                                     n_ws, _lib.cur_stream())
        assert r == _lib.FVS_OK, (name, lib.fvs_last_error())
        assert lib.fvs_launch_count() - n0 == launches, name
        outs.append(buf)
        wss.append(ws)
        fbufs.append(fb)
    torch.cuda.synchronize()
    probs = E.report(name, outs, wss, n_ws, fbufs, [j.frames.numel() for j in jobs])
    return outs[0][E.GUARD:E.GUARD + n_out], [int(plan[4 * i + 2]) for i in range(n)], probs


def mismatch(got: np.ndarray, want: np.ndarray):
    """None when the bits are equal, else (elements that differ, the largest absolute difference)"""
    if got.shape == want.shape and np.array_equal(got.view(f"u{got.itemsize}"), want.view(f"u{want.itemsize}")):
        return None
    if got.shape != want.shape:
        return f"shape {got.shape} != {want.shape}"
    d = np.abs(got.astype(np.float64) - want.astype(np.float64))
    return f"{int((got.view(f'u{got.itemsize}') != want.view(f'u{want.itemsize}')).sum())} elements differ, largest " \
           f"|difference| {np.nanmax(d) if np.isfinite(d).any() else 'nan'}"


def compare(name, out, offsets, wants, probs):
    """each job's slice of `out` against its reference; fails with every problem, the largest mismatch per job"""
    flat = out.cpu().numpy()
    for i, (off, want) in enumerate(zip(offsets, wants)):
        got = flat[off:off + want.size].reshape(want.shape)
        m = mismatch(got, want)
        if m:
            probs.append(f"{name}: job {i}: {m}")
    assert not probs, "\n".join(probs[:20])


def pillow(img, h, w):
    """uint8 [..., H, W, 3] -> [..., h, w, 3], each image through Image.resize((w, h), BICUBIC)"""
    lead = img.shape[:-3]
    flat = img.reshape((-1,) + img.shape[-3:])
    out = np.stack([np.asarray(Image.fromarray(x).resize((w, h), Image.BICUBIC)) for x in flat])
    return out.reshape(lead + out.shape[1:])


_frames, _resized = {}, {}


def sweep_frames(i):
    """pair i's seeded frames, 1 to 3 of them (host, and the device copy)"""
    if i not in _frames:
        h, w, _, _ = PAIRS[i]
        f = np.random.default_rng(1000 + i).integers(0, 256, (1 + i % 3, h, w, 3), dtype=np.uint8)
        _frames[i] = (f, torch.from_numpy(f).cuda())
    return _frames[i]


def resized(i, h=None, w=None):
    """Pillow's resize of pair i's frames to (h, w), by default the pair's (H, W)"""
    _, _, H, W = PAIRS[i]
    key = (i, h or H, w or W)
    if key not in _resized:
        _resized[key] = pillow(sweep_frames(i)[0], key[1], key[2])
    return _resized[key]


# ---- the resize sweep ------------------------------------------------------------------------------------------------
def test_rgb8_sweep_equals_pillow_as_one_table_and_one_job_per_call(dev):
    jobs = [Job(sweep_frames(i)[1], axis(w, W), axis(h, H)) for i, (h, w, H, W) in enumerate(PAIRS)]
    wants = [resized(i) for i in range(len(PAIRS))]
    out, offsets, probs = call("rgb8 table", jobs, _lib.PRE_RGB8, 1, dev)
    assert len(PAIRS) == 220 and -(-len(jobs) // 32) == 7
    compare("rgb8 table", out, offsets, wants, probs)
    for i, j in enumerate(jobs):
        one, _, probs = call(f"rgb8 job {i} {PAIRS[i]}", [j], _lib.PRE_RGB8, 1, dev)
        assert not probs, "\n".join(probs)
        assert torch.equal(one, out[offsets[i]:offsets[i] + one.numel()]), (i, PAIRS[i])


def test_two_stage_sweep_equals_pillow_twice(dev):
    """every pair there and back, (h, w) -> (H, W) -> (h, w), as two-stage jobs in one table"""
    jobs = [Job(sweep_frames(i)[1], axis(w, W), axis(h, H), axis(W, w), axis(H, h))
            for i, (h, w, H, W) in enumerate(PAIRS)]
    out, offsets, probs = call("two-stage rgb8", jobs, _lib.PRE_RGB8, 1, dev)
    compare("two-stage rgb8", out, offsets, [pillow(resized(i), h, w) for i, (h, w, _, _) in enumerate(PAIRS)], probs)


def crop_windows(n, c):
    """the offsets 0, centre and far edge of a c-long window in an n-long axis (deduplicated)"""
    return sorted({0, (n - c) // 2, n - c})


@pytest.mark.parametrize("top", ["0", "centre", "far edge"])
def test_clip_crop_windows_equal_oracle(dev, top):
    """a crop of about two thirds of each axis (the whole of a 1-pixel axis) with its top at offset 0, the centre or the
    far edge, and its left at each of the three, in the CLIP f16 layout: the oracle's crop and lookup of Pillow's
    bytes.  Past offset 0 the windows must start inside the source (a span that does not start at row or column 0), so
    the kernels' row0 / span0 offsets are exercised."""
    jobs, wants = [], []
    for i, (h, w, H, W) in enumerate(PAIRS):
        ch, cw = H - H // 3, W - W // 3
        tops = crop_windows(H, ch)
        y0 = {"0": tops[0], "centre": tops[len(tops) // 2], "far edge": tops[-1]}[top]
        for x0 in crop_windows(W, cw):
            jobs.append(Job(sweep_frames(i)[1], axis(w, W, x0, cw), axis(h, H, y0, ch)))
            wants.append(O.lookup(resized(i)[:, y0:y0 + ch, x0:x0 + cw], REF_TABLE).astype(np.float16))
    inside_y = sum(j.y.span_first > 0 for j in jobs)
    inside_x = sum(j.x.span_first > 0 for j in jobs)
    assert inside_x >= 150 and (inside_y == 0 if top == "0" else inside_y >= 150), (inside_x, inside_y)
    out, offsets, probs = call(f"clip top {top}", jobs, _lib.PRE_CLIP, 1, dev)
    compare(f"clip top {top}", out, offsets, wants, probs)


def qwen_targets(pool):
    """[(pair, T, H', W')]: the pairs whose resized size is a multiple of 28 * pool, then every pair resized to the
    multiple of 28 * pool nearest its (H, W) (its (h, w) when that is large), T cycling through 1, 2, 4"""
    f = 28 * pool
    out = [(i, H, W) for i, (h, w, H, W) in enumerate(PAIRS) if H % f == 0 and W % f == 0]
    for i, (h, w, H, W) in enumerate(PAIRS):
        a, b = (max(f, round(v / f) * f) for v in (H, W))
        if a * b > 448 * 448:
            a, b = (max(f, round(v / f) * f) for v in (h, w))
        out.append((i, a, b))
    return [(i, (1, 2, 4)[k % 3], a, b) for k, (i, a, b) in enumerate(out)]


def qwen_frames(i, T):
    """pair i's seeded frames, T of them"""
    h, w, _, _ = PAIRS[i]
    return np.random.default_rng(2000 + i * 7 + T).integers(0, 256, (T, h, w, 3), dtype=np.uint8)


@pytest.mark.parametrize("pool", [1, 2])
def test_qwen_rows_and_codes_equal_oracle(dev, pool):
    jobs, rows, codes = [], [], []
    for i, T, a, b in qwen_targets(pool):
        h, w, _, _ = PAIRS[i]
        f = qwen_frames(i, T)
        jobs.append(Job(torch.from_numpy(f).cuda(), axis(w, b), axis(h, a)))
        r = pillow(f, a, b)
        rows.append(O.qwen_patchify(O.lookup(r, REF_TABLE))[0])
        codes.append(O.qwen_patchify(np.moveaxis(r, -1, 1))[0])
    assert {t for _, t, _, _ in qwen_targets(pool)} == {1, 2, 4} and len(jobs) > 32
    out, offsets, probs = call(f"qwen rows pool {pool}", jobs, _lib.PRE_QWEN, pool, dev)
    compare(f"qwen rows pool {pool}", out, offsets, rows, probs)
    out, offsets, probs = call(f"qwen codes pool {pool}", jobs, _lib.PRE_QWEN_CODES, pool, dev)
    compare(f"qwen codes pool {pool}", out, offsets, codes, probs)


# ---- limits ----------------------------------------------------------------------------------------------------------
def widest_window(in_size, out_size, span):
    """the longest window [1, 1 + count) of in_size -> out_size whose source span is at most `span` columns"""
    lo, hi = 1, out_size - 1
    while lo < hi:
        mid = (lo + hi + 1) // 2
        if P.resample_plan(in_size, out_size, 1, mid)[0].span_count <= span:
            lo = mid
        else:
            hi = mid - 1
    return lo


def refused(jobs, layout, pool, dev, match):
    """fvs_preprocess_multi refuses the table naming `match`, launches nothing and leaves a sentinel output as it was"""
    lib = _lib.load()
    n = len(jobs)
    arr = (_lib.PreprocessJob * n)(*[j.struct() for j in jobs])
    for i, j in enumerate(jobs):
        arr[i].frames = j.frames.data_ptr()
    out = torch.full((1 << 16,), 7, dtype=torch.uint8, device="cuda")
    ws = torch.full((1 << 16,), 7, dtype=torch.uint8, device="cuda")
    torch.cuda.synchronize()
    n0 = lib.fvs_launch_count()
    r = lib.fvs_preprocess_multi(arr, n, dev["table"].data_ptr(), layout, pool, out.data_ptr(), ws.data_ptr(),
                                 ws.numel(), _lib.cur_stream())
    torch.cuda.synchronize()
    assert r == _lib.FVS_EINVAL and match in lib.fvs_last_error().decode(), lib.fvs_last_error()
    assert lib.fvs_launch_count() == n0 and bool((out == 7).all()) and bool((ws == 7).all())


def test_row_span_limit(dev):
    """a window reading 16384 source columns (the 48 KB shared-memory row) runs and is exact; 16385 is refused, alone
    or as the 41st job of a table whose first 40 jobs are good, and in the second stage"""
    rng = np.random.default_rng(5)
    f = rng.integers(0, 256, (2, 3, 16384, 3), dtype=np.uint8)
    whole = Job(torch.from_numpy(f).cuda(), axis(16384, 8191), axis(3, 2))
    assert whole.x.span_count == 16384
    wide = rng.integers(0, 256, (1, 4, 20000, 3), dtype=np.uint8)
    c = widest_window(20000, 17000, 16384)
    crop = Job(torch.from_numpy(wide).cuda(), axis(20000, 17000, 1, c), axis(4, 5))
    assert crop.x.span_count == 16384 and P.resample_plan(20000, 17000, 1, c + 1)[0].span_count == 16385
    out, offsets, probs = call("row span 16384", [whole, crop], _lib.PRE_RGB8, 1, dev)
    compare("row span 16384", out, offsets, [pillow(f, 2, 8191), pillow(wide, 5, 17000)[:, :, 1:1 + c]], probs)
    over = Job(torch.from_numpy(wide).cuda(), axis(20000, 17000, 1, c + 1), axis(4, 5))
    small = [Job(sweep_frames(i)[1], axis(w, W), axis(h, H)) for i, (h, w, H, W) in enumerate(PAIRS[:40])]
    for jobs in ([over], small + [over]):
        refused(jobs, _lib.PRE_RGB8, 1, dev, f"job {len(jobs) - 1}: a window reading 16385 source columns")
    half = torch.from_numpy(np.ascontiguousarray(f[:, :, :8192])).cuda()
    two = Job(half, axis(8192, 16385), axis(3, 3), axis(16385, 100), axis(3, 3))
    refused(small[:3] + [two], _lib.PRE_RGB8, 1, dev, "job 3: a window reading 16385 source columns")


def test_frame_count_limit(dev):
    """T = 65535 frames of 2 x 3 pixels runs (RGB8 and CLIP) and is exact; 65536 is refused with nothing launched"""
    f = np.random.default_rng(6).integers(0, 256, (65535, 2, 3, 3), dtype=np.uint8)
    job = Job(torch.from_numpy(f).cuda(), axis(3, 5), axis(2, 3))
    out, offsets, probs = call("T 65535 rgb8", [job], _lib.PRE_RGB8, 1, dev)
    want = O.resize(f, 3, 5)
    compare("T 65535 rgb8", out, offsets, [want], probs)
    out, offsets, probs = call("T 65535 clip", [job], _lib.PRE_CLIP, 1, dev)
    compare("T 65535 clip", out, offsets, [O.lookup(want, REF_TABLE).astype(np.float16)], probs)
    big = Job(torch.zeros(65536, 2, 3, 3, dtype=torch.uint8, device="cuda"), axis(3, 5), axis(2, 3))
    refused([job, big], _lib.PRE_RGB8, 1, dev, "job 1: 65536 frames in one call (at most 65535)")


def test_one_pixel_axes_in_both_stages(dev):
    """H = 1 and W = 1 as source, first-stage and final sizes, RGB8 and (second stage to 56 x 28) Qwen2-VL codes"""
    rng = np.random.default_rng(8)
    shapes = [((1, 1), (1, 1), (1, 1)), ((1, 9), (1, 1), (4, 1)), ((9, 1), (1, 1), (1, 4)), ((1, 7), (1, 3), (1, 1)),
              ((6, 1), (2, 1), (1, 1)), ((5, 7), (1, 1), (3, 4)), ((5, 7), (1, 4), (3, 1)), ((5, 7), (3, 1), (1, 6)),
              ((1, 1), (7, 5), (1, 1))]
    jobs, wants, qjobs, qwants = [], [], [], []
    for k, ((h, w), (h1, w1), (h2, w2)) in enumerate(shapes):
        f = rng.integers(0, 256, (1 + k % 2 * 3, h, w, 3), dtype=np.uint8)
        d = torch.from_numpy(f).cuda()
        jobs.append(Job(d, axis(w, w1), axis(h, h1), axis(w1, w2), axis(h1, h2)))
        jobs.append(Job(d, axis(w, w2), axis(h, h2)))                       # and in one stage
        wants += [pillow(pillow(f, h1, w1), h2, w2), pillow(f, h2, w2)]
        qjobs.append(Job(d, axis(w, w1), axis(h, h1), axis(w1, 28), axis(h1, 56)))
        qwants.append(O.qwen_patchify(np.moveaxis(pillow(pillow(f, h1, w1), 56, 28), -1, 1))[0])
    out, offsets, probs = call("one-pixel rgb8", jobs, _lib.PRE_RGB8, 1, dev)
    compare("one-pixel rgb8", out, offsets, wants, probs)
    out, offsets, probs = call("one-pixel codes", qjobs, _lib.PRE_QWEN_CODES, 1, dev)
    compare("one-pixel codes", out, offsets, qwants, probs)


# ---- the evaluation drivers' chain at real sizes ---------------------------------------------------------------------
NAMES = list(QS.CASES)


def fetcher(pool):
    return P.Qwen2VLVideoFetcher(P.Qwen2VLFramePreprocessor(QS.PROC_MIN_PIXELS, QS.PROC_MAX_PIXELS, pool))


def sha256(a) -> str:
    return hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest()


def stage2(fx, stage1):
    """(the oracle's fp32 rows, its codes) of the processor on the fetched bytes"""
    h2, w2 = fx.pre.resized(*stage1.shape[1:3])
    r = O.resize(stage1, h2, w2)
    return O.qwen_patchify(O.lookup(r, REF_TABLE))[0], O.qwen_patchify(np.moveaxis(r, -1, 1))[0]


@pytest.mark.parametrize("name", NAMES)
def test_fetcher_at_real_sizes(golden, name):
    f, ele, pool = case(name)
    fx = fetcher(pool)
    got = fx.fetch(dict(ele, video=list(f)))
    picks = [int(v) for v in golden[f"{name}_picks"]]
    h1, w1 = (int(v) for v in golden[f"{name}_size"])
    assert got.is_cuda and tuple(got.shape) == (len(picks), h1, w1, 3)
    got = got.cpu().numpy()
    m = mismatch(got, pillow(f[picks], h1, w1))
    assert m is None, f"{name}: stage 1 against Pillow: {m}"
    assert sha256(got) == str(golden[f"{name}_stage1_sha256"]), name
    rows, codes = stage2(fx, got)
    assert sha256(rows.astype(np.float32)) == str(golden[f"{name}_pixels_sha256"]), f"{name}: the oracle's rows"
    res = fx(dict(ele, video=list(f)))
    assert res["video_grid_thw"].tolist() == [golden[f"{name}_grid"].tolist()]
    m = mismatch(res["pixel_values_videos"].cpu().numpy(), rows)
    assert m is None, f"{name}: rows against the oracle: {m}"
    m = mismatch(fx(dict(ele, video=list(f)), codes=True)["pixel_values_videos"].cpu().numpy(), codes)
    assert m is None, f"{name}: codes against the oracle: {m}"


@pytest.mark.parametrize("codes", [False, True])
def test_fetcher_many_over_every_case(golden, codes):
    """every case twice in one many() call per pool (two-stage jobs of equal sizes in one group) against the golden's
    digests (rows) or the oracle (codes)"""
    for pool in (1, 2):
        names = [n for n in NAMES if QS.CASES[n][3] == pool] * 2
        fx = fetcher(pool)
        res = fx.many([dict(case(n)[1], video=list(case(n)[0])) for n in names], codes=codes)
        out = res["pixel_values_videos"].cpu().numpy()
        assert res["video_grid_thw"].tolist() == [golden[f"{n}_grid"].tolist() for n in names]
        wants = {}
        for n in dict.fromkeys(names) if codes else ():
            f, _, _ = case(n)
            h1, w1 = (int(v) for v in golden[f"{n}_size"])
            wants[n] = stage2(fx, pillow(f[[int(v) for v in golden[f"{n}_picks"]]], h1, w1))[1]
        r = 0
        for k, n in enumerate(names):
            t, gh, gw = golden[f"{n}_grid"].tolist()
            part = out[r:r + t * gh * gw]
            r += t * gh * gw
            if codes:
                m = mismatch(part, wants[n])
                assert m is None, (pool, k, n, m)
            else:
                assert sha256(part) == str(golden[f"{n}_pixels_sha256"]), (pool, k, n)
        assert r == out.shape[0]
