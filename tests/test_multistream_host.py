"""CPU tests of the batched streaming step's host side: fvs_stream_step_multi refuses a bad batch with FVS_EINVAL before any
CUDA call (there is no GPU here, so a CUDA call would fail differently) and leaves every bank counter alone, and the launch
planner fvs_stream_plan gives every job disjoint, ordered blocks at or above its minimum within every launch's budget."""
import ctypes as C

import pytest

from flash_vstream_b200 import _lib as L

CFG = L.StarConfig(1024, 24, 8, 4, 25, 25, 1, 3, 32, 0.2)


def fake_bank(i, *, step=40, chunk_cap=1, n_frames=40, frames_cap=256):
    """a bank struct with dummy (never dereferenced) device pointers, at the steady state of a single-frame stream"""
    base = (i + 1) << 32
    warm = step > 0
    return L.Bank(base + 0x1000, base + 0x2000, base + 0x3000, base + 0x4000, base + 0x5000, frames_cap, chunk_cap,
                  25 if warm else 0, 25 if warm else 0, 4 if warm else 0, n_frames, step)


def jobs_for(banks, frames=1, draws=True):
    lib = L.load()
    ws = lib.fvs_stream_workspace_bytes(C.byref(CFG), banks[0].chunk_cap)
    jobs = (L.StreamJob * len(banks))()
    ntm = L.NtmWeights(0x10, 0x20, 0x30, 0x40)
    for i, b in enumerate(banks):
        jobs[i].bank = C.pointer(b)
        jobs[i].ntm = C.pointer(ntm)
        jobs[i].frames = frames if isinstance(frames, int) else frames[i]
        jobs[i].init_idx = jobs[i].refill_idx = (0x9000 + i) if draws else None
        jobs[i].workspace, jobs[i].workspace_bytes = ((i + 1) << 40), ws
    jobs._keep = (ntm, banks)
    return jobs


def counters(b):
    return (b.n_long, b.n_tur, b.n_cur, b.n_frames, b.step)


def step_multi(jobs, n, max_blocks=0):
    return L.load().fvs_stream_step_multi(C.byref(CFG), jobs, n, None, 0x7000, L.INPUT_FEATURES, None, 0, max_blocks, None)


@pytest.mark.parametrize("case, message", [
    ("duplicate", b"same bank"), ("shared_workspace", b"share a workspace"), ("over_chunk_cap", b"frames per call"),
    ("buffer_full", b"frame buffer full"), ("no_draws", b"draws"), ("small_workspace", b"workspace too small"),
    ("max_blocks", b"at least 2 blocks"),
])
def test_bad_batch_is_refused_before_any_cuda_call(case, message):
    lib = L.load()
    banks = [fake_bank(i) for i in range(4)]
    if case == "buffer_full":
        banks[2].n_frames = banks[2].frames_cap
    jobs = jobs_for(banks, draws=case != "no_draws")
    if case == "duplicate":
        jobs[3].bank = C.pointer(banks[1])
    elif case == "shared_workspace":
        jobs[3].workspace = jobs[0].workspace
    elif case == "over_chunk_cap":
        jobs[1].frames = 2
    elif case == "small_workspace":
        jobs[2].workspace_bytes -= 1
    before = [counters(b) for b in banks]
    rc = step_multi(jobs, 4, max_blocks=1 if case == "max_blocks" else 0)
    assert rc == L.FVS_EINVAL, (rc, lib.fvs_last_error())
    assert message in lib.fvs_last_error(), lib.fvs_last_error()
    assert [counters(b) for b in banks] == before
    assert lib.fvs_launch_count() == 0


def check_plan(banks, frames, budget):
    lib = L.load()
    n = len(banks)
    jobs = jobs_for(banks, frames)
    blocks, wave = (C.c_int32 * (2 * n))(), (C.c_int32 * n)()
    waves = lib.fvs_stream_plan(C.byref(CFG), jobs, n, budget, blocks, wave)
    assert waves > 0, lib.fvs_last_error()
    km, ab, wv = list(blocks[0::2]), list(blocks[1::2]), list(wave[:])
    assert wv == sorted(wv) and wv[0] == 0 and wv[-1] == waves - 1 and set(wv) == set(range(waves))   # in order, no gaps
    for w in range(waves):
        members = [i for i in range(n) if wv[i] == w]
        assert members == list(range(members[0], members[-1] + 1)) and len(members) <= 32
        assert sum(km[i] + ab[i] for i in members) <= budget                    # job ranges are disjoint and fit the launch
    for i, b in enumerate(banks):
        folds = b.step > 0 and b.n_tur + (frames if isinstance(frames, int) else frames[i]) > CFG.tur_len
        assert km[i] >= 1 and ab[i] >= (1 if folds else 0), (i, km[i], ab[i])
        assert ab[i] == 0 or folds
    return km, ab, wv, waves


def test_plan_single_job_is_the_single_stream_grid():
    km, ab, _, waves = check_plan([fake_bank(0)], 1, 132)
    assert waves == 1 and km == [50] and ab == [16]       # K*S/8 = 25*16/8 Lloyd blocks + 16 abstract blocks
    km, ab, _, waves = check_plan([fake_bank(0, step=0, n_frames=0)], 1, 132)
    assert waves == 1 and km == [8] and ab == [0]         # first step: no k-means, no fold


@pytest.mark.parametrize("n, budget, want_waves", [(32, 132, 1), (33, 132, 2), (6, 4, 3), (6, 2, 6), (66, 132, 3), (8, 132, 1)])
def test_plan_packs_jobs_into_few_waves(n, budget, want_waves):
    banks = [fake_bank(i) for i in range(n)]
    km, ab, wv, waves = check_plan(banks, 1, budget)
    assert waves == want_waves
    if n == 8:
        assert sum(km) + sum(ab) == budget        # the spare blocks are all handed out


def test_plan_mixed_positions():
    banks = [fake_bank(0), fake_bank(1, step=0, n_frames=0), fake_bank(2, step=10, n_frames=10)]
    banks[2].n_long = banks[2].n_tur = 10
    check_plan(banks, 1, 132)
    check_plan(banks, 1, 3)
