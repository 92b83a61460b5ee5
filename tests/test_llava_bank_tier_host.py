"""CPU tests of the LLaVA bank's device window (DESIGN.md §3.14): the placement arithmetic of a capped frame buffer at its
boundaries, the minimum window and its refusals (in Python and in the C ABI, before any CUDA call), and the ctypes
`Bank` layout against include/fvs_b200.h."""
import ctypes as C
import os
import shutil
import subprocess

import pytest

from flash_vstream_b200 import _lib as L
from flash_vstream_b200 import host_tier as HT
from flash_vstream_b200 import ops

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
CFG = dict(D=1024, grid=24, cur_size=8, long_size=4, long_len=25, tur_len=25, cur_len=1, key_len=3, ntm_dim=32, ratio=0.2)
SC = L.StarConfig(1024, 24, 8, 4, 25, 25, 1, 3, 32, 0.2)


def frame_row(g, clip_first, window):
    """frame_row of csrc/stream_kernels.cu, restated: the row of `frames` holding global frame g"""
    return g if window == 0 or g < window else window + g - max(clip_first, window)


def test_minimum_window():
    assert ops.min_device_frames(CFG, 1) == 26                 # max(25, 1) + 1: the default config, one frame per step
    assert ops.min_device_frames(CFG, 32) == 64                # max(25, 32) + 32: 32-frame clips
    assert ops.min_device_frames(dict(CFG, long_len=0), 4) == 8
    assert ops.device_window(CFG, 1, None) is None
    assert ops.device_window(CFG, 1, 26) == 26
    for bad, msg in ((25, "25 < 26"), (0, "0 < 26"), (-1, ">= 0"), (2.0, "integer"), (True, "integer")):
        with pytest.raises(ValueError, match=msg):
            ops.device_window(CFG, 1, bad)
    with pytest.raises(ValueError, match="fvs_bank_device_frames 63 < 64"):
        ops.device_window(CFG, 32, 63, "fvs_bank_device_frames")


@pytest.mark.parametrize("window, chunk_cap", [(26, 1), (31, 1), (64, 32), (69, 32)])
def test_placement_at_the_boundaries(window, chunk_cap):
    """every clip of a stream whose clip lengths hit the window exactly, straddle it and lie past it (the first clip
    longer than long_len when chunk_cap = 32): device rows are contiguous per clip and inside [0, window + chunk_cap),
    frames below the window keep their index, and the host spans (HT.placement) hold exactly the frames at or past it,
    in order, with no gap or overlap"""
    lens = [chunk_cap] if chunk_cap == 1 else [32, 7, 19, 1, 32, 25, 3, 32, 32, 11]
    per_chunk = 5
    n0, host, k = 0, [], 0
    while n0 < 3 * window:
        t = lens[k % len(lens)]
        k += 1
        rows = [frame_row(g, n0, window) for g in range(n0, n0 + t)]
        assert rows == list(range(rows[0], rows[0] + t)), "a clip is contiguous in `frames`"
        assert rows[0] == min(n0, window) and rows[-1] < window + chunk_cap
        assert all(r == g for r, g in zip(rows, range(n0, n0 + t)) if g < window)
        spans = HT.placement(n0, t, window, per_chunk)
        dev = [s for s in spans if s[0] < 0]
        assert sum(s[3] for s in dev) == max(0, min(t, window - n0))
        for c, dst, s, cnt in spans:
            if c >= 0:
                for i in range(cnt):
                    g = n0 + s + i
                    assert g >= window and rows[s + i] >= window          # a host frame is read from the slot
                    host.append((g, c * per_chunk + dst + i))
        n0 += t
    assert [h for _, h in host] == list(range(n0 - window))                # host frame g - window, in order
    assert [g for g, _ in host] == list(range(window, n0))


def test_cap_met_exactly():
    """a clip that ends exactly at the window keeps everything on the device; the next frame is host frame 0"""
    assert HT.placement(20, 6, 26, 2048) == [(-1, 20, 0, 6)]
    assert HT.placement(26, 1, 26, 2048) == [(0, 0, 0, 1)]
    assert frame_row(26, 26, 26) == 26 and frame_row(27, 27, 26) == 26      # the slot's first row, every step
    assert HT.placement(60, 32, 64, 2048) == [(-1, 60, 0, 4), (0, 0, 4, 28)]  # straddling: 4 device, 28 host frames
    assert [frame_row(g, 60, 64) for g in (60, 63, 64, 91)] == [60, 63, 64, 91]
    assert [frame_row(g, 64, 64) for g in (64, 95)] == [64, 95]
    assert [frame_row(g, 96, 64) for g in (96, 127)] == [64, 95]


def fake_bank(*, chunk_cap=1, frames_cap=27, window=26):
    base = 1 << 32
    return L.Bank(base + 0x1000, base + 0x2000, base + 0x3000, base + 0x4000, base + 0x5000, frames_cap, chunk_cap,
                  7, 8, 2, 40, 40, window)


@pytest.mark.parametrize("window, frames_cap, message", [
    (25, 27, b"frames_window 25 < 26"), (-3, 27, b"frames_window -3 < 26"), (26, 26, b"frames_cap 26 < frames_window 26"),
])
def test_step_refuses_a_bad_window_before_any_cuda_call(window, frames_cap, message):
    lib = L.load()
    bank = fake_bank(window=window, frames_cap=frames_cap)
    n0 = lib.fvs_launch_count()
    ws = C.create_string_buffer(16)
    rc = lib.fvs_stream_step(C.byref(SC), C.byref(bank), None, None, C.c_void_p(0xE000), L.INPUT_FEATURES, 1, None, None,
                             None, 0, C.cast(ws, C.c_void_p), 1 << 30, None)
    assert rc != 0 and message in lib.fvs_last_error()
    assert lib.fvs_launch_count() == n0 and (bank.n_frames, bank.step) == (40, 40)


@pytest.mark.parametrize("window, frames_cap, message", [
    (25, 27, b"frames_window 25 < 26"), (26, 26, b"frames_cap 26 < frames_window 26"),
])
def test_restore_refuses_a_bad_window_before_any_cuda_call(window, frames_cap, message):
    lib = L.load()
    bank = fake_bank(window=window, frames_cap=frames_cap)
    n0 = lib.fvs_launch_count()
    rc = lib.fvs_bank_restore(C.byref(SC), C.byref(bank), 25, 25, 4, 1000, 1000, 0xA000, 0xB000, 0xC000, 0xD000, None)
    assert rc != 0 and message in lib.fvs_last_error()
    assert lib.fvs_launch_count() == n0 and (bank.n_frames, bank.step, bank.n_long) == (40, 40, 7)


def test_uncapped_restore_still_bounded_by_frames_cap():
    lib = L.load()
    bank = fake_bank(window=0, frames_cap=256)
    rc = lib.fvs_bank_restore(C.byref(SC), C.byref(bank), 25, 25, 4, 257, 257, 0xA000, 0xB000, 0xC000, 0xD000, None)
    assert rc != 0 and b"257 frames > frames_cap 256" in lib.fvs_last_error()


def test_bank_struct_layout_matches_the_header(tmp_path):
    fields = [n for n, _ in L.Bank._fields_]
    assert fields[-1] == "frames_window" and C.sizeof(L.Bank) == 88 and L.Bank.frames_window.offset == 80
    cc = shutil.which("cc") or shutil.which("gcc")
    if cc is None:
        pytest.skip("no C compiler to read the header's layout")
    src = tmp_path / "layout.c"
    src.write_text('#include <stdio.h>\n#include <stddef.h>\n#include "fvs_b200.h"\nint main(void) {\n'
                   + "".join(f'  printf("%zu\\n", offsetof(fvs_bank, {n}));\n' for n in fields)
                   + '  printf("%zu\\n", sizeof(fvs_bank));\n  return 0;\n}\n')
    exe = tmp_path / "layout"
    r = subprocess.run([cc, "-I", os.path.join(ROOT, "include"), "-I", "/usr/local/cuda/include", str(src), "-o", str(exe)],
                       capture_output=True, text=True)
    if r.returncode != 0:
        pytest.skip(f"the header does not compile standalone here: {r.stderr[:200]}")
    got = [int(v) for v in subprocess.run([str(exe)], capture_output=True, text=True, check=True).stdout.split()]
    assert got == [getattr(L.Bank, n).offset for n in fields] + [C.sizeof(L.Bank)]
