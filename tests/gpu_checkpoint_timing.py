"""Timing of stream checkpoints (DESIGN.md §3.12): checkpoint (device -> pinned host) and restore (pinned host -> device)
of LLaVA banks of 100 / 1 000 / 10 000 frames at the reference's full size (D = 1024, 8x8 frames, 25 / 25 / 1 memories),
of Qwen2-VL stream states of 100 / 1 000 temporal patches (24x24 grid, 1280-wide features, 3584-wide merged rows, bf16),
and of fvs_bank_restore's restore_kernel alone (the 681-row prefix and header, from pinned host and from device memory).
The states are synthetic (random rows, a full memory): the times depend on bytes only.  Prints one JSON line with the
card name and power limit read in the same run.

    python tests/gpu_checkpoint_timing.py
"""
import ctypes as C
import json
import os
import subprocess
import sys
import time
from types import SimpleNamespace

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from flash_vstream_b200 import _lib as L  # noqa: E402
from flash_vstream_b200 import checkpoint as CK  # noqa: E402
from flash_vstream_b200 import ops  # noqa: E402

REPS = 5


def card():
    try:
        out = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader", "-i", "0"],
                             capture_output=True, text=True, timeout=30).stdout.strip()
        name, limit = [s.strip() for s in out.split(",")]
        return name, limit
    except Exception as e:      # the numbers are still printed; the card is then named by torch only
        return torch.cuda.get_device_name(0), f"unknown ({e.__class__.__name__})"


def timed(fn):
    """median wall time of fn() (each call returns once its copies have landed)"""
    fn()
    ts = []
    for _ in range(REPS):
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        fn()
        torch.cuda.synchronize()
        ts.append(time.perf_counter() - t0)
    return sorted(ts)[len(ts) // 2]


def llava(n_frames):
    cfg = dict(D=1024, grid=24, cur_size=8, long_size=4, long_len=25, tur_len=25, cur_len=1, key_len=3, ntm_dim=32, ratio=0.2)
    w = tuple(torch.zeros(s, dtype=torch.float16, device="cuda") for s in ((32, 1024), (32,), (32, 1024), (32,)))
    bank = ops.StreamBank(cfg, w, chunk_cap=1, frames_cap=n_frames)
    cnt = dict(n_tur=25, n_long=25, n_cur=4, n_frames=n_frames, step=n_frames)
    r = lambda *s: torch.ones(*s, dtype=torch.float16)   # the bytes matter, not their values
    src = CK.llava(CK.star_config(cfg), cnt, r(681, 1024), r(25, 16, 1024), r(25, 1, 1024), r(n_frames, 64, 1024))
    bank.restore(src)
    t_ck = timed(bank.checkpoint)
    ck = bank.checkpoint()
    t_rs = timed(lambda: bank.restore(ck))
    nb = ck.nbytes()
    return {"frames": n_frames, "bytes": nb, "checkpoint_ms": t_ck * 1e3, "restore_ms": t_rs * 1e3,
            "checkpoint_GBps": nb / t_ck / 1e9, "restore_GBps": nb / t_rs / 1e9}


def qwen(n_frames):
    from flash_vstream_b200.qwen.stream_state import QwenStreamState
    from flash_vstream_b200.qwen.vstream_qwen2vl_realtime import FlashMemory
    flash = FlashMemory()                              # 120 / 60 tokens: 60 CSM frames, 30 DAM frames
    merger = SimpleNamespace(dim=3584)                 # restore reads only the merged width
    h = w = 24
    hs = ws = 12
    D, md, dt = 1280, 3584, torch.bfloat16
    n_tem, n_spa = min(60, n_frames), min(30, n_frames)
    r = lambda *s: torch.ones(*s, dtype=dt)         # the bytes matter, not their values
    cfg = {"flash": dict(flash.config), "grid": [h, w], "small_grid": [hs, ws], "dtype": "bfloat16", "dim": D,
           "merger_dim": md}
    cnt = {"n_frames": n_frames, "steps": n_frames, "n_tem": n_tem, "n_spa": n_spa, "fast_steps": n_frames, "redone_steps": 0,
           "merged": 1, "tem_weights_dtype": "float32", "tem_timestamp_dtype": "float32"}
    tensors = {"bank_x": r(n_frames, h * w, D), "bank_small": r(n_frames, hs * ws, D), "bank_merged": r(n_frames, h * w // 4, md),
               "tem_x": r(n_tem * hs * ws, D), "tem_weights": torch.rand(n_tem), "tem_timestamp": torch.rand(n_tem),
               "spa_positions": torch.arange(n_spa), "video_embeds": r(n_spa * h * w // 4 + n_tem * hs * ws // 4, md)}
    src = CK.qwen(cfg, cnt, tensors)
    state = QwenStreamState.restore(src, flash, merger, "cuda")
    t_ck = timed(state.checkpoint)
    ck = state.checkpoint()
    t_rs = timed(lambda: QwenStreamState.restore(ck, flash, merger, "cuda"))
    nb = ck.nbytes()
    return {"temporal_patches": n_frames, "bytes": nb, "checkpoint_ms": t_ck * 1e3, "restore_ms": t_rs * 1e3,
            "checkpoint_GBps": nb / t_ck / 1e9, "restore_GBps": nb / t_rs / 1e9}


def restore_kernel_alone():
    """one fvs_bank_restore with one frame (a 128 KB copy) and the full 681-row prefix: CUDA events around the call"""
    cfg = dict(D=1024, grid=24, cur_size=8, long_size=4, long_len=25, tur_len=25, cur_len=1, key_len=3, ntm_dim=32, ratio=0.2)
    w = tuple(torch.zeros(s, dtype=torch.float16, device="cuda") for s in ((32, 1024), (32,), (32, 1024), (32,)))
    bank = ops.StreamBank(cfg, w, chunk_cap=1)
    lib = L.load()
    out = {}
    for where in ("pinned", "device"):
        pre = torch.randn(681, 1024, dtype=torch.float16)
        pre = pre.pin_memory() if where == "pinned" else pre.cuda()
        fr = torch.randn(1, 64, 1024, dtype=torch.float16).cuda()
        lw = torch.zeros(25, 16, 1024, dtype=torch.float16, device="cuda")
        tw = torch.zeros(25, 1, 1024, dtype=torch.float16, device="cuda")
        ms = []
        for i in range(REPS + 1):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            L.check(lib.fvs_bank_restore(C.byref(bank.cfg), C.byref(bank.bank), 25, 25, 4, 1, 1, pre.data_ptr(), lw.data_ptr(),
                                         tw.data_ptr(), fr.data_ptr(), L.cur_stream()), "fvs_bank_restore")
            e1.record()
            torch.cuda.synchronize()
            if i:
                ms.append(e0.elapsed_time(e1))
        t = sorted(ms)[len(ms) // 2]
        # the two working-set copies (device to device, 0.8 MB) run in the same bracket
        out[where] = {"prefix_bytes": pre.numel() * 2, "call_us": t * 1e3, "prefix_GBps": pre.numel() * 2 / (t * 1e-3) / 1e9}
    return out


def main():
    assert torch.cuda.is_available()
    torch.set_grad_enabled(False)
    name, limit = card()
    res = {"card": name, "power_limit": limit, "llava": [llava(n) for n in (100, 1000, 10000)],
           "qwen": [qwen(n) for n in (100, 1000)], "restore_kernel": restore_kernel_alone()}
    print(json.dumps(res))


if __name__ == "__main__":
    main()
