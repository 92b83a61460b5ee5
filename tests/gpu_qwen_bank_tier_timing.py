"""Timing of the two-tier feature bank of the Qwen2-VL streaming state (not a test):
    python tests/gpu_qwen_bank_tier_timing.py [--prefill 500 5000] [--rounds 4] [--steps 5] > bank_tier_timing.json
A 336 px stream through embed_new_video_clip (32-layer tower, 8-patch clips, memory full: 60 CSM + 30 DAM frames) whose
banks are pre-filled with synthetic features to each --prefill length, once with every frame in HBM
(fvs_bank_device_frames=None) and once with every frame of the full-resolution and merged banks in pinned host memory
(fvs_bank_device_frames=0).  All configurations live side by side and are stepped in alternation (`--steps` clips each per
round).  Per configuration: ms per step (CUDA events around the call), retrieved frames read from the host per step
(median, max), the PCIe bytes that makes, and the HBM the banks hold.  The capped 5000-patch configuration holds about
12.5 GB of pinned host memory."""
import argparse
import json
import os
import subprocess
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from flash_vstream_b200.qwen import vstream_qwen2vl_realtime as rt  # noqa: E402
from flash_vstream_b200.qwen.vision_tower import QwenVisionBlocksB200  # noqa: E402
from tests import qwen_rt_inputs as RI  # noqa: E402
from tests import qwen_vit_inputs as VI  # noqa: E402

T_CLIP = 8


def _gpu_info():
    try:
        return subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                              text=True, timeout=30).stdout.strip()
    except Exception as e:           # the numbers stand without it, but say why it is missing
        return f"unavailable: {e!r}"


def _bank_bytes(st):
    return sum(rb.buf.numel() * rb.buf.element_size() for rb in (st.bank_x, st.bank_small, st.bank_merged)
               if rb.buf is not None)


def _prefill(st, patches):
    """append `patches` temporal patches of synthetic features to the banks (full resolution, half resolution, merged),
    placed by the state's cap — the state of a stream that has run for 2 x patches frames"""
    gd = torch.Generator(device="cuda").manual_seed(1)
    for c0 in range(0, patches, 256):
        n = min(256, patches - c0)
        x = torch.randn(n, 576, 1280, device="cuda", generator=gd).bfloat16()
        m = torch.randn(n, 144, 3584, device="cuda", generator=gd).bfloat16()
        st._append_frames(x, m, x.device)
        st.bank_small.append(torch.randn(n, 144, 1280, device="cuda", generator=gd).bfloat16())
        st.n_frames += n
    torch.cuda.synchronize()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--prefill", type=int, nargs="+", default=[500, 5000])
    ap.add_argument("--rounds", type=int, default=4)
    ap.add_argument("--steps", type=int, default=5)
    ap.add_argument("--depth", type=int, default=32)
    a = ap.parse_args()
    torch.set_grad_enabled(False)
    gpu = _gpu_info()
    sd = VI.state_dict(dict(depth=a.depth, embed=1280, heads=16, seed=5), "bf16")
    tower = QwenVisionBlocksB200(sd, depth=a.depth, heads=16, dtype=torch.bfloat16)
    merger = rt.PatchMerger.from_weights({k: v.cuda() for k, v in RI.merger_weights(1280, 3584, "bf16", 7).items()})
    g = torch.Generator().manual_seed(0)
    scenes = [torch.randn(576, 1176, generator=g) for _ in range(12)]
    n_clips = 60 // T_CLIP + 2 + a.rounds * a.steps
    clips = [torch.cat([scenes[(s * T_CLIP + i) // 5 % 12] + 0.3 * torch.randn(576, 1176, generator=g)
                        for i in range(T_CLIP)]).bfloat16().pin_memory() for s in range(n_clips)]
    thw = torch.tensor([[T_CLIP, 24, 24]])
    frame_bytes = (576 * 1280 + 144 * 3584) * 2
    hosts = {}
    for p in a.prefill:
        for cap in (None, 0):
            host = rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(rt.FlashMemory(), merger, encode_patches=tower))
            host.fvs_bank_device_frames = cap
            torch.manual_seed(0)
            for s in range(60 // T_CLIP + 2):            # fill the memory (60 CSM centroids), then the long bank
                host.embed_new_video_clip(clips[s], thw, s * T_CLIP)
            _prefill(host.stream_state, p)
            hosts[(p, cap)] = {"host": host, "cursor": 60 // T_CLIP + 2, "ms": [], "fetch": []}
    for r in range(a.rounds):
        for key, h in hosts.items():
            host, st = h["host"], h["host"].stream_state
            for i in range(a.steps):
                s = h["cursor"]
                f0 = st.host_fetch_count()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                host.embed_new_video_clip(clips[s], thw, st.n_frames)
                e1.record()
                torch.cuda.synchronize()
                if r or i:                               # the first step of a configuration is its warm-up
                    h["ms"].append(e0.elapsed_time(e1))
                    h["fetch"].append(st.host_fetch_count() - f0)
                h["cursor"] += 1
                if h["cursor"] == len(clips):
                    h["cursor"] = 60 // T_CLIP + 2
    rows = []
    for (p, cap), h in hosts.items():
        st = h["host"].stream_state
        f = np.array(h["fetch"])
        rows.append({"prefill_patches": p, "device_frames": cap, "bank_frames": st.n_frames, "steps_timed": len(h["ms"]),
                     "ms_per_step_median": float(np.median(h["ms"])), "ms_per_step_min": float(np.min(h["ms"])),
                     "host_frames_per_step_median": float(np.median(f)), "host_frames_per_step_max": int(f.max()),
                     "pcie_bytes_per_step_median": float(np.median(f)) * frame_bytes,
                     "pcie_bytes_per_step_max": int(f.max()) * frame_bytes,
                     "hbm_bank_bytes": _bank_bytes(st), "host_bank_bytes": sum(c.numel() * 2 for c in st.host_chunks)})
    print(json.dumps({"gpu": gpu, "depth": a.depth, "t_clip": T_CLIP, "memory_allocated_bytes": torch.cuda.memory_allocated(),
                      "rows": rows}))
    tower.close()


if __name__ == "__main__":
    main()
