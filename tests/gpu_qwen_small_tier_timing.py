"""Timing of the half-resolution host tier of the Qwen2-VL streaming state (not a test):
    python tests/gpu_qwen_small_tier_timing.py [--prefill 732 5232] [--metric cosine] [--rounds 3] [--steps 4] > out.json
The setup of gpu_qwen_bank_tier_timing.py: a 336 px stream through embed_new_video_clip (32-layer tower, 8-patch clips,
memory full: 60 CSM + 30 DAM frames) whose banks are pre-filled with synthetic features to each --prefill length, for
(small_device_frames, device_frames) in (None, None), (None, 0) and (0, 0), with spatial_method klarge_retrieve (or
klarge_retrieve_cos: --metric cosine).  All configurations live side by side and are stepped in alternation (`--steps`
clips each per round).
Per configuration: ms per step (CUDA events around the call), the host bytes the retrieval sweeps per step, the retrieval
alone (CUDA events around one klarge_retrieve over the state's bank after each step, same centroids as the step) and its
achieved host-read rate, and the bank bytes in HBM and in pinned memory.  The (0, 0) configuration at 5232 patches holds
about 15 GB of pinned host memory, the (None, None) one up to twice its 15 GB of banks in HBM (capacity doubling)."""
import argparse
import json
import os
import sys

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from flash_vstream_b200 import ops as O  # noqa: E402
from flash_vstream_b200.qwen import ops as Q  # noqa: E402
from flash_vstream_b200.qwen import vstream_qwen2vl_realtime as rt  # noqa: E402
from flash_vstream_b200.qwen.vision_tower import QwenVisionBlocksB200  # noqa: E402
from tests import qwen_rt_inputs as RI  # noqa: E402
from tests import qwen_vit_inputs as VI  # noqa: E402
from tests.gpu_qwen_bank_tier_timing import T_CLIP, _gpu_info  # noqa: E402

SMALL_FRAME = 144 * 1280 * 2          # bytes of one half-resolution temporal patch at 336 px


def _prefill(st, patches):
    """append `patches` temporal patches of synthetic features to the three banks, placed by the state's two caps"""
    gd = torch.Generator(device="cuda").manual_seed(1)
    for c0 in range(0, patches, 256):
        n = min(256, patches - c0)
        x = torch.randn(n, 576, 1280, device="cuda", generator=gd).bfloat16()
        m = torch.randn(n, 144, 3584, device="cuda", generator=gd).bfloat16()
        st._append_frames(x, m, x.device)
        st._append_small(torch.randn(n, 144, 1280, device="cuda", generator=gd).bfloat16(), x.device)
        st.n_frames += n
    torch.cuda.synchronize()


def _bytes(st):
    hbm = sum(rb.buf.numel() * rb.buf.element_size() for rb in (st.bank_x, st.bank_small, st.bank_merged)
              if rb.buf is not None)
    host = sum(c.numel() * c.element_size() for c in st.host_chunks + st.small_chunks)
    return hbm, host


def _retrieval_ms(st):
    """one klarge retrieval of the step's kind over the state's bank (the 30 heaviest centroids), timed alone"""
    flash = st.flash
    D = st.tem_x.shape[-1]
    heaviest = O.argsort_desc(st.tem_weights)[: flash.spatial_length]
    metric = "cosine" if flash.spatial_method == "klarge_retrieve_cos" else "euclidean"
    tem = st.tem_x.reshape(st.n_tem, -1)
    bank = st._small_bank(D, st.tem_x.device)
    bank = bank.reshape(st.n_frames, -1) if torch.is_tensor(bank) else bank
    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    e0.record()
    Q.klarge_retrieve(tem, heaviest, bank, metric=metric)
    e1.record()
    torch.cuda.synchronize()
    return e0.elapsed_time(e1)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--prefill", type=int, nargs="+", default=[732, 5232])
    ap.add_argument("--rounds", type=int, default=3)
    ap.add_argument("--steps", type=int, default=4)
    ap.add_argument("--depth", type=int, default=32)
    ap.add_argument("--metric", choices=["euclidean", "cosine"], default="euclidean")
    a = ap.parse_args()
    torch.set_grad_enabled(False)
    gpu = _gpu_info()
    sd = VI.state_dict(dict(depth=a.depth, embed=1280, heads=16, seed=5), "bf16")
    tower = QwenVisionBlocksB200(sd, depth=a.depth, heads=16, dtype=torch.bfloat16)
    merger = rt.PatchMerger.from_weights({k: v.cuda() for k, v in RI.merger_weights(1280, 3584, "bf16", 7).items()})
    g = torch.Generator().manual_seed(0)
    scenes = [torch.randn(576, 1176, generator=g) for _ in range(12)]
    fill = 60 // T_CLIP + 2
    n_clips = fill + a.rounds * a.steps
    clips = [torch.cat([scenes[(s * T_CLIP + i) // 5 % 12] + 0.3 * torch.randn(576, 1176, generator=g)
                        for i in range(T_CLIP)]).bfloat16().pin_memory() for s in range(n_clips)]
    thw = torch.tensor([[T_CLIP, 24, 24]])
    method = {"euclidean": "klarge_retrieve", "cosine": "klarge_retrieve_cos"}[a.metric]
    configs = [(p, small, cap, method) for p in a.prefill for small, cap in ((None, None), (None, 0), (0, 0))]
    hosts = {}
    for key in configs:
        p, small, cap, _ = key
        host = rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(rt.FlashMemory(flash_memory_spatial_method=method), merger,
                                                                encode_patches=tower))
        host.fvs_bank_device_frames, host.fvs_bank_small_device_frames = cap, small
        torch.manual_seed(0)
        for s in range(fill):                        # fill the memory (60 CSM centroids), then the long bank
            host.embed_new_video_clip(clips[s], thw, s * T_CLIP)
        _prefill(host.stream_state, p)
        hosts[key] = {"host": host, "cursor": fill, "ms": [], "sweep_ms": []}
    for r in range(a.rounds):
        for key, h in hosts.items():
            host, st = h["host"], h["host"].stream_state
            for i in range(a.steps):
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                host.embed_new_video_clip(clips[h["cursor"]], thw, st.n_frames)
                e1.record()
                torch.cuda.synchronize()
                sweep = _retrieval_ms(st)
                if r or i:                               # the first step of a configuration is its warm-up
                    h["ms"].append(e0.elapsed_time(e1))
                    h["sweep_ms"].append(sweep)
                h["cursor"] += 1
                if h["cursor"] == len(clips):
                    h["cursor"] = fill
    rows = []
    for (p, small, cap, method), h in hosts.items():
        st = h["host"].stream_state
        passes = 2 if method == "klarge_retrieve_cos" else 1
        host_bytes = st.n_small_host * SMALL_FRAME * passes           # swept over PCIe per step, at the final bank length
        sweep = float(np.median(h["sweep_ms"]))
        hbm, pinned = _bytes(st)
        rows.append({"prefill_patches": p, "small_device_frames": small, "device_frames": cap, "spatial_method": method,
                     "bank_frames": st.n_frames, "steps_timed": len(h["ms"]),
                     "ms_per_step_median": float(np.median(h["ms"])), "ms_per_step_min": float(np.min(h["ms"])),
                     "host_bytes_per_step": host_bytes, "retrieval_ms_median": sweep,
                     "retrieval_ms_min": float(np.min(h["sweep_ms"])),
                     "retrieval_host_gb_per_s": host_bytes / sweep / 1e6 if host_bytes else None,
                     "hbm_bank_bytes": hbm, "pinned_bank_bytes": pinned})
    print(json.dumps({"gpu": gpu, "depth": a.depth, "t_clip": T_CLIP, "memory_allocated_bytes": torch.cuda.memory_allocated(),
                      "rows": rows}))
    tower.close()


if __name__ == "__main__":
    main()
