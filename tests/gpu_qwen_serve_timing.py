"""Measurement script (not a test): cost of publishing the Qwen2-VL streaming memory at full size (60 CSM + 30 DAM frames,
24x24 / 12x12 grids, features 1280, merger 1280 -> 3584 bf16).

  * the writer's per-clip time with and without publication: two hosts on the same clips and draws, stepped alternately,
    CUDA events around each embed_new_video_clip (which ends in the step's read-back);
  * the publish launch alone, and snapshot time / bytes per second on the same GPU (and peer to peer when 2 GPUs exist);
  * the Manager path's per-clip publish (host copies of the 13 items pickled through a Manager list), for comparison.
Prints one JSON line with the card name and power limit; with --out also writes it there.

    python tests/gpu_qwen_serve_timing.py [--clips 24] [--reads 50] [--out qwen_serve_timing.json]
"""
from __future__ import annotations

import argparse
import json
import os
import random
import subprocess
import sys
import time
from statistics import median

import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

T, H, W, DIM = 4, 24, 24, 1280


def card():
    name = torch.cuda.get_device_name(0)
    try:
        limit = subprocess.run(["nvidia-smi", "--query-gpu=power.limit", "--format=csv,noheader", "-i", "0"],
                               capture_output=True, text=True, timeout=30).stdout.strip()
    except Exception as e:     # the number is reported without it, and says so
        limit = f"unknown ({e})"
    return name, limit


def make_host(rt, RI, device):
    gen = {"g": torch.Generator(device=device).manual_seed(7)}

    def encode(patch_rows, total_grid_thw):
        return (torch.randn(T * H * W + T * H * W // 4, DIM, generator=gen["g"], device=device) * 0.5).bfloat16()
    w = {k: v.to(device) for k, v in RI.merger_weights(DIM, 3584, "bf16", 77).items()}
    host = rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(rt.FlashMemory(), rt.PatchMerger.from_weights(w, device=device),
                                                            encode_patches=encode, device=device))
    return host, gen


def timed(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--clips", type=int, default=24)
    ap.add_argument("--reads", type=int, default=50)
    ap.add_argument("--out", default=None)
    args = ap.parse_args()
    assert torch.cuda.is_available(), "this script measures on the GPU"
    torch.set_grad_enabled(False)
    import flash_vstream_b200.qwen.vstream_qwen2vl_realtime as rt
    from flash_vstream_b200.qwen.serve import QwenMemoryReader, export_qwen_memory
    from tests import qwen_rt_inputs as RI
    dev = torch.device("cuda", 0)
    plain, g1 = make_host(rt, RI, dev)
    pubd, g2 = make_host(rt, RI, dev)
    export = export_qwen_memory(pubd, grid=(H, W))
    px, grid = torch.zeros(T * H * W, 1176), torch.tensor([[T, H, W]])
    per = {"plain": [], "published": []}
    for s in range(args.clips):
        order = (("plain", plain), ("published", pubd)) if s % 2 == 0 else (("published", pubd), ("plain", plain))
        for name, host in order:
            torch.manual_seed(100 + s)
            random.seed(100 + s)
            ms = timed(lambda: host.embed_new_video_clip(px, grid, s * T))
            if s >= 16:                               # CSM and DAM full from clip 16 on (64 frames): the steady state
                per[name].append(ms)
    pub = pubd._qwen_publication
    publish_ms = [timed(lambda: pub.publish(pubd.stream_state)) for _ in range(args.reads)][5:]
    ve = pubd.stream_state.video_embeds
    nbytes = ve.numel() * ve.element_size() + 4 * 60 + 8 * 30
    res = {"card": None, "power_limit": None, "rows": int(ve.shape[0]), "dim": int(ve.shape[1]), "bytes": nbytes,
           "clip_ms_plain_median": median(per["plain"]), "clip_ms_published_median": median(per["published"]),
           "clip_ms_plain_mean": sum(per["plain"]) / max(len(per["plain"]), 1),
           "clip_ms_published_mean": sum(per["published"]) / max(len(per["published"]), 1),
           "clips_timed": len(per["plain"]),
           "publish_ms_median": median(publish_ms)}
    for label, rdev in (("same_gpu", 0), ("peer", 1)):
        if rdev >= torch.cuda.device_count():
            res[f"snapshot_{label}"] = "not measured (1 GPU)"
            continue
        try:
            reader = QwenMemoryReader(*export, device=rdev)
        except Exception as e:
            res[f"snapshot_{label}"] = f"refused: {e}"
            continue
        with torch.cuda.device(rdev):
            reader.read()
            ms = [timed(lambda: reader.read()) for _ in range(args.reads)][5:]
        avg = median(ms)
        res[f"snapshot_{label}_ms_median"] = avg
        res[f"snapshot_{label}_GBps"] = nbytes / avg / 1e6
    # the Manager path: the same 13 items as host copies through a Manager list, per clip
    import torch.multiprocessing as mp
    with mp.get_context("spawn").Manager() as manager:
        pubd.video_embedding_memory = manager.list()
        lst = pubd.stream_state.as_list()
        ms = []
        for _ in range(10):
            t0 = time.perf_counter()
            pubd._publish(lst)
            ms.append(1e3 * (time.perf_counter() - t0))
        res["manager_publish_ms"] = sum(ms[2:]) / len(ms[2:])
    res["card"], res["power_limit"] = card()
    line = json.dumps(res)
    print(line)
    if args.out:
        os.makedirs(os.path.dirname(args.out) or ".", exist_ok=True)
        with open(args.out, "w") as f:
            f.write(line + "\n")


if __name__ == "__main__":
    main()
