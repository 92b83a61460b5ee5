"""Measure the offline Qwen2-VL vision pass (VisualB200.forward) against the unpruned composition it is bit-identical to.

    python tests/gpu_qwen_offline_timing.py [--t 384] [--depth 32] [--reps 3] [--out result.json]

One video of t temporal patches (768 frames at the default) on the CLI's 32x32 grid (max_pixels = 4*224*224), a bf16
tower of `depth` blocks at the Qwen2-VL width with seeded random weights, the default memory (60 CSM centroids, 30 DAM
frames).  The pruned pass encodes t*256 + 30*1024 tower rows, the unpruned one t*(1024 + 256).  The two run alternately,
after one warm-up of each; every timing is a host clock around a call that ends in a device synchronise."""
from __future__ import annotations

import argparse
import json
import os
import random
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tests import qwen_offline_inputs as OI  # noqa: E402
from tests import qwen_vit_inputs as VI  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--t", type=int, default=384)
    ap.add_argument("--depth", type=int, default=32)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    torch.set_grad_enabled(False)
    from flash_vstream_b200.qwen import vision_tower, vstream_qwen2vl_model as M, vstream_qwen2vl_realtime as rt
    t, h, w = a.t, 32, 32
    tower = vision_tower.QwenVisionBlocksB200(VI.state_dict(dict(depth=a.depth, embed=1280, seed=7), "bf16"), depth=a.depth,
                                              heads=16, dtype=torch.bfloat16)
    mw = OI.merger_weights("bf16", out=3584)
    merger = rt.PatchMerger.from_weights({"ln_w": mw["ln_q.weight"], "ln_b": mw["ln_q.bias"], "fc1_w": mw["mlp.0.weight"],
                                          "fc1_b": mw["mlp.0.bias"], "fc2_w": mw["mlp.2.weight"], "fc2_b": mw["mlp.2.bias"]})
    fm = M.FlashMemory()
    visual = rt.VisualB200(fm, merger, encode_patches=tower)
    g = torch.Generator(device="cuda").manual_seed(11)
    px = (torch.randn(t * h * w, 1176, generator=g, device="cuda") * 1.2).bfloat16()
    thw = torch.tensor([[t, h, w]], device="cuda")
    pos, vis = OI.positions([OI.n_visual((t, h, w), fm.temporal_length, fm.spatial_length)])
    pos, vis = pos.cuda(), vis.cuda()

    def pruned():
        return visual(px, thw, pos.clone(), vis)

    def unpruned():
        feats, _, small_thw = visual.forward_simple_not_merge(px, thw)
        mem, p = fm.forward(feats, thw, small_thw, pos.clone(), vis)
        return merger(mem), p

    def timed(fn, seed):
        torch.manual_seed(seed)
        random.seed(seed)
        torch.cuda.synchronize()
        t0 = time.perf_counter()
        out = fn()
        torch.cuda.synchronize()
        return (time.perf_counter() - t0) * 1e3, out

    peaks, outs = {}, {}
    for name, fn in (("pruned", pruned), ("unpruned", unpruned)):        # warm-up, identity and peak memory
        torch.cuda.reset_peak_memory_stats()
        base = torch.cuda.memory_allocated()
        _, outs[name] = timed(fn, 3)
        peaks[name] = (torch.cuda.max_memory_allocated() - base) / 2 ** 30
    identical = all(torch.equal(x, y) for x, y in zip(outs["pruned"], outs["unpruned"]))
    del outs
    ms = {"pruned": [], "unpruned": []}
    for r in range(a.reps):
        for name, fn in (("pruned", pruned), ("unpruned", unpruned)):
            ms[name].append(timed(fn, 3)[0])
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    rows = {"pruned": t * h * w // 4 + min(t, fm.spatial_length) * h * w, "unpruned": t * (h * w + h * w // 4)}
    res = dict(gpu=smi, t=t, frames=2 * t, grid=[h, w], depth=a.depth, identical=identical, tower_rows=rows,
               token_ratio=rows["unpruned"] / rows["pruned"], peak_gib=peaks,
               ms=ms, median_ms={k: statistics.median(v) for k, v in ms.items()},
               temporal_patches_per_s={k: t / statistics.median(v) * 1e3 for k, v in ms.items()})
    res["speedup"] = res["median_ms"]["unpruned"] / res["median_ms"]["pruned"]
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    tower.close()


if __name__ == "__main__":
    main()
