"""Measure the Qwen2-VL evaluation drivers' pre-processing of one video: the CPU steps against Qwen2VLVideoFetcher.

    python tests/gpu_qwen_fetch_timing.py [--frames 768] [--reps 3] [--depth 32] [--out result.json]

One list of `frames` decoded uint8 host frames (16 distinct seeded frames, repeated) at 1280x720 and at 640x360, the
drivers' default fetch_video keys (none besides 'video') and the image processor of their Qwen2-VL checkpoint
(min_pixels 56*56, max_pixels 28*28*16384) with additional_pool_size 2.

- cpu: what the drivers run per video (inference_mcq_vqa.py:322-333), restated with the same libraries: fetch_image's
  Pillow resize of every picked frame (.convert('RGB').resize), then the image processor's transformers resize,
  rescale, normalize and the patchify, then the copy of the fp32 rows to the GPU.  Single-threaded, as the drivers
  run it; the host's core count is reported.
- gpu: Qwen2VLVideoFetcher(ele), from the host frames to the rows on the device (the host stacks the picks into pinned
  memory, copies them, and two launch pairs run), timed with a host clock around a call that ends in a device
  synchronise, and with CUDA events around the same call.
- forward: VisualB200.forward (a bf16 tower of `depth` blocks, seeded weights, the default memory) on the rows.

The GPU rows are checked bit for bit against the CPU rows at every size."""
from __future__ import annotations

import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import numpy as np
import torch
from PIL import Image

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from tests import preprocess_oracle as O  # noqa: E402
from tests import qwen_offline_inputs as OI  # noqa: E402
from tests import qwen_vit_inputs as VI  # noqa: E402
from tests.qwen_fetch_inputs import PROC_MAX_PIXELS, PROC_MIN_PIXELS  # noqa: E402

POOL = 2


def cpu_chain(ele, pre):
    """fetch_video's list branch with fetch_image's Pillow resize, then the processor's steps, then the copy"""
    from transformers.image_transforms import normalize, rescale, resize
    from transformers.image_utils import ChannelDimension, PILImageResampling
    from flash_vstream_b200 import preprocess as P
    video = ele["video"]
    picks = P.fetch_video_picks(len(video), ele)
    images = {}
    for i in sorted(set(picks)):
        im = Image.fromarray(video[i]).convert("RGB")
        h1, w1 = P.fetch_video_size(im.height, im.width, len(video), ele)
        images[i] = im.resize((w1, h1))
    h2, w2 = pre.resized(h1, w1)
    out = []
    for i in picks:
        x = resize(np.asarray(images[i]), size=(h2, w2), resample=PILImageResampling.BICUBIC,
                   input_data_format=ChannelDimension.LAST)
        x = rescale(x, 1 / 255, input_data_format=ChannelDimension.LAST)
        x = normalize(x, P.OPENAI_CLIP_MEAN, P.OPENAI_CLIP_STD, input_data_format=ChannelDimension.LAST)
        out.append(x.transpose(2, 0, 1))
    rows, grid = O.qwen_patchify(np.asarray(out))
    return torch.from_numpy(rows).cuda(), grid


def clock(fn):
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    out = fn()
    torch.cuda.synchronize()
    return (time.perf_counter() - t0) * 1e3, out


def events(fn):
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    torch.cuda.synchronize()
    a.record()
    out = fn()
    b.record()
    torch.cuda.synchronize()
    return a.elapsed_time(b), out


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", type=int, default=768)
    ap.add_argument("--reps", type=int, default=3)
    ap.add_argument("--depth", type=int, default=32)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    assert torch.cuda.is_available(), "this measurement needs a GPU"
    torch.set_grad_enabled(False)
    from flash_vstream_b200 import preprocess as P
    from flash_vstream_b200.qwen import vision_tower, vstream_qwen2vl_model as M, vstream_qwen2vl_realtime as rt
    fetcher = P.Qwen2VLVideoFetcher(P.Qwen2VLFramePreprocessor(PROC_MIN_PIXELS, PROC_MAX_PIXELS, POOL))
    tower = vision_tower.QwenVisionBlocksB200(VI.state_dict(dict(depth=a.depth, embed=1280, seed=7), "bf16"),
                                              depth=a.depth, heads=16, dtype=torch.bfloat16)
    mw = OI.merger_weights("bf16", out=3584)
    merger = rt.PatchMerger.from_weights({"ln_w": mw["ln_q.weight"], "ln_b": mw["ln_q.bias"], "fc1_w": mw["mlp.0.weight"],
                                          "fc1_b": mw["mlp.0.bias"], "fc2_w": mw["mlp.2.weight"], "fc2_b": mw["mlp.2.bias"]})
    fm = M.FlashMemory()
    visual = rt.VisualB200(fm, merger, encode_patches=tower)
    sizes = {}
    for H, W in ((720, 1280), (360, 640)):
        distinct = np.random.default_rng(H).integers(0, 256, (16, H, W, 3), dtype=np.uint8)
        ele = {"type": "video", "video": [distinct[i % 16] for i in range(a.frames)]}
        want, grid = cpu_chain(ele, fetcher.pre)                  # warm-up, and the rows the GPU must give
        got = fetcher(ele)
        identical = torch.equal(got["pixel_values_videos"], want) and got["video_grid_thw"].tolist() == [list(grid)]
        thw = got["video_grid_thw"].cuda()
        pos, vis = OI.positions([OI.n_visual(tuple(grid), fm.temporal_length, fm.spatial_length)])
        pos, vis = pos.cuda(), vis.cuda()
        px = got["pixel_values_videos"].bfloat16()
        del got, want
        visual(px, thw, pos.clone(), vis)
        ms = {"cpu": [], "gpu": [], "gpu_events": [], "forward": []}
        for _ in range(a.reps):
            ms["cpu"].append(clock(lambda: cpu_chain(ele, fetcher.pre))[0])
            ms["gpu"].append(clock(lambda: fetcher(ele))[0])
            ms["gpu_events"].append(events(lambda: fetcher(ele))[0])
            ms["forward"].append(clock(lambda: visual(px, thw, pos.clone(), vis))[0])
        med = {k: statistics.median(v) for k, v in ms.items()}
        sizes[f"{W}x{H}"] = dict(identical=identical, grid=list(grid), fetched=list(P.fetch_video_size(H, W, a.frames, ele)),
                                 ms=ms, median_ms=med, speedup=med["cpu"] / med["gpu"],
                                 cpu_share_of_cpu_plus_forward=med["cpu"] / (med["cpu"] + med["forward"]),
                                 gpu_share_of_gpu_plus_forward=med["gpu"] / (med["gpu"] + med["forward"]))
        del px
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm,clocks.sm", "--format=csv,noheader"],
                         capture_output=True, text=True).stdout.strip()
    res = dict(gpu=smi, host_cores=os.cpu_count(), frames=a.frames, depth=a.depth, pool=POOL, sizes=sizes)
    print(json.dumps(res))
    if a.out:
        with open(a.out, "w") as f:
            json.dump(res, f, indent=1)
    tower.close()


if __name__ == "__main__":
    main()
