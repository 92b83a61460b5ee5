"""Generate tests/golden/qwen_fetch_sizes.npz by EXECUTING the two steps the reference's Qwen2-VL evaluation drivers run
per video (Flash-VStream-Qwen/inference_mcq_vqa.py:322-330) on CPU, at the frame sizes real videos have (360p to 1080p,
portrait, 4:3, ultra-wide) and with the drivers' default video pixel budget:

- qwen_vl_utils.vision_process.fetch_video, list-of-frames branch (vision_process.py:192-222), unmodified, on PIL
  images built from seeded uint8 arrays (no files, no network);
- FlashVStreamQwen2VLImageProcessor._preprocess (models/vstream_qwen2vl_processor.py:38-157) on the PIL images it
  returns, through make_golden_preprocess.qwen_reference (its import shim and stand-in `self`), with the min / max
  pixels of the drivers' Qwen2-VL checkpoint.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_qwen_fetch_sizes.py

Stored per case, digests only (the frames are seeded noise and the outputs are tens of MB, so the file stays a few kB):
the checksum of the seeded frames, the picks (for each image fetch_video returns, padding included, the index of the
frame it was made from, recorded by wrapping fetch_image for the call), the fetched size (h1, w1), video_grid_thw,
and the SHA-256 of the stage-1 bytes np.stack(fetch_video(ele)) and of pixel_values_videos as float32 bytes."""
from __future__ import annotations

import hashlib
import importlib
import os
import sys
import zlib

import numpy as np
import torch
from PIL import Image

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, "/root/reference/Flash-VStream-Qwen")
sys.dont_write_bytecode = True

from tests.golden.make_golden_preprocess import qwen_reference  # noqa: E402  (installs the import shims)
from tests import qwen_fetch_sizes_inputs as QS  # noqa: E402

vision_process = importlib.import_module("qwen_vl_utils.vision_process")


def sha256(a) -> np.ndarray:
    return np.asarray(hashlib.sha256(np.ascontiguousarray(a).tobytes()).hexdigest())


def fetch_traced(pil, keys):
    """(fetch_video's images, the index into `pil` of the frame each one was made from): fetch_image is wrapped for the
    call to record which frame it was given; the padding repeats the last image object"""
    made = {}
    fetch_image = vision_process.fetch_image

    def traced(ele, *args, **kwargs):
        im = fetch_image(ele, *args, **kwargs)
        made[id(im)] = next(i for i, p in enumerate(pil) if p is ele["image"])
        return im
    vision_process.fetch_image = traced
    try:
        images = vision_process.fetch_video({"type": "video", "video": pil, **keys})
    finally:
        vision_process.fetch_image = fetch_image
    return images, [made[id(im)] for im in images]


def main():
    out = {}
    for name, (seed, shape, keys, pool) in QS.CASES.items():
        f = QS.frames(seed, shape)
        pil = [Image.fromarray(x) for x in f]
        images, picks = fetch_traced(pil, keys)
        out[f"{name}_crc"] = np.int64(zlib.crc32(f.tobytes()))
        out[f"{name}_picks"] = np.asarray(picks, np.int64)
        stage1 = np.stack([np.asarray(im) for im in images])
        out[f"{name}_stage1_sha256"] = sha256(stage1)
        out[f"{name}_size"] = np.asarray(stage1.shape[1:3], np.int64)
        pixels, out[f"{name}_grid"] = qwen_reference(images, QS.PROC_MIN_PIXELS, QS.PROC_MAX_PIXELS, pool)
        out[f"{name}_pixels_sha256"] = sha256(np.ascontiguousarray(pixels, np.float32))
        print(name, out[f"{name}_picks"].tolist(), out[f"{name}_size"].tolist(), out[f"{name}_grid"].tolist())
    path = os.path.join(HERE, "qwen_fetch_sizes.npz")
    np.savez(path, **out)
    print(f"wrote {path} ({os.path.getsize(path) / 1e3:.0f} kB): {len(out)} arrays")


if __name__ == "__main__":
    torch.set_grad_enabled(False)
    main()
