"""Generate tests/golden/qwen_fetch.npz by EXECUTING the two steps the reference's Qwen2-VL evaluation drivers run per
video (Flash-VStream-Qwen/inference_mcq_vqa.py:322-330) on CPU:

- qwen_vl_utils.vision_process.fetch_video, list-of-frames branch (vision_process.py:192-222), unmodified, on PIL
  images built from seeded uint8 arrays (no files, no network);
- FlashVStreamQwen2VLImageProcessor._preprocess (models/vstream_qwen2vl_processor.py:38-157) on the PIL images it
  returns, through make_golden_preprocess.qwen_reference (its import shim and stand-in `self`), with the min / max
  pixels of the drivers' Qwen2-VL checkpoint.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_qwen_fetch.py

Stored per case: the checksum of the seeded frames, the fetched size (h1, w1), the stage-1 bytes
np.stack(fetch_video(ele)) without the even-count padding (the padding repeats the last image, so the tests repeat the
last frame), the SHA-256 of pixel_values_videos as float32 bytes and video_grid_thw; for the ratio case, the
ValueError's message.  The rows are a function of the stage-1 bytes, so the tests recompute them with the oracle and
hold those, and the device's rows, to the reference's digest; the frames are seeded noise, which does not compress, and
the stored rows would be the bulk of the file."""
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
from tests import qwen_fetch_inputs as QF  # noqa: E402

vision_process = importlib.import_module("qwen_vl_utils.vision_process")


def fetch_reference(seed, shape, keys):
    f = QF.frames(seed, shape)
    return f, vision_process.fetch_video({"type": "video", "video": [Image.fromarray(x) for x in f], **keys})


def main():
    out = {}
    for name, (seed, shape, keys, pool) in QF.CASES.items():
        f, images = fetch_reference(seed, shape, keys)
        out[f"{name}_crc"] = np.int64(zlib.crc32(f.tobytes()))
        stage1 = np.stack([np.asarray(im) for im in images])
        unpadded = len(stage1) - 1 if len(images) > 1 and images[-1] is images[-2] else len(stage1)
        assert all((stage1[i] == stage1[unpadded - 1]).all() for i in range(unpadded, len(stage1)))
        out[f"{name}_stage1"] = stage1[:unpadded]
        out[f"{name}_size"] = np.asarray(stage1.shape[1:3], np.int64)
        pixels, out[f"{name}_grid"] = qwen_reference(images, QF.PROC_MIN_PIXELS, QF.PROC_MAX_PIXELS, pool)
        out[f"{name}_pixels_sha256"] = np.asarray(hashlib.sha256(np.ascontiguousarray(pixels, np.float32).tobytes())
                                                  .hexdigest())
    seed, shape, keys, _ = QF.RATIO_CASE
    try:
        fetch_reference(seed, shape, keys)
        raise AssertionError("the ratio case did not raise")
    except ValueError as e:
        out["ratio_error"] = np.asarray(str(e))
    path = os.path.join(HERE, "qwen_fetch.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path) / 1e3:.0f} kB): {sorted(out)}")


if __name__ == "__main__":
    torch.set_grad_enabled(False)
    main()
