"""Generate tests/golden/preprocess.npz by EXECUTING the two reference pre-processing paths on CPU:

- LLaVA: the PIL-backed CLIP image processor of the installed transformers (CLIPImageProcessorPil: Pillow BICUBIC
  shortest-edge resize, center crop, numpy rescale / normalize), what the reference's transformers 4.31
  CLIPImageProcessor.preprocess computes (cli_video_stream.py:186), then .half() as the reference does;
- Qwen2-VL: FlashVStreamQwen2VLImageProcessor._preprocess of the reference (models/vstream_qwen2vl_processor.py:38-157),
  called unbound on a stand-in `self`.

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_preprocess.py

Import shim (reference untouched): the make_golden_qwen.py shim, plus the three names the processor module imports from
transformers' Qwen2-VL image processor that transformers 5.5 no longer defines there (logger, make_batched_images,
make_batched_videos; _preprocess uses only logger), and image_utils.VideoInput, a type alias now in video_utils.  The stand-in `self` carries what _preprocess reads: patch_size 14,
merge_size 2, temporal_patch_size 2, min_pixels, max_pixels and the numpy rescale / normalize of BaseImageProcessor.

Frames are seeded noise (tests/preprocess_inputs.py), stored as seeds with a checksum; outputs are stored whole."""
from __future__ import annotations

import importlib
import os
import sys
import types
import zlib

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.dont_write_bytecode = True

from tests.golden.make_golden_qwen import _quiet  # noqa: E402,F401  (installs the import shim)
import transformers.models.qwen2_vl.image_processing_qwen2_vl as _hf_ip  # noqa: E402
from transformers.utils import logging as _hf_logging  # noqa: E402

for _name in ("make_batched_images", "make_batched_videos"):
    if not hasattr(_hf_ip, _name):
        setattr(_hf_ip, _name, None)
if not hasattr(_hf_ip, "logger"):
    _hf_ip.logger = _hf_logging.get_logger(_hf_ip.__name__)
import transformers.image_utils as _hf_iu  # noqa: E402
if not hasattr(_hf_iu, "VideoInput"):                     # a type alias, moved to transformers.video_utils
    from transformers.video_utils import VideoInput as _VideoInput
    _hf_iu.VideoInput = _VideoInput
ref_proc = importlib.import_module("models.vstream_qwen2vl_processor")

from transformers.image_transforms import normalize, rescale  # noqa: E402
from transformers.image_utils import ChannelDimension, PILImageResampling  # noqa: E402
from transformers.models.clip.image_processing_pil_clip import CLIPImageProcessorPil  # noqa: E402

from tests import preprocess_inputs as PI  # noqa: E402


def clip_reference(frames, shortest_edge, crop):
    proc = CLIPImageProcessorPil(size={"shortest_edge": shortest_edge}, crop_size={"height": crop, "width": crop})
    return proc.preprocess(list(frames), return_tensors="pt")["pixel_values"].half().numpy()


def qwen_reference(frames, min_pixels, max_pixels, pool):
    me = types.SimpleNamespace(
        patch_size=14, merge_size=2, temporal_patch_size=2, min_pixels=min_pixels, max_pixels=max_pixels,
        rescale=lambda image, scale, input_data_format=None, **k: rescale(image, scale, input_data_format=input_data_format),
        normalize=lambda image, mean, std, input_data_format=None, **k: normalize(image, mean, std,
                                                                                  input_data_format=input_data_format))
    patches, grid = ref_proc.FlashVStreamQwen2VLImageProcessor._preprocess(
        me, frames, do_resize=True, resample=PILImageResampling.BICUBIC, do_rescale=True, rescale_factor=1 / 255,
        do_normalize=True, image_mean=PI.OPENAI_CLIP_MEAN, image_std=PI.OPENAI_CLIP_STD, do_convert_rgb=True,
        data_format=ChannelDimension.FIRST, additional_pool_size=pool)
    return np.asarray(patches, dtype=np.float32), np.asarray(grid, dtype=np.int64)


def main():
    out = {}
    for name, (seed, shape, se, crop) in PI.CLIP_CASES.items():
        f = PI.frames(seed, shape)
        out[f"clip_{name}_crc"] = np.int64(zlib.crc32(f.tobytes()))
        out[f"clip_{name}"] = clip_reference(f, se, crop)
    for name, (seed, shape, mn, mx, pool) in PI.QWEN_CASES.items():
        f = PI.frames(seed, shape)
        out[f"qwen_{name}_crc"] = np.int64(zlib.crc32(f.tobytes()))
        out[f"qwen_{name}"], out[f"qwen_{name}_grid"] = qwen_reference(f, mn, mx, pool)
    path = os.path.join(HERE, "preprocess.npz")
    np.savez_compressed(path, **out)
    print(f"wrote {path} ({os.path.getsize(path) / 1e3:.0f} kB): {sorted(out)}")


if __name__ == "__main__":
    torch.set_grad_enabled(False)
    main()
