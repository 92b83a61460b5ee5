"""Seeded frame lists at the sizes real videos have, and the cases of tests/golden/qwen_fetch_sizes.npz
(make_golden_qwen_fetch_sizes.py): qwen_vl_utils.fetch_video on a list of frames with the video pixel budget the
evaluation drivers use, then FlashVStreamQwen2VLImageProcessor on what it returns."""
from __future__ import annotations

from tests import preprocess_inputs as PI
from tests.qwen_fetch_inputs import PROC_MAX_PIXELS, PROC_MIN_PIXELS  # noqa: F401  (the drivers' processor)

# name -> (seed, (frames in the list, H, W), fetch_video keys besides 'video', additional_pool_size).  No key: the
# default budget (VIDEO_MIN_PIXELS, VIDEO_MAX_PIXELS, VIDEO_TOTAL_PIXELS / nframes).  The comments give fetch_image's
# resize (stage 1), then the processor's (stage 2).
CASES = {
    "360p": (61, (4, 360, 640), {}, 2),                        # 364x644 -> 336x672
    "480p": (62, (16, 480, 854), {}, 2),                       # 476x840 -> 448x840
    "720p": (63, (8, 720, 1280), {}, 2),                       # 560x1008 (the VIDEO_MAX_PIXELS cap) -> 560x1008
    "1080p": (64, (16, 1080, 1920), {}, 1),                    # 560x1008 -> 560x1008
    "portrait": (65, (2, 1920, 1080), {}, 2),                  # 1008x560 -> 1008x560
    "4:3": (66, (6, 768, 1024), {}, 1),                        # 672x896 -> 672x896
    "ultrawide": (67, (3, 1080, 2560), {}, 2),                 # 3 frames, padded to 4; 504x1176 -> 504x1176
    "max_frames": (68, (12, 720, 1280), {"max_frames": 5}, 1),             # 4 of 12 frames picked; 560x1008
    "total_pixels": (69, (10, 1080, 1920), {"total_pixels": 10 * 128 * 28 * 28}, 2),   # 336x588 -> 336x560
    "max_pixels": (70, (4, 480, 640), {"max_pixels": 200 * 28 * 28}, 1),               # 336x448 -> 336x448
    "resized": (71, (2, 720, 1280), {"resized_height": 400, "resized_width": 700}, 2),  # 392x700 -> 392x672
}


def frames(seed: int, shape):
    """uint8 [n, H, W, 3]"""
    return PI.frames(seed, shape)
