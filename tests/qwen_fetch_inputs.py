"""Seeded frame lists and the cases of tests/golden/qwen_fetch.npz (make_golden_qwen_fetch.py): qwen_vl_utils.fetch_video
on a list of frames, then FlashVStreamQwen2VLImageProcessor on what it returns."""
from __future__ import annotations

from tests import preprocess_inputs as PI

# The image processor of the Qwen2-VL checkpoints the drivers load (preprocessor_config.json): min / max pixels.
PROC_MIN_PIXELS, PROC_MAX_PIXELS = 56 * 56, 28 * 28 * 16384
REPRODUCE_MIN_PIXELS = 32 * 28 * 28          # inference_mcq_vqa.py:298, the drivers' --reproduce setting

# name -> (seed, (frames in the list, H, W), fetch_video keys besides 'video', additional_pool_size); the comments give
# fetch_image's resize (stage 1), then the processor's (stage 2).  The sizes are small and most lists hold one frame
# (padded to two) so that the golden stays small.
CASES = {
    "down_down": (31, (1, 150, 375), {"min_pixels": 56 * 56, "max_pixels": 60 * 150}, 2),   # 150x375 -> 56x140 -> 56x112
    "up_up": (32, (1, 20, 25), {"min_pixels": 56 * 84}, 2),                      # 20x25 -> 84x84 -> 112x112
    "noop": (33, (1, 56, 112), {"min_pixels": 56 * 56}, 2),                      # 56x112 unchanged in both stages
    "noop_then_resize": (34, (1, 56, 140), {"min_pixels": 56 * 56}, 2),          # 56x140 unchanged -> 56x112
    "odd": (35, (3, 30, 30), {"min_pixels": 56 * 56}, 1),                        # 3 frames, padded to 4; 30x30 -> 56x56
    "max_frames": (36, (12, 30, 40), {"max_frames": 3, "min_pixels": 56 * 56}, 1),   # 2 of 12 frames picked
    "reproduce": (37, (1, 36, 64), {"min_pixels": REPRODUCE_MIN_PIXELS}, 2),    # the drivers' --reproduce setting
    "total_pixels": (38, (4, 60, 90), {"total_pixels": 2 * 56 * 84, "min_pixels": 56 * 56}, 2),   # -> 56x84 -> 56x112
    "max_pixels": (39, (1, 150, 200), {"max_pixels": 56 * 84, "min_pixels": 56 * 56}, 2),
    "resized": (40, (1, 64, 80), {"resized_height": 50, "resized_width": 60}, 2),  # fetch_image's defaults apply
    "pool1": (41, (2, 70, 45), {"min_pixels": 56 * 56}, 1),
}
# past fetch_image's MAX_RATIO (200): fetch_video raises ValueError
RATIO_CASE = (42, (2, 10, 2010), {"min_pixels": 4 * 28 * 28}, 2)


def frames(seed: int, shape):
    """uint8 [n, H, W, 3]"""
    return PI.frames(seed, shape)
