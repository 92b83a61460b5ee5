"""Seeded uint8 RGB frames and the cases of tests/golden/preprocess.npz (make_golden_preprocess.py)."""
from __future__ import annotations

import numpy as np

OPENAI_CLIP_MEAN = [0.48145466, 0.4578275, 0.40821073]
OPENAI_CLIP_STD = [0.26862954, 0.26130258, 0.27577711]

# name -> (seed, (T, H, W), shortest_edge, crop)
CLIP_CASES = {
    "down": (11, (2, 120, 160), 56, 56),         # 120x160 -> 56x74, crop 56
    "up": (12, (1, 45, 50), 84, 84),             # 45x50 -> 84x93 (upscale), crop 84
    "portrait": (13, (1, 150, 84), 84, 84),      # 150x84 -> 150x84 (both axes unchanged), crop 84 of the height
}
# name -> (seed, (T, H, W), min_pixels, max_pixels, additional_pool_size)
QWEN_CASES = {
    "down": (21, (2, 120, 160), 56 * 56, 56 * 112, 2),        # -> 56x56
    "one_axis": (22, (2, 56, 70), 56 * 56, 28 * 28 * 1280, 1),    # -> 56x56: the height is unchanged
    "one_frame": (23, (1, 56, 60), 56 * 56, 28 * 28 * 1280, 1),   # -> 56x56, one frame in both temporal slots
    "min_pixels": (24, (2, 20, 24), 56 * 84, 28 * 28 * 1280, 1),  # upscale to reach min_pixels: -> 84x84
}


def frames(seed: int, shape) -> np.ndarray:
    T, H, W = shape
    return np.random.default_rng(seed).integers(0, 256, (T, H, W, 3), dtype=np.uint8)
