"""Qwen2-VL variant of the Flash Memory on sm_90a: drop-in mirrors of Flash-VStream-Qwen/models/compress_functions.py
(weighted_kmeans_ordered_feature), Flash-VStream-Qwen/models/vstream_qwen2vl_model.py (class FlashMemory, offline) and
Flash-VStream-Qwen/models/vstream_qwen2vl_realtime.py (streaming FlashMemory + the per-clip state update, kept in a
device-resident QwenStreamState), plus the Qwen2-VL PatchMerger the streaming step ends in."""
from .compress_functions import weighted_kmeans_ordered_feature  # noqa: F401
from .patch_merger import PatchMerger  # noqa: F401
from .vstream_qwen2vl_model import (FlashMemory, get_real_grid_thw, get_real_grid_thws,  # noqa: F401
                                    get_spatial_real_grid_thw)
from .stream_state import QwenStreamState  # noqa: F401
from .multistream import QwenStreamPool  # noqa: F401
from . import vstream_qwen2vl_realtime  # noqa: F401
