"""install(): rebind the reference's Python seam to the sm_90a implementations so the reference's own callers
(serve/cli_video_stream.py:192, language_model/vstream_llama.py:71-102, eval loaders) run unmodified on top of
libfvs_b200.so.  The reference has no plugin registry — the seam is attribute lookup (SURVEY.md §8b) — so this is
plain attribute assignment on the already-imported reference modules."""
from __future__ import annotations

import importlib


def install():
    from . import clip_encoder as my_clip
    from . import compress_functions as my_cf
    from . import vstream_arch as my_arch

    ref_cf = importlib.import_module("flash_vstream.model.compress_functions")
    ref_arch = importlib.import_module("flash_vstream.model.vstream_arch")
    ref_clip = importlib.import_module("flash_vstream.model.multimodal_encoder.clip_encoder")
    ref_builder = importlib.import_module("flash_vstream.model.multimodal_encoder.builder")

    patched = []
    for name in ("weighted_kmeans_feature", "attention_feature", "drop_feature", "merge_feature", "kmeans_feature",
                 "k_drop_feature", "k_merge_feature"):
        setattr(ref_cf, name, getattr(my_cf, name))
        setattr(ref_arch, name, getattr(my_cf, name))  # vstream_arch imported the names (vstream_arch.py:31)
        patched.append(f"compress_functions.{name}")
    Ref = ref_arch.VStreamMetaForCausalLM
    Mine = my_arch.VStreamMetaForCausalLM
    for name in ("encode_images", "attention", "compress_spatial_features", "compress_temporal_features",
                 "embed_video_streaming", "consolidate_streaming", "memory_prefix", "cat_proj", "reset_video_stream",
                 "_star_cfg", "_compress_fn", "_order", "_compress_long", "_append_buffer", "_fused_cfg", "_get_bank",
                 "_stream_step_fused", "_publish", "encode_video_memory", "reshape_2x2_image_features"):
        setattr(Ref, name, getattr(Mine, name))
        patched.append(f"VStreamMetaForCausalLM.{name}")
    Ref.fvs_tie_order = Mine.fvs_tie_order
    Ref.fvs_fused_stream, Ref.fvs_chunk_cap = Mine.fvs_fused_stream, Mine.fvs_chunk_cap
    Ref.fvs_bank_device_frames = Mine.fvs_bank_device_frames
    from . import multimodal_projector as my_proj
    ref_proj = importlib.import_module("flash_vstream.model.multimodal_projector.builder")
    ref_proj.build_vision_projector = my_proj.build_vision_projector
    ref_arch.build_vision_projector = my_proj.build_vision_projector   # imported by name at vstream_arch.py:28
    patched.append("multimodal_projector.build_vision_projector")
    ref_clip.CLIPVisionTower = my_clip.CLIPVisionTower
    ref_builder.CLIPVisionTower = my_clip.CLIPVisionTower
    patched.append("multimodal_encoder.CLIPVisionTower")
    return patched


def install_qwen():
    """Same for the Qwen2-VL variant (Flash-VStream-Qwen/models): rebind FlashMemory (offline + streaming) and
    weighted_kmeans_ordered_feature on the already-imported reference modules `models.*` (INTEGRATION.md §5)."""
    from . import qwen as my_qwen
    from .qwen import vstream_qwen2vl_realtime as my_rt

    patched = []
    ref_cf = importlib.import_module("models.compress_functions")
    ref_cf.weighted_kmeans_ordered_feature = my_qwen.weighted_kmeans_ordered_feature
    patched.append("models.compress_functions.weighted_kmeans_ordered_feature")
    for mod, cls in (("models.vstream_qwen2vl_model", my_qwen.FlashMemory), ("models.vstream_qwen2vl_realtime", my_rt.FlashMemory)):
        try:
            ref = importlib.import_module(mod)
        except Exception:  # the realtime module is optional in a given deployment
            continue
        ref.FlashMemory = cls
        ref.weighted_kmeans_ordered_feature = my_qwen.weighted_kmeans_ordered_feature   # imported by name there
        patched.append(mod + ".FlashMemory")
    return patched
