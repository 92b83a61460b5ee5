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


def install_qwen_fetch(processor=None, device=None, vision_utils=None):
    """GPU pre-processing for the unmodified Qwen2-VL evaluation drivers (inference_mcq_vqa.py:322-330, INTEGRATION.md
    §7a).  Rebinds process_vision_info on qwen_vl_utils and qwen_vl_utils.vision_process (or on `vision_utils`, a module
    with the same names) so that a video given as a list of frames comes back as the device uint8 [n, h, w, 3] tensor
    of Qwen2VLVideoFetcher.fetch, the bytes of fetch_video's PIL images; images and path videos stay fetch_image's and
    fetch_video's own.  With `processor` (a FlashVStreamQwen2VLProcessor), its image_processor becomes a
    Qwen2VLVideoImageProcessor, so processor(text=..., videos=...) pre-processes those tensors on the GPU while the token
    expansion and visual_position_ids stay the processor's own code.  Install it before the driver imports
    process_vision_info by name (`from qwen_vl_utils import process_vision_info`)."""
    from . import preprocess as P

    patched = []
    mods = [vision_utils] if vision_utils is not None else [importlib.import_module("qwen_vl_utils.vision_process"),
                                                              importlib.import_module("qwen_vl_utils")]
    vp = mods[0]
    extract_vision_info, fetch_image, fetch_video = vp.extract_vision_info, vp.fetch_image, vp.fetch_video
    fetcher = P.Qwen2VLVideoFetcher(P.Qwen2VLFramePreprocessor(device=device))

    def process_vision_info(conversations):
        """qwen_vl_utils.process_vision_info (vision_process.py:243-261), a list-of-frames video fetched on the GPU"""
        image_inputs, video_inputs = [], []
        for info in extract_vision_info(conversations):
            if "image" in info or "image_url" in info:
                image_inputs.append(fetch_image(info))
            elif "video" in info:
                video_inputs.append(fetcher.fetch(info) if isinstance(info["video"], (list, tuple)) else fetch_video(info))
            else:
                raise ValueError("image, image_url or video should in content.")
        return image_inputs or None, video_inputs or None

    for mod in mods:
        mod.process_vision_info = process_vision_info
        patched.append(f"{mod.__name__}.process_vision_info")
    if processor is not None:
        processor.image_processor = P.Qwen2VLVideoImageProcessor(processor.image_processor, device)
        patched.append(f"{type(processor).__name__}.image_processor")
    return patched
