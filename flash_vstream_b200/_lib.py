"""ctypes binding of libfvs_b200.so (the C ABI declared in include/fvs_b200.h).

There is deliberately NO fallback: if the library is missing or a call fails, an exception is raised.
"""
from __future__ import annotations

import ctypes as C
from pathlib import Path

from . import _build

F16, BF16, F32 = 0, 1, 2
EPI_BIAS, EPI_BIAS_QUICKGELU, EPI_BIAS_RESIDUAL, EPI_ROWTABLE, EPI_BIAS_RESIDUAL_F32, EPI_BIAS_GELU = 0, 1, 2, 3, 4, 5

FVS_OK, FVS_EINVAL, FVS_ECUDA, FVS_ENOTIMPL = 0, -1, -2, -3


class FvsError(RuntimeError):
    pass


class VitLayerWeights(C.Structure):
    _fields_ = [(n, C.c_void_p) for n in (
        "ln1_w", "ln1_b", "qkv_w", "qkv_b", "o_w", "o_b", "ln2_w", "ln2_b", "fc1_w", "fc1_b", "fc2_w", "fc2_b")]


class VitConfig(C.Structure):
    _fields_ = [("image_size", C.c_int), ("patch_size", C.c_int), ("hidden", C.c_int), ("heads", C.c_int),
                ("mlp", C.c_int), ("layers_run", C.c_int), ("ln_eps", C.c_float), ("dtype", C.c_int), ("keep_cls", C.c_int)]


class VitWeights(C.Structure):
    _fields_ = [("patch_w", C.c_void_p), ("class_emb", C.c_void_p), ("pos_emb", C.c_void_p),
                ("pre_ln_w", C.c_void_p), ("pre_ln_b", C.c_void_p), ("layers_h", C.POINTER(VitLayerWeights))]


class QwenVitConfig(C.Structure):
    _fields_ = [("embed_dim", C.c_int), ("heads", C.c_int), ("mlp_dim", C.c_int), ("depth", C.c_int),
                ("patch_dim", C.c_int), ("ln_eps", C.c_float), ("dtype", C.c_int)]


class StarConfig(C.Structure):   # fvs_star_config
    _fields_ = [(n, C.c_int) for n in ("D", "grid", "cur_size", "long_size", "long_len", "tur_len", "cur_len", "key_len",
                                       "ntm_dim")] + [("ratio", C.c_float)]


class NtmWeights(C.Structure):   # fvs_ntm_weights
    _fields_ = [(n, C.c_void_p) for n in ("q_w", "q_b", "k_w", "k_b")]


class Bank(C.Structure):         # fvs_bank
    _fields_ = [("prefix", C.c_void_p), ("long_work", C.c_void_p), ("tur_work", C.c_void_p), ("frames", C.c_void_p),
                ("header", C.c_void_p), ("frames_cap", C.c_int64), ("chunk_cap", C.c_int32), ("n_long", C.c_int32),
                ("n_tur", C.c_int32), ("n_cur", C.c_int32), ("n_frames", C.c_int64), ("step", C.c_uint64),
                ("frames_window", C.c_int64)]


class StreamJob(C.Structure):    # fvs_stream_job
    _fields_ = [("bank", C.POINTER(Bank)), ("ntm", C.POINTER(NtmWeights)), ("frames", C.c_int), ("init_idx", C.c_void_p),
                ("refill_idx", C.c_void_p), ("workspace", C.c_void_p), ("workspace_bytes", C.c_size_t)]


class ResampleAxis(C.Structure):  # fvs_resample_axis
    _fields_ = [(n, C.c_int) for n in ("in_size", "out_size", "first", "count", "taps", "span_first", "span_count")] + \
               [("bounds", C.c_void_p), ("coeffs", C.c_void_p)]


class PreprocessJob(C.Structure):  # fvs_preprocess_job
    _fields_ = [("frames", C.c_void_p)] + [(n, C.c_int) for n in ("T", "H", "W", "C")] + \
               [("x", ResampleAxis), ("y", ResampleAxis), ("x2", ResampleAxis), ("y2", ResampleAxis)]


class QwenMemJob(C.Structure):  # fvs_qwen_mem_job
    _fields_ = [("X", C.c_void_p)] + [(n, C.c_int) for n in ("T", "K", "PD", "x_dtype")] + \
               [(n, C.c_void_p) for n in ("w", "init_idx", "refill_idx")] + [("max_iter", C.c_int), ("tol", C.c_float)] + \
               [(n, C.c_void_p) for n in ("uniq_idx", "n_unique", "uniq_workspace")] + [("uniq_workspace_bytes", C.c_size_t)] + \
               [(n, C.c_void_p) for n in ("C", "wsum", "labels", "info", "km_workspace")] + \
               [("km_workspace_bytes", C.c_size_t)] + \
               [(n, C.c_void_p) for n in ("order_in", "sorted_idx", "ts", "w_sorted", "flags", "out")] + [("out_dtype", C.c_int)]


class QwenRetrieveJob(C.Structure):  # fvs_qwen_retrieve_job
    _fields_ = [(n, C.c_void_p) for n in ("tem_x", "klarge_idx", "bank")] + \
               [(n, C.c_int) for n in ("k", "t_total", "n_dev", "PD")] + \
               [(n, C.c_void_p) for n in ("idx_out", "dist_out", "workspace")] + [("workspace_bytes", C.c_size_t)]


class QwenGatherJob(C.Structure):  # fvs_qwen_gather_job
    _fields_ = [("picks", C.c_void_p), ("n", C.c_int), ("n_frames", C.c_int64), ("dev_x", C.c_void_p),
                ("dev_merged", C.c_void_p), ("n_dev", C.c_int64), ("host_chunks", C.c_void_p), ("chunk_frames", C.c_int),
                ("prev_picks", C.c_void_p), ("m", C.c_int), ("prev_x", C.c_void_p), ("prev_merged", C.c_void_p),
                ("x_frame_elems", C.c_int64), ("merged_frame_elems", C.c_int64), ("spa_x_out", C.c_void_p),
                ("merged_out", C.c_void_p), ("host_fetches", C.c_void_p), ("fresh_frames", C.c_void_p),
                ("n_fresh", C.c_int), ("fresh_x", C.c_void_p), ("fresh_merged", C.c_void_p), ("n_base", C.c_int64)]


class QwenPickPlanJob(C.Structure):  # fvs_qwen_pick_plan_job
    _fields_ = [("picks", C.c_void_p), ("n", C.c_int), ("n_frames", C.c_int64), ("frames", C.c_void_p),
                ("plan", C.c_void_p), ("count", C.c_void_p), ("prev_picks", C.c_void_p), ("m", C.c_int),
                ("re_encodes", C.c_void_p), ("stored", C.c_uint8)]


class QwenPixelJob(C.Structure):  # fvs_qwen_pixel_job
    _fields_ = [("plan", C.c_void_p), ("n", C.c_int), ("n_frames", C.c_int64), ("base", C.c_int64),
                ("host_chunks", C.c_void_p), ("chunk_frames", C.c_int), ("frame_elems", C.c_int64), ("out", C.c_void_p),
                ("table", C.c_void_p)]


class QwenScatterJob(C.Structure):  # fvs_qwen_scatter_job
    _fields_ = [("plan", C.c_void_p), ("n", C.c_int), ("n_frames", C.c_int64), ("x_rows", C.c_void_p),
                ("merged_rows", C.c_void_p), ("dev_x", C.c_void_p), ("dev_merged", C.c_void_p), ("n_dev", C.c_int64),
                ("host_chunks", C.c_void_p), ("chunk_frames", C.c_int), ("x_frame_elems", C.c_int64),
                ("merged_frame_elems", C.c_int64)]


QWEN_MEM_JOBS_PER_LAUNCH = 16
PRE_CLIP, PRE_QWEN, PRE_QWEN_CODES, PRE_RGB8 = 0, 1, 2, 3
KLARGE_EUCLIDEAN, KLARGE_COSINE = 0, 1
INPUT_PIXELS, INPUT_FEATURES = 0, 1

_vp, _i, _f, _sz = C.c_void_p, C.c_int, C.c_float, C.c_size_t
_i64p = C.POINTER(C.c_int64)

# name -> (restype, argtypes); must list every symbol include/fvs_b200.h declares (tests check this)
SIGNATURES = {
    "fvs_version": (_i, []),
    "fvs_last_error": (C.c_char_p, []),
    "fvs_launch_count": (C.c_uint64, []),
    "fvs_prof_enable": (_i, [_i]),
    "fvs_prof_collect": (_i, [_vp, _vp, _vp, _i]),
    "fvs_prof_pause": (_i, [_i]),
    "fvs_linear": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _i, _i, _vp]),
    "fvs_attention": (_i, [_vp, _vp, _i, _i, _i, _f, _i, _vp]),
    "fvs_attention80": (_i, [_vp, _vp, _i, _i, _i, _f, _i, _vp]),
    "fvs_layernorm": (_i, [_vp, _vp, _vp, _vp, _i, _i, _f, _i, _i, _i, _vp]),
    "fvs_add_layernorm": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _f, _i, _vp]),
    "fvs_vit_create": (_i, [C.POINTER(_vp), C.POINTER(VitConfig), C.POINTER(VitWeights), _vp]),
    "fvs_vit_destroy": (_i, [_vp]),
    "fvs_vit_workspace_bytes": (_sz, [_vp, _i]),
    "fvs_vit_encode": (_i, [_vp, _vp, _vp, _i, _vp, _sz, _vp]),
    "fvs_vit_encode_pool3": (_i, [_vp, _vp, _vp, _vp, _vp, _i, _i, _i, _vp, _sz, _vp]),
    # streaming step on a persistent bank
    "fvs_stream_workspace_bytes": (_sz, [C.POINTER(StarConfig), _i]),
    "fvs_bank_rows": (_i, [C.POINTER(StarConfig), _i, _i64p, _i64p, _i64p]),
    "fvs_bank_reset": (_i, [C.POINTER(Bank), _vp]),
    "fvs_bank_restore": (_i, [C.POINTER(StarConfig), C.POINTER(Bank), C.c_int32, C.c_int32, C.c_int32, C.c_int64, C.c_uint64,
                              _vp, _vp, _vp, _vp, _vp]),
    "fvs_bank_prefix": (_i,[C.POINTER(StarConfig), C.POINTER(Bank), C.POINTER(_vp), _i64p]),
    "fvs_stream_step": (_i, [C.POINTER(StarConfig), C.POINTER(Bank), C.POINTER(NtmWeights), _vp, _vp, _i, _i, _vp, _vp,
                             _vp, _sz, _vp, _sz, _vp]),
    "fvs_stream_step_multi": (_i, [C.POINTER(StarConfig), C.POINTER(StreamJob), _i, _vp, _vp, _i, _vp, _sz, _i, _vp]),
    "fvs_stream_plan": (_i, [C.POINTER(StarConfig), C.POINTER(StreamJob), _i, _i, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "fvs_stream_step_info": (_i, [C.POINTER(StarConfig), C.POINTER(Bank), _vp, C.POINTER(_vp), C.POINTER(_vp), C.POINTER(_vp),
                                  C.POINTER(_vp)]),
    "fvs_bank_snapshot": (_i, [_vp, _vp, _vp, C.c_int64, _i, _i, _i, _vp, _vp]),
    "fvs_spatial_pool": (_i, [_vp, _vp, _i, _i, _i, _i, _i, _vp]),
    "fvs_spatial_pool3": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _i, _i, _vp]),
    "fvs_kmeans_workspace_bytes": (_sz, [_i, _i, _i]),
    "fvs_weighted_kmeans": (_i, [_vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _vp, _vp, _vp, _vp, _vp, _sz, _i, _vp]),
    "fvs_abstract_update": (_i, [_vp, _vp, _vp, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _i, _vp]),
    "fvs_argsort_desc": (_i, [_vp, _i, _vp, _i, _vp]),
    "fvs_key_retrieve": (_i, [_vp, _vp, _i, _i, _i, _i, _vp, _i, _vp]),
    "fvs_gather_rows": (_i, [_vp, _vp, _vp, _i, C.c_int64, _i, _vp]),
    "fvs_qwen_vit_create": (_i, [C.POINTER(_vp), C.POINTER(QwenVitConfig), _vp, C.POINTER(VitLayerWeights), C.POINTER(C.c_float), _vp]),
    "fvs_qwen_vit_destroy": (_i, [_vp]),
    "fvs_qwen_vit_workspace_bytes": (_sz, [_vp, C.c_int64]),
    "fvs_qwen_vit_encode": (_i, [_vp, _vp, _vp, C.POINTER(C.c_int32), _i, _vp, _sz, _vp]),
    # alternate temporal compressors
    "fvs_alt_workspace_bytes": (_sz, [_i, _i, _i, _i]),
    "fvs_alt_sequential": (_i, [_i, _vp, _i, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp, _vp, _sz, _i, _vp]),
    "fvs_alt_kmeans": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _f, _vp, _vp, _vp, _vp, _sz, _i, _vp]),
    # Qwen2-VL Flash Memory
    "fvs_qwen_temporal_pool": (_i, [_vp, _vp, _i, _i, _i, _i, _vp]),
    "fvs_qwen_unique_workspace_bytes": (_sz, [_i]),
    "fvs_qwen_unique_rows": (_i, [_vp, _i, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "fvs_qwen_kmeans_workspace_bytes": (_sz, [_i, _i, _i]),
    "fvs_qwen_kmeans": (_i, [_vp, _i, _vp, _vp, _vp, _vp, _i, _i, _i, _i, _f, _vp, _vp, _vp, _vp, _vp, _sz, _vp]),
    "fvs_qwen_kmeans_finalize": (_i, [_vp, _vp, _i, _i, _vp, _vp, _vp, _vp, _vp, _vp]),
    "fvs_gather_rows_cast": (_i, [_vp, _vp, _vp, _i, C.c_int64, _i, _vp]),
    "fvs_qwen_mem_plan": (_i, [C.POINTER(QwenMemJob), _i, _i, C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "fvs_qwen_unique_rows_multi": (_i, [C.POINTER(QwenMemJob), _i, _i, _vp]),
    "fvs_qwen_kmeans_multi": (_i, [C.POINTER(QwenMemJob), _i, _i, _vp]),
    "fvs_qwen_kmeans_finalize_multi": (_i, [C.POINTER(QwenMemJob), _i, _i, _vp]),
    "fvs_gather_rows_cast_multi": (_i, [C.POINTER(QwenMemJob), _i, _i, _vp]),
    "fvs_qwen_klarge_retrieve_multi": (_i, [C.POINTER(QwenRetrieveJob), _i, _i, _i, _vp]),
    "fvs_qwen_dam_gather_multi": (_i, [C.POINTER(QwenGatherJob), _i, _i, _vp]),
    "fvs_qwen_klarge_workspace_bytes": (_sz, [_i, _i, _i]),
    "fvs_qwen_klarge_retrieve": (_i, [_vp, _vp, _vp, _i, _i, _i, _i, _i, _vp, _vp, _vp, _sz, _vp]),
    "fvs_qwen_klarge_retrieve_tiered": (_i, [_vp, _vp, _vp, _i, C.POINTER(_vp), _i, _i, _i, _i, _i, _i, _vp, _vp, _vp, _sz,
                                             _vp]),
    "fvs_qwen_am_rope": (_i, [_vp, _i, _i, _i, _vp, _i, _i, _i, C.c_int64, _vp, _vp]),
    # feature bank of the Qwen2-VL streaming state
    "fvs_host_device_ptr": (_i, [_vp, C.POINTER(_vp)]),
    "fvs_qwen_pick_plan_multi": (_i, [C.POINTER(QwenPickPlanJob), _i, _vp]),
    "fvs_qwen_pixel_gather_multi": (_i, [C.POINTER(QwenPixelJob), _i, _i, _vp]),
    "fvs_qwen_bank_scatter_multi": (_i, [C.POINTER(QwenScatterJob), _i, _i, _vp]),
    # 8-bit pixel codes
    "fvs_qwen_pixel_decode": (_i, [_vp, C.c_int64, _vp, _i, _vp, _vp]),
    # publication of the Qwen2-VL streaming memory (seqlock)
    "fvs_qwen_pub_layout": (_i, [_i, _i, _i, _i, _i, _i, _i, _i64p]),
    "fvs_qwen_publish": (_i, [_vp, _sz, _i, _i, C.c_int64, _i, _vp, C.c_int64, _vp, _i, _vp, _i, _i, _i, _i, _i, C.c_uint64,
                              C.c_uint64, C.c_int64, _vp]),
    "fvs_qwen_snapshot": (_i, [_vp, _sz, _i, _i, C.c_int64, _i, _vp, C.c_int64, _vp, C.c_int64, _vp, C.c_int64, _vp, _vp]),
    # frame pre-processing (uint8 RGB frames -> tower pixels)
    "fvs_resample_plan": (_i, [_i, _i, _i, _i, C.POINTER(ResampleAxis), C.POINTER(C.c_int32), C.POINTER(C.c_int32)]),
    "fvs_preprocess_workspace_bytes": (_sz, [C.POINTER(ResampleAxis), C.POINTER(ResampleAxis), _i]),
    "fvs_preprocess": (_i, [_vp, _i, _i, _i, _i, C.POINTER(ResampleAxis), C.POINTER(ResampleAxis), _vp, _i, _i, _vp, _vp, _sz,
                            _vp]),
    "fvs_preprocess_plan": (_i, [C.POINTER(PreprocessJob), _i, _i, _i, _i64p, _i64p]),
    "fvs_preprocess_multi": (_i, [C.POINTER(PreprocessJob), _i, _vp, _i, _i, _vp, _vp, _sz, _vp]),
}

_lib = None


def lib_path() -> Path:
    import os
    override = os.environ.get("FVS_LIB_PATH")      # A/B benchmarking of two builds; never a fallback
    return Path(override) if override else _build.LIB_PATH


def load(build_if_missing: bool = True) -> C.CDLL:
    """Load (building first if needed and possible) the native library; raises if unavailable."""
    global _lib
    if _lib is not None:
        return _lib
    path = lib_path()
    if not path.exists():
        if not build_if_missing:
            raise FvsError(f"{path} is missing: run `python -c 'import __graft_entry__ as g; g.build()'`")
        _build.build()
    elif path == _build.LIB_PATH and not _build.is_fresh():
        # a library built from other sources than the ones next to it (older ABI): never load it silently
        if build_if_missing and _build.can_build():
            _build.build()
        else:
            raise FvsError(f"{path} is stale (csrc/ or include/fvs_b200.h changed since it was built): run "
                           f"`python -c 'import __graft_entry__ as g; g.build()'`")
    lib = C.CDLL(str(path))
    for name, (res, args) in SIGNATURES.items():
        fn = getattr(lib, name)  # AttributeError if the symbol is not exported
        fn.restype = res
        fn.argtypes = args
    _lib = lib
    return lib


def check(code: int, what: str = "") -> None:
    if code == FVS_OK:
        return
    msg = load().fvs_last_error().decode(errors="replace")
    text = f"{what}: {msg}" if what else msg
    if code == FVS_ENOTIMPL:
        raise NotImplementedError(text)
    if code == FVS_EINVAL:
        raise ValueError(text)
    raise FvsError(text)


def dtype_code(t) -> int:
    import torch
    if t == torch.float16:
        return F16
    if t == torch.bfloat16:
        return BF16
    if t == torch.float32:
        return F32
    raise ValueError(f"unsupported dtype {t}")


def ptr(t) -> int | None:
    """Device pointer of a CUDA tensor (None -> NULL). Refuses CPU tensors: there is no CPU path."""
    if t is None:
        return None
    if not t.is_cuda:
        raise FvsError("flash_vstream_b200 kernels need CUDA tensors (no CPU fallback exists)")
    return t.data_ptr()


def cur_stream() -> int:
    import torch
    return torch.cuda.current_stream().cuda_stream
