"""Frame pre-processing on the GPU: decoded uint8 RGB frames -> the pixels the vision towers take, bit-identical to the
reference's CPU image processors (fvs_preprocess, csrc/preprocess_kernels.cu).

    CLIPFramePreprocessor(image_processor)(frames)   == image_processor.preprocess(clip)['pixel_values'].half()
                                                        (Flash-VStream-LLaVA/flash_vstream/serve/cli_video_stream.py:186)
    Qwen2VLFramePreprocessor(...)(frames)            == the {'pixel_values_videos', 'video_grid_thw'} of
                                                        FlashVStreamQwen2VLImageProcessor (cli_server_2gpu.py:214-219)
    Qwen2VLVideoFetcher(...).fetch(ele)              == np.stack(qwen_vl_utils.fetch_video(ele)), a list of frames
    Qwen2VLVideoFetcher(...)(ele)                    == FlashVStreamQwen2VLImageProcessor(videos=[fetch_video(ele)])
                                                        (inference_mcq_vqa.py:290-334)

Frames are [T, H, W, 3] uint8 (what decord and np.asarray(PIL image) give): a CUDA tensor, or a host tensor / array
that is copied to the device (non_blocking, so a pinned one does not block the host).  The resize is Pillow's BICUBIC
resample, which is integer arithmetic; rescale + normalize are a function of one byte per channel, so they are a
float32 [3, 256] table built here with transformers' numpy operations.  Inference only, like the rest of the package.
"""
from __future__ import annotations

import ctypes as C
import math
import os
from concurrent.futures import ThreadPoolExecutor

import numpy as np

from . import _lib

BICUBIC = 3                                        # PILImageResampling.BICUBIC
OPENAI_CLIP_MEAN = (0.48145466, 0.4578275, 0.40821073)
OPENAI_CLIP_STD = (0.26862954, 0.26130258, 0.27577711)
QWEN_PATCH, QWEN_MERGE, QWEN_TEMPORAL = 14, 2, 2


# ---- host restatements of the reference's size arithmetic ---------------------------------------------------------
def clip_resize_size(height: int, width: int, shortest_edge: int) -> tuple[int, int]:
    """transformers.image_transforms.get_resize_output_image_size(image, shortest_edge, default_to_square=False)"""
    short, long = (width, height) if width <= height else (height, width)
    new_long = int(shortest_edge * long / short)
    return (new_long, shortest_edge) if width <= height else (shortest_edge, new_long)


def center_crop_offsets(height: int, width: int, crop_height: int, crop_width: int) -> tuple[int, int]:
    """top, left of transformers.image_transforms.center_crop"""
    return (height - crop_height) // 2, (width - crop_width) // 2


def smart_resize(height: int, width: int, factor: int = 28, min_pixels: int = 56 * 56,
                 max_pixels: int = 14 * 14 * 4 * 1280) -> tuple[int, int]:
    """transformers.models.qwen2_vl.image_processing_qwen2_vl.smart_resize (what the Qwen2-VL reference imports)"""
    if max(height, width) / min(height, width) > 200:
        raise ValueError(f"absolute aspect ratio must be smaller than 200, got {max(height, width) / min(height, width)}")
    h_bar = round(height / factor) * factor
    w_bar = round(width / factor) * factor
    if h_bar * w_bar > max_pixels:
        beta = math.sqrt((height * width) / max_pixels)
        h_bar = max(factor, math.floor(height / beta / factor) * factor)
        w_bar = max(factor, math.floor(width / beta / factor) * factor)
    elif h_bar * w_bar < min_pixels:
        beta = math.sqrt(min_pixels / (height * width))
        h_bar = math.ceil(height * beta / factor) * factor
        w_bar = math.ceil(width * beta / factor) * factor
    return h_bar, w_bar


def value_table(rescale_factor=None, mean=None, std=None) -> np.ndarray:
    """float32 [3, 256]: what transformers' numpy rescale (float32(float64(u8) * factor)) and normalize ((v - mean) / std
    in float32) make of each byte of each channel; None skips a step."""
    x = np.tile(np.arange(256, dtype=np.uint8), (3, 1))
    if rescale_factor is not None:
        x = (x.astype(np.float64) * rescale_factor).astype(np.float32)
    if mean is not None:
        x = x.astype(np.float32)
        m = np.broadcast_to(np.asarray(mean, dtype=np.float32), (3,))[:, None]
        s = np.broadcast_to(np.asarray(std, dtype=np.float32), (3,))[:, None]
        x = (x - m) / s
    return np.ascontiguousarray(x, dtype=np.float32)


def resample_plan(in_size: int, out_size: int, first: int = 0, count: int | None = None):
    """The library's host plan of one axis: (fvs_resample_axis, bounds int32 [count, 2], coeffs int32 [count, taps])."""
    count = out_size - first if count is None else count
    lib = _lib.load()
    ax = _lib.ResampleAxis()
    _lib.check(lib.fvs_resample_plan(in_size, out_size, first, count, C.byref(ax), None, None), "fvs_resample_plan")
    bounds = np.empty((count, 2), np.int32)
    coeffs = np.empty((count, ax.taps), np.int32)
    i32 = C.POINTER(C.c_int32)
    _lib.check(lib.fvs_resample_plan(in_size, out_size, first, count, C.byref(ax), bounds.ctypes.data_as(i32),
                                     coeffs.ctypes.data_as(i32)), "fvs_resample_plan")
    return ax, bounds, coeffs


def _field(d, key):
    """a size dict of transformers 4.x (dict) or 5.x (SizeDict)"""
    if d is None:
        return None
    return d.get(key) if isinstance(d, dict) else getattr(d, key, None)


class _FramePreprocessor:
    """Device tables (the [3, 256] table once per device, the two axis plans once per device and input size) and the
    one library call."""
    _layout = None

    def __init__(self, table: np.ndarray, device=None):
        self.table = table
        self.device = device
        self._tables = {}
        self._plans = {}

    def _windows(self, height: int, width: int):
        """((out_h, first_y, count_y), (out_w, first_x, count_x), pool) for a height x width input"""
        raise NotImplementedError

    def _device(self, frames=None):
        import torch
        if frames is not None and frames.is_cuda:
            return frames.device
        device = torch.device(self.device if self.device is not None else "cuda")
        return device if device.index is not None else torch.device(device.type, torch.cuda.current_device())

    def _axes(self, device, height, width, rows, cols):
        """(x, y, device tables) of height x width -> rows = (out_h, first_y, count_y), cols = (out_w, first_x,
        count_x) on `device`, planned once"""
        import torch
        key = (device, height, width, rows, cols)
        plan = self._plans.get(key)
        if plan is None:
            keep, axes = [], []
            for size_in, (size_out, first, count) in ((width, cols), (height, rows)):
                ax, bounds, coeffs = resample_plan(size_in, size_out, first, count)
                b, k = torch.from_numpy(bounds).to(device), torch.from_numpy(coeffs).to(device)
                ax.bounds, ax.coeffs = b.data_ptr(), k.data_ptr()
                keep += [b, k]
                axes.append(ax)
            plan = self._plans[key] = (axes[0], axes[1], keep)
        return plan

    def _plan(self, device, height, width):
        rows, cols, pool = self._windows(height, width)
        x, y, keep = self._axes(device, height, width, rows, cols)
        return x, y, pool, keep

    def _table(self, device):
        import torch
        device = torch.device(device)
        if device.type == "cuda" and device.index is None:
            device = torch.device("cuda", torch.cuda.current_device())
        t = self._tables.get(device)
        if t is None:
            t = self._tables[device] = torch.from_numpy(self.table).to(device)
        return t

    @staticmethod
    def _tensor(frames, what="frames"):
        import torch
        if isinstance(frames, np.ndarray):
            frames = torch.from_numpy(frames)
        if not isinstance(frames, torch.Tensor):
            raise TypeError(f"{what} must be a uint8 tensor or array [T, H, W, 3], got {type(frames).__name__}")
        if frames.dtype != torch.uint8 or frames.dim() != 4:
            raise ValueError(f"{what} must be uint8 [T, H, W, 3], got {frames.dtype} {tuple(frames.shape)}")
        return frames

    def _frames(self, frames):
        frames = self._tensor(frames)
        device = self._device(frames)
        if not frames.is_cuda:
            frames = frames.to(device, non_blocking=True)
        return frames.contiguous(), device

    def output_shape(self, frames: int, height: int, width: int) -> tuple:
        raise NotImplementedError

    def workspace_bytes(self, frames: int, height: int, width: int, device=None) -> int:
        """bytes of the uint8 workspace a call on `frames` height x width frames needs (pass it as workspace=)"""
        import torch
        x, y, _, _ = self._plan(torch.device(device) if device is not None else self._device(), height, width)
        return int(_lib.load().fvs_preprocess_workspace_bytes(C.byref(x), C.byref(y), frames))

    @staticmethod
    def _out_dtype(layout):
        import torch
        return {_lib.PRE_CLIP: torch.float16, _lib.PRE_QWEN: torch.float32, _lib.PRE_QWEN_CODES: torch.uint8,
                _lib.PRE_RGB8: torch.uint8}[layout]

    def _run(self, frames, out=None, workspace=None, layout=None):
        import torch
        frames, device = self._frames(frames)
        layout = self._layout if layout is None else layout
        T, H, W, ch = frames.shape
        x, y, pool, _ = self._plan(device, H, W)
        shape, dtype = self.output_shape(T, H, W), self._out_dtype(layout)
        if out is None:
            out = torch.empty(shape, dtype=dtype, device=device)
        elif tuple(out.shape) != shape or out.dtype != dtype or out.device != device or not out.is_contiguous():
            raise ValueError(f"out must be a contiguous {dtype} {shape} tensor on {device}")
        need = int(_lib.load().fvs_preprocess_workspace_bytes(C.byref(x), C.byref(y), T))
        if workspace is None:
            workspace = torch.empty(need, dtype=torch.uint8, device=device)
        elif workspace.device != device:
            raise ValueError(f"workspace must be on {device}")
        with torch.cuda.device(device):
            _lib.check(_lib.load().fvs_preprocess(frames.data_ptr(), T, H, W, ch, C.byref(x), C.byref(y),
                                                  self._table(device).data_ptr(), layout, pool, out.data_ptr(),
                                                  workspace.data_ptr(), workspace.numel() * workspace.element_size(),
                                                  _lib.cur_stream()), "fvs_preprocess")
        return out

    def _many(self, clips, out=None, workspace=None, layout=None):
        """-> (out, one view of `out` per clip): every clip through one fvs_preprocess_multi call"""
        import torch
        layout = self._layout if layout is None else layout
        if not isinstance(clips, (list, tuple)):
            raise TypeError(f"clips must be a list of uint8 [T, H, W, 3] clips, got {type(clips).__name__}")
        if not clips:
            raise ValueError("clips is empty")
        clips = [self._tensor(f, f"clip {i}") for i, f in enumerate(clips)]
        devices = {f.device for f in clips if f.is_cuda}
        if len(devices) > 1:
            raise ValueError(f"the clips are on more than one device: {sorted(map(str, devices))}")
        device = devices.pop() if devices else self._device()
        n = len(clips)
        jobs = (_lib.PreprocessJob * n)()
        for i, f in enumerate(clips):           # planned from the shapes: a refused call copies nothing to the device
            T, H, W, ch = f.shape
            x, y, pool, _ = self._plan(device, H, W)
            jobs[i] = _lib.PreprocessJob(f.data_ptr(), T, H, W, ch, x, y)
        lib = _lib.load()
        plan, totals = (C.c_int64 * (4 * n))(), (C.c_int64 * 2)()
        launches = lib.fvs_preprocess_plan(jobs, n, layout, pool, plan, totals)
        if launches < 0:
            _lib.check(launches, "fvs_preprocess_plan")
        frames = [(f if f.is_cuda else f.to(device, non_blocking=True)).contiguous() for f in clips]
        for i, f in enumerate(frames):
            jobs[i].frames = f.data_ptr()
        shapes = [self.output_shape(*(int(v) for v in f.shape[:3])) for f in frames]
        if len({s[1:] for s in shapes}) == 1:       # CLIP with one crop, and every Qwen2-VL call: one stacked tensor
            shape = (sum(s[0] for s in shapes),) + shapes[0][1:]
        else:
            shape = (int(totals[0]),)
        dtype = self._out_dtype(layout)
        if out is None:
            out = torch.empty(shape, dtype=dtype, device=device)
        elif tuple(out.shape) != shape or out.dtype != dtype or out.device != device or not out.is_contiguous():
            raise ValueError(f"out must be a contiguous {dtype} {shape} tensor on {device}")
        if workspace is None:
            workspace = torch.empty(int(totals[1]), dtype=torch.uint8, device=device)
        elif workspace.device != device:
            raise ValueError(f"workspace must be on {device}")
        with torch.cuda.device(device):
            _lib.check(lib.fvs_preprocess_multi(jobs, n, self._table(device).data_ptr(), layout, pool, out.data_ptr(),
                                                workspace.data_ptr(), workspace.numel() * workspace.element_size(),
                                                _lib.cur_stream()), "fvs_preprocess_multi")
        flat = out.view(-1)
        views = [flat[plan[4 * i + 2]: plan[4 * i + 2] + math.prod(s)].view(s) for i, s in enumerate(shapes)]
        return out, views


class CLIPFramePreprocessor(_FramePreprocessor):
    """LLaVA side: frames -> f16 [T, 3, crop, crop] on the device, equal to image_processor.preprocess(clip)
    ['pixel_values'].half() of a PIL-backed CLIPImageProcessor (bicubic shortest-edge resize, center crop, rescale,
    normalize), configured from that processor (the tower's `image_processor`, clip_encoder.py:54)."""
    _layout = _lib.PRE_CLIP

    def __init__(self, image_processor, device=None):
        p = image_processor
        resample = getattr(p, "resample", None)
        if resample is None or int(resample) != BICUBIC:
            raise NotImplementedError(f"resample={resample!r}: only bicubic ({BICUBIC}) is implemented")
        if getattr(p, "do_pad", None):
            raise NotImplementedError("do_pad=True: padding is not implemented")
        self.do_resize = bool(getattr(p, "do_resize", True))
        size = getattr(p, "size", None)
        self.shortest_edge = _field(size, "shortest_edge")
        if self.do_resize and (self.shortest_edge is None or any(_field(size, k) for k in (
                "longest_edge", "height", "width", "max_height", "max_width"))):
            raise NotImplementedError(f"size={size!r}: only a shortest-edge resize ({{'shortest_edge': N}}) is implemented")
        self.do_center_crop = bool(getattr(p, "do_center_crop", True))
        crop = getattr(p, "crop_size", None)
        self.crop = (_field(crop, "height"), _field(crop, "width")) if self.do_center_crop else None
        if self.do_center_crop and None in self.crop:
            raise NotImplementedError(f"crop_size={crop!r}: only {{'height': h, 'width': w}} is implemented")
        rescale = p.rescale_factor if getattr(p, "do_rescale", True) else None
        norm = getattr(p, "do_normalize", True)
        super().__init__(value_table(rescale, p.image_mean if norm else None, p.image_std if norm else None), device)

    def sizes(self, height: int, width: int):
        """(resized (h, w), crop window (top, left, h, w)) for a height x width frame"""
        rh, rw = clip_resize_size(height, width, self.shortest_edge) if self.do_resize else (height, width)
        ch, cw = self.crop if self.crop is not None else (rh, rw)
        top, left = center_crop_offsets(rh, rw, ch, cw)
        return (rh, rw), (top, left, ch, cw)

    def _windows(self, height, width):
        (rh, rw), (top, left, ch, cw) = self.sizes(height, width)
        return (rh, top, ch), (rw, left, cw), 1

    def output_shape(self, frames, height, width):
        _, (_, _, ch, cw) = self.sizes(height, width)
        return (frames, 3, ch, cw)

    def __call__(self, frames, out=None, workspace=None):
        return self._run(frames, out, workspace)

    def many(self, clips, out=None, workspace=None):
        """Many clips (a list of uint8 [T, H, W, 3], host or device, any mix of sizes) in one launch pair per 32 clips ->
        (out, views): out f16 [sum T, 3, crop, crop] (1-D when the clips' crops differ), views[i] the [T_i, 3, h, w] slice
        of clip i, bit-identical to self(clips[i]).  out and workspace (the sum of workspace_bytes
        over the clips) may be given."""
        return self._many(clips, out, workspace)


class Qwen2VLFramePreprocessor(_FramePreprocessor):
    """Qwen2-VL side: frames -> {'pixel_values_videos': fp32 [t*gh*gw, 1176] on the device, 'video_grid_thw': int64
    [[t, gh, gw]] on the host}, the dict embed_new_video_clip(**video_inputs) takes, equal to what
    FlashVStreamQwen2VLImageProcessor makes of the clip (smart_resize to a multiple of 28 * additional_pool_size, bicubic
    resize, rescale, normalize, patchify).  A one-frame clip fills both temporal slots; an odd frame count > 1 is refused,
    as the reference's reshape fails there.  The defaults are Qwen2VLImageProcessor's.
    codes=True returns uint8 rows instead (FVS_PRE_QWEN_CODES, DESIGN.md §3.20): the same rows and columns holding the
    resampled byte u, which the fp32 row element table[column // 392][u] is a function of; `device_table` is that
    table, which qwen.ops.pixel_decode decodes them through."""
    _layout = _lib.PRE_QWEN

    def __init__(self, min_pixels: int = 56 * 56, max_pixels: int = 28 * 28 * 1280, additional_pool_size: int = 1,
                 image_mean=OPENAI_CLIP_MEAN, image_std=OPENAI_CLIP_STD, rescale_factor: float = 1 / 255, device=None):
        self.min_pixels, self.max_pixels, self.pool = int(min_pixels), int(max_pixels), int(additional_pool_size)
        super().__init__(value_table(rescale_factor, image_mean, image_std), device)

    def resized(self, height: int, width: int) -> tuple[int, int]:
        return smart_resize(height, width, QWEN_PATCH * QWEN_MERGE * self.pool, self.min_pixels, self.max_pixels)

    def grid_thw(self, frames: int, height: int, width: int) -> tuple[int, int, int]:
        rh, rw = self.resized(height, width)
        return max(frames, QWEN_TEMPORAL) // QWEN_TEMPORAL, rh // QWEN_PATCH, rw // QWEN_PATCH

    def _windows(self, height, width):
        rh, rw = self.resized(height, width)
        return (rh, 0, rh), (rw, 0, rw), self.pool

    def output_shape(self, frames, height, width):
        t, gh, gw = self.grid_thw(frames, height, width)
        return (t * gh * gw, 3 * QWEN_TEMPORAL * QWEN_PATCH * QWEN_PATCH)

    def device_table(self, device=None):
        """the float32 [3, 256] value table on `device` (default: this preprocessor's), the one a call reads"""
        return self._table(device if device is not None else self._device())

    def __call__(self, frames, out=None, workspace=None, codes: bool = False):
        import torch
        pixels = self._run(frames, out, workspace, _lib.PRE_QWEN_CODES if codes else None)
        T, H, W = (int(v) for v in frames.shape[:3])
        return {"pixel_values_videos": pixels, "video_grid_thw": torch.tensor([self.grid_thw(T, H, W)], dtype=torch.int64)}

    def many(self, clips, out=None, workspace=None, codes: bool = False):
        """Many clips (a list of uint8 [T, H, W, 3], host or device, any mix of sizes) in one launch pair per 32 clips ->
        (out, views, grids): out fp32 [sum t*gh*gw, 1176] (uint8 with codes=True), views[i] clip i's rows and grids[i]
        its int64 [[t, gh, gw]] (host), bit-identical to self(clips[i]).  out and workspace (the sum of workspace_bytes
        over the clips) may be given."""
        import torch
        out, views = self._many(clips, out, workspace, _lib.PRE_QWEN_CODES if codes else None)
        grids = [torch.tensor([self.grid_thw(*(int(v) for v in f.shape[:3]))], dtype=torch.int64) for f in clips]
        return out, views, grids


# ---- qwen_vl_utils.fetch_video, list-of-frames branch (Flash-VStream-Qwen/qwen_vl_utils/vision_process.py) ----------
FETCH_IMAGE_FACTOR, FETCH_MIN_PIXELS, FETCH_MAX_PIXELS, FETCH_MAX_RATIO = 28, 4 * 28 * 28, 16384 * 28 * 28, 200  # :15-18
VIDEO_MIN_PIXELS, VIDEO_MAX_PIXELS, VIDEO_TOTAL_PIXELS = 128 * 28 * 28, 768 * 28 * 28, 24576 * 28 * 28        # :20-22
FRAME_FACTOR, FPS_MAX_FRAMES = 2, 768                                                                         # :23, :26


def fetch_smart_resize(height: int, width: int, factor: int = FETCH_IMAGE_FACTOR, min_pixels=FETCH_MIN_PIXELS,
                       max_pixels=FETCH_MAX_PIXELS) -> tuple[int, int]:
    """qwen_vl_utils' smart_resize (vision_process.py:44-70), the one fetch_image calls: unlike transformers' it keeps
    each rounded side at least `factor`, and max_pixels may be a float"""
    if max(height, width) / min(height, width) > FETCH_MAX_RATIO:
        raise ValueError(f"absolute aspect ratio must be smaller than {FETCH_MAX_RATIO}, got "
                         f"{max(height, width) / min(height, width)}")
    h_bar = max(factor, round(height / factor) * factor)
    w_bar = max(factor, round(width / factor) * factor)
    if h_bar * w_bar > max_pixels:
        beta = math.sqrt((height * width) / max_pixels)
        h_bar = math.floor(height / beta / factor) * factor
        w_bar = math.floor(width / beta / factor) * factor
    elif h_bar * w_bar < min_pixels:
        beta = math.sqrt(min_pixels / (height * width))
        h_bar = math.ceil(height * beta / factor) * factor
        w_bar = math.ceil(width * beta / factor) * factor
    return h_bar, w_bar


def _fetch_budget(n_frames: int, ele: dict):
    """(nframes, min_pixels, max_pixels) of fetch_video's list branch (vision_process.py:197-211): max_pixels comes from
    the frame count before the even-count padding"""
    nframes = n_frames
    if nframes > ele.get("max_frames", FPS_MAX_FRAMES):
        nframes = math.floor(ele.get("max_frames", FPS_MAX_FRAMES) / FRAME_FACTOR) * FRAME_FACTOR
    if nframes < 1:    # the reference divides by it next
        raise ValueError(f"no frame to fetch: {n_frames} frames, max_frames {ele.get('max_frames', FPS_MAX_FRAMES)}")
    min_pixels = ele.get("min_pixels", VIDEO_MIN_PIXELS)
    total_pixels = ele.get("total_pixels", VIDEO_TOTAL_PIXELS)
    max_pixels = max(min(VIDEO_MAX_PIXELS, total_pixels / nframes * FRAME_FACTOR), min_pixels * 1.05)
    return nframes, min_pixels, ele.get("max_pixels", max_pixels)


def fetch_video_picks(n_frames: int, ele: dict) -> list[int]:
    """the indices into ele['video'] of the frames fetch_video returns, in order (vision_process.py:217-221): the
    torch.linspace(...).round() pick, the `i in idx` selection, then the last pick repeated up to an even count"""
    import torch
    nframes, _, _ = _fetch_budget(n_frames, ele)
    idx = set(torch.linspace(0, n_frames - 1, nframes).round().long().tolist())
    picks = [i for i in range(n_frames) if i in idx]
    return picks + picks[-1:] * (math.ceil(len(picks) / FRAME_FACTOR) * FRAME_FACTOR - len(picks))


def fetch_video_size(height: int, width: int, n_frames: int, ele: dict) -> tuple[int, int]:
    """(resized_height, resized_width) fetch_image gives a height x width frame of a list of n_frames
    (vision_process.py:207-215, :96-113): resized_height / resized_width, when both are given, go through smart_resize
    with fetch_image's default pixel bounds; otherwise the frame's own size does, with the video's bounds"""
    if "resized_height" in ele and "resized_width" in ele:
        h, w = fetch_smart_resize(ele["resized_height"], ele["resized_width"])
    else:
        _, min_pixels, max_pixels = _fetch_budget(n_frames, ele)
        h, w = fetch_smart_resize(height, width, min_pixels=min_pixels, max_pixels=max_pixels)
    if h <= 0 or w <= 0:
        raise ValueError(f"a {height}x{width} frame resizes to {h}x{w}")
    return h, w


def _decoded(frame) -> np.ndarray:
    """one frame of a fetch_video list as uint8 [H, W, 3]: a path or PIL image the way fetch_image reads it (PIL,
    .convert('RGB')), an array as it is"""
    from PIL import Image
    if isinstance(frame, (str, os.PathLike)):
        path = os.fspath(frame)
        with Image.open(path[7:] if path.startswith("file://") else path) as im:
            return np.asarray(im.convert("RGB"))
    if isinstance(frame, Image.Image):
        return np.asarray(frame.convert("RGB"))
    a = np.asarray(frame)
    if a.dtype != np.uint8 or a.ndim != 3 or a.shape[2] != 3:
        raise ValueError(f"a frame must be a path, a PIL image or uint8 [H, W, 3], got {a.dtype} {a.shape}")
    return a


class Qwen2VLVideoFetcher:
    """The two pre-processing steps of Qwen2-VL's evaluation drivers (inference_mcq_vqa.py:290-334) on the GPU,
    bit-identical: qwen_vl_utils.fetch_video on a list of frames (vision_process.py:192-222: the frame pick, fetch_image's
    Pillow BICUBIC resize to a multiple of 28, the even-count padding), then FlashVStreamQwen2VLImageProcessor on its
    result (the second resize to a multiple of 28 * additional_pool_size, rescale, normalize, patchify), the second
    step configured by `preprocessor` (default: Qwen2VLImageProcessor's settings).

    An element is fetch_video's {'video': [frame, ...], 'max_frames', 'min_pixels', 'max_pixels', 'total_pixels',
    'resized_height', 'resized_width'}, all keys but 'video' optional.  A frame is a decoded uint8 [H, W, 3] array, a
    PIL image, or a path, which is decoded and converted to RGB with PIL on the host, in a thread pool.  Only the picked
    frames are decoded and copied to the device, and every size is worked out before the copy, so a refused element
    copies nothing.  The frames of one video must decode to one size (fetch_image would resize each on its own)."""

    def __init__(self, preprocessor: Qwen2VLFramePreprocessor | None = None, decode_threads: int | None = None):
        self.pre = preprocessor if preprocessor is not None else Qwen2VLFramePreprocessor()
        self.decode_threads = int(decode_threads or min(32, os.cpu_count() or 1))

    def _load(self, ele):
        """-> (host uint8 [n, H, W, 3] frames of the fetched video, padding included, as a list of arrays, (h1, w1))"""
        video = ele.get("video") if isinstance(ele, dict) else None
        if not isinstance(video, (list, tuple)):
            raise TypeError("a fetch_video element with a list of frames ({'video': [frame, ...], ...}) is expected")
        picks = fetch_video_picks(len(video), ele)
        unique = sorted(set(picks))
        if any(isinstance(video[i], (str, os.PathLike)) for i in unique) and len(unique) > 1:
            with ThreadPoolExecutor(min(self.decode_threads, len(unique))) as pool:
                decoded = dict(zip(unique, pool.map(lambda i: _decoded(video[i]), unique)))
        else:
            decoded = {i: _decoded(video[i]) for i in unique}
        sizes = {decoded[i].shape[:2] for i in unique}
        if len(sizes) != 1:
            raise ValueError(f"the frames of one video decode to more than one size: {sorted(sizes)}")
        (H, W), = sizes
        return [decoded[i] for i in picks], fetch_video_size(H, W, len(video), ele)

    def _submit(self, eles, codes=None):
        """every element through one fvs_preprocess_multi call -> (flat out, [(element offset, T, (h1, w1))])
        codes=None: the fetched images themselves (FVS_PRE_RGB8); else the processor's rows (two-stage jobs)"""
        import torch
        if not isinstance(eles, (list, tuple)) or not eles:
            raise ValueError("a non-empty list of fetch_video elements is expected")
        loaded = [self._load(e) for e in eles]          # every refusal of the host arithmetic happens here
        pre, device = self.pre, self.pre._device()
        layout = _lib.PRE_RGB8 if codes is None else _lib.PRE_QWEN_CODES if codes else _lib.PRE_QWEN
        n = len(loaded)
        jobs = (_lib.PreprocessJob * n)()
        hosts = []
        for i, (frames, (h1, w1)) in enumerate(loaded):
            T, (H, W) = len(frames), frames[0].shape[:2]
            x, y, _ = pre._axes(device, H, W, (h1, 0, h1), (w1, 0, w1))
            host = torch.empty((T, H, W, 3), dtype=torch.uint8, pin_memory=True)
            np.stack(frames, out=host.numpy())
            hosts.append(host)
            jobs[i] = _lib.PreprocessJob(host.data_ptr(), T, H, W, 3, x, y)
            if codes is not None:
                h2, w2 = pre.resized(h1, w1)
                jobs[i].x2, jobs[i].y2, _ = pre._axes(device, h1, w1, (h2, 0, h2), (w2, 0, w2))
        lib = _lib.load()
        plan, totals = (C.c_int64 * (4 * n))(), (C.c_int64 * 2)()
        r = lib.fvs_preprocess_plan(jobs, n, layout, pre.pool, plan, totals)
        if r < 0:
            _lib.check(r, "fvs_preprocess_plan")
        frames = [h.to(device, non_blocking=True) for h in hosts]
        for i, f in enumerate(frames):
            jobs[i].frames = f.data_ptr()
        out = torch.empty(int(totals[0]), dtype=pre._out_dtype(layout), device=device)
        workspace = torch.empty(int(totals[1]), dtype=torch.uint8, device=device)
        with torch.cuda.device(device):
            _lib.check(lib.fvs_preprocess_multi(jobs, n, pre._table(device).data_ptr(), layout, pre.pool,
                                                out.data_ptr(), workspace.data_ptr(), workspace.numel(),
                                                _lib.cur_stream()), "fvs_preprocess_multi")
        return out, [(int(plan[4 * i + 2]), len(f), s) for i, (f, s) in enumerate(loaded)]

    def fetch(self, ele):
        """-> uint8 [n, h1, w1, 3] on the device: np.stack([np.asarray(im) for im in fetch_video(ele)])"""
        out, [(_, T, (h1, w1))] = self._submit([ele])
        return out.view(T, h1, w1, 3)

    def many(self, eles, codes: bool = False):
        """-> {'pixel_values_videos': fp32 [sum t*gh*gw, 1176] on the device (uint8 codes with codes=True, as
        Qwen2VLFramePreprocessor gives), 'video_grid_thw': int64 [len(eles), 3] on the host}: what the image processor
        returns for videos=[fetch_video(e) for e in eles], every video in one launch group per 32 videos"""
        import torch
        out, parts = self._submit(eles, codes=bool(codes))
        grids = [self.pre.grid_thw(T, h1, w1) for _, T, (h1, w1) in parts]
        return {"pixel_values_videos": out.view(-1, 3 * QWEN_TEMPORAL * QWEN_PATCH * QWEN_PATCH),
                "video_grid_thw": torch.tensor(grids, dtype=torch.int64)}

    def __call__(self, ele, codes: bool = False):
        return self.many([ele], codes)


def qwen_preprocessor_of(image_processor, additional_pool_size: int = 1, device=None) -> Qwen2VLFramePreprocessor:
    """the Qwen2VLFramePreprocessor that computes what `image_processor` (a FlashVStreamQwen2VLImageProcessor, or
    transformers' Qwen2VLImageProcessor) does to a video with additional_pool_size; raises NotImplementedError for a
    configuration the kernels do not reproduce"""
    p = image_processor
    resample = getattr(p, "resample", None)
    if resample is None or int(resample) != BICUBIC:
        raise NotImplementedError(f"resample={resample!r}: only bicubic ({BICUBIC}) is implemented")
    if not getattr(p, "do_resize", True):
        raise NotImplementedError("do_resize=False is not implemented")
    if (getattr(p, "patch_size", QWEN_PATCH), getattr(p, "merge_size", QWEN_MERGE),
            getattr(p, "temporal_patch_size", QWEN_TEMPORAL)) != (QWEN_PATCH, QWEN_MERGE, QWEN_TEMPORAL):
        raise NotImplementedError("only patch_size 14, merge_size 2 and temporal_patch_size 2 are implemented")
    size = getattr(p, "size", None)
    min_pixels = getattr(p, "min_pixels", None) or _field(size, "shortest_edge")
    max_pixels = getattr(p, "max_pixels", None) or _field(size, "longest_edge")
    norm = getattr(p, "do_normalize", True)
    return Qwen2VLFramePreprocessor(min_pixels, max_pixels, additional_pool_size,
                                    p.image_mean if norm else None, p.image_std if norm else None,
                                    p.rescale_factor if getattr(p, "do_rescale", True) else None, device)


class Qwen2VLVideoImageProcessor:
    """A stand-in for a Qwen2-VL processor's `image_processor` (install.install_qwen_fetch): a videos= call whose videos
    are all device uint8 [n, h, w, 3] tensors (what Qwen2VLVideoFetcher.fetch returns) is pre-processed on the GPU, one
    launch pair per 32 videos, into the BatchFeature the wrapped processor returns for the same frames: the fp32 rows
    'pixel_values_videos' on the device and the int64 'video_grid_thw' on the host.  Any other call, and every other
    attribute, is the wrapped processor's own."""

    def __init__(self, image_processor, device=None):
        self.__dict__["image_processor"] = image_processor
        self.__dict__["device"] = device
        self.__dict__["_pre"] = {}

    def __getattr__(self, name):
        return getattr(self.__dict__["image_processor"], name)

    def __call__(self, images=None, videos=None, return_tensors=None, additional_pool_size: int = 1, **kwargs):
        import torch
        if (images is not None or kwargs or not isinstance(videos, (list, tuple)) or not videos or
                not all(isinstance(v, torch.Tensor) and v.is_cuda and v.dtype == torch.uint8 for v in videos)):
            return self.image_processor(images=images, videos=videos, return_tensors=return_tensors,
                                        additional_pool_size=additional_pool_size, **kwargs)
        pre = self._pre.get(additional_pool_size)
        if pre is None:
            pre = self._pre[additional_pool_size] = qwen_preprocessor_of(self.image_processor, additional_pool_size,
                                                                         self.device)
        out, _, grids = pre.many(list(videos))
        from transformers.feature_extraction_utils import BatchFeature
        return BatchFeature(data={"pixel_values_videos": out, "video_grid_thw": torch.cat(grids)})
