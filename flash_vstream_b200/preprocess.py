"""Frame pre-processing on the GPU: decoded uint8 RGB frames -> the pixels the vision towers take, bit-identical to the
reference's CPU image processors (fvs_preprocess, csrc/preprocess_kernels.cu).

    CLIPFramePreprocessor(image_processor)(frames)   == image_processor.preprocess(clip)['pixel_values'].half()
                                                        (Flash-VStream-LLaVA/flash_vstream/serve/cli_video_stream.py:186)
    Qwen2VLFramePreprocessor(...)(frames)            == the {'pixel_values_videos', 'video_grid_thw'} of
                                                        FlashVStreamQwen2VLImageProcessor (cli_server_2gpu.py:214-219)

Frames are [T, H, W, 3] uint8 (what decord and np.asarray(PIL image) give): a CUDA tensor, or a host tensor / array
that is copied to the device (non_blocking, so a pinned one does not block the host).  The resize is Pillow's BICUBIC
resample, which is integer arithmetic; rescale + normalize are a function of one byte per channel, so they are a
float32 [3, 256] table built here with transformers' numpy operations.  Inference only, like the rest of the package.
"""
from __future__ import annotations

import ctypes as C
import math

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

    def _plan(self, device, height, width):
        import torch
        key = (device, height, width)
        plan = self._plans.get(key)
        if plan is None:
            (oh, fy, cy), (ow, fx, cx), pool = self._windows(height, width)
            keep, axes = [], []
            for size_in, size_out, first, count in ((width, ow, fx, cx), (height, oh, fy, cy)):
                ax, bounds, coeffs = resample_plan(size_in, size_out, first, count)
                b, k = torch.from_numpy(bounds).to(device), torch.from_numpy(coeffs).to(device)
                ax.bounds, ax.coeffs = b.data_ptr(), k.data_ptr()
                keep += [b, k]
                axes.append(ax)
            plan = self._plans[key] = (axes[0], axes[1], pool, keep)
        return plan

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
        return {_lib.PRE_CLIP: torch.float16, _lib.PRE_QWEN: torch.float32, _lib.PRE_QWEN_CODES: torch.uint8}[layout]

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
