"""numpy restatement of the frame pre-processing (test infrastructure only): Pillow's fixed-point BICUBIC resample of an
8-bit RGB image, the rescale/normalize table, the CLIP center crop and both output layouts.

The resample follows Pillow's src/libImaging/Resample.c: per-axis coefficients in double (filter a = -0.5, support
2 * max(scale, 1), PIL's center / xmin / xmax rounding), normalised by their sum and converted to int32 with 22
fractional bits rounding half away from zero; a horizontal pass into a clipped uint8 intermediate, then a vertical pass;
each accumulator starts at 1 << 21, is shifted right by 22 and clamped to [0, 255].  A pass whose length does not change
is skipped, as Pillow does (it is the identity anyway)."""
from __future__ import annotations

import math

import numpy as np

PRECISION_BITS = 22


def bicubic(x: float) -> float:
    a = -0.5
    if x < 0.0:
        x = -x
    if x < 1.0:
        return ((a + 2.0) * x - (a + 3.0)) * x * x + 1
    if x < 2.0:
        return (((x - 5) * x + 8) * x - 4) * a
    return 0.0


def axis_plan(in_size: int, out_size: int):
    """bounds int64 [out, 2] = {xmin, n}, coeffs int64 [out, taps] of the whole in_size -> out_size axis"""
    scale = float(in_size) / out_size
    filterscale = max(scale, 1.0)
    support = 2.0 * filterscale
    taps = int(math.ceil(support)) * 2 + 1
    bounds = np.zeros((out_size, 2), np.int64)
    coeffs = np.zeros((out_size, taps), np.int64)
    ss = 1.0 / filterscale
    for xx in range(out_size):
        center = (xx + 0.5) * scale
        xmin = max(int(center - support + 0.5), 0)
        xmax = min(int(center + support + 0.5), in_size) - xmin
        k = [bicubic((x + xmin - center + 0.5) * ss) for x in range(xmax)]
        ww = 0.0
        for w in k:
            ww += w
        for x, w in enumerate(k):
            if ww != 0.0:
                w = w / ww
            coeffs[xx, x] = int(-0.5 + w * (1 << PRECISION_BITS)) if w < 0 else int(0.5 + w * (1 << PRECISION_BITS))
        bounds[xx] = (xmin, xmax)
    return bounds, coeffs


def _pass(img: np.ndarray, bounds, coeffs, axis: int) -> np.ndarray:
    """one 1-D pass over `axis` of a uint8 array"""
    src = np.moveaxis(img, axis, 0).astype(np.int64)
    taps = coeffs.shape[1]
    idx = np.minimum(bounds[:, :1] + np.arange(taps)[None, :], src.shape[0] - 1)   # unused taps carry coefficient 0
    acc = np.full((bounds.shape[0],) + src.shape[1:], 1 << (PRECISION_BITS - 1), np.int64)
    for j in range(taps):
        k = coeffs[:, j].reshape((-1,) + (1,) * (src.ndim - 1))
        acc += src[idx[:, j]] * k
    out = np.clip(acc >> PRECISION_BITS, 0, 255).astype(np.uint8)
    return np.moveaxis(out, 0, axis)


def resize(img: np.ndarray, out_h: int, out_w: int) -> np.ndarray:
    """== np.asarray(PIL.Image.fromarray(img).resize((out_w, out_h), BICUBIC)) for uint8 [..., H, W, 3]"""
    h, w = img.shape[-3], img.shape[-2]
    if out_w != w:
        img = _pass(img, *axis_plan(w, out_w), axis=img.ndim - 2)
    if out_h != h:
        img = _pass(img, *axis_plan(h, out_h), axis=img.ndim - 3)
    return img


def value_table(rescale_factor=None, mean=None, std=None) -> np.ndarray:
    """float32 [3, 256]: transformers' numpy rescale and normalize applied to every byte"""
    x = np.tile(np.arange(256, dtype=np.uint8), (3, 1))
    if rescale_factor is not None:
        x = (x.astype(np.float64) * rescale_factor).astype(np.float32)
    if mean is not None:
        x = x.astype(np.float32)
        x = (x - np.asarray(mean, np.float32)[:, None]) / np.asarray(std, np.float32)[:, None]
    return x.astype(np.float32)


def lookup(img_u8: np.ndarray, table: np.ndarray) -> np.ndarray:
    """[T, H, W, 3] uint8 -> float32 [T, 3, H, W] through the per-channel table"""
    return np.stack([table[c][img_u8[..., c]] for c in range(3)], axis=1)


def clip_pixels(frames: np.ndarray, resized: tuple, crop: tuple, table: np.ndarray) -> np.ndarray:
    """float32 [T, 3, ch, cw]: resize to `resized` (h, w), center crop (top, left, ch, cw), table"""
    top, left, ch, cw = crop
    r = resize(frames, *resized)[:, top:top + ch, left:left + cw]
    return lookup(r, table)


def qwen_patchify(pix: np.ndarray, patch=14, merge=2, temporal=2) -> tuple[np.ndarray, tuple]:
    """float32 [T, 3, H, W] -> ([t*gh*gw, 3*temporal*patch*patch], (t, gh, gw)): vstream_qwen2vl_processor.py:135-155"""
    if pix.shape[0] == 1:
        pix = np.tile(pix, (temporal, 1, 1, 1))
    T, C, H, W = pix.shape
    gt, gh, gw = T // temporal, H // patch, W // patch
    p = pix.reshape(gt, temporal, C, gh // merge, merge, patch, gw // merge, merge, patch)
    p = p.transpose(0, 3, 6, 4, 7, 2, 1, 5, 8)
    return np.ascontiguousarray(p.reshape(gt * gh * gw, C * temporal * patch * patch)), (gt, gh, gw)


def qwen_pixels(frames: np.ndarray, resized: tuple, table: np.ndarray):
    return qwen_patchify(lookup(resize(frames, *resized), table))
