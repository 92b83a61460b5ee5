"""CPU checks of the frame pre-processing: the numpy oracle against Pillow and the transformers processors, the library's
host plans against the oracle, the size restatements against transformers, and the refusals of fvs_preprocess."""
from __future__ import annotations

import ctypes as C
import os
import zlib

import numpy as np
import pytest
from PIL import Image

from flash_vstream_b200 import _lib
from flash_vstream_b200 import preprocess as P
from tests import preprocess_inputs as PI
from tests import preprocess_oracle as O

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "preprocess.npz")


def _size_pairs():
    rng = np.random.default_rng(2026)
    pairs = [(1, 1, 1, 1), (1, 7, 8, 56), (5, 1, 40, 8), (7, 9, 56, 72), (12, 3, 1, 1), (3, 40, 3, 1), (480, 640, 336, 448),
             (720, 1280, 336, 597), (100, 90, 336, 302), (1080, 1920, 448, 784), (333, 501, 224, 336)]
    while len(pairs) < 220:
        h, w = (int(v) for v in rng.integers(1, 200, 2))
        kind = rng.integers(0, 3)
        if kind == 0:                                  # downscale, up to 12x
            H, W = (int(max(1, v // rng.integers(1, 13))) for v in (h, w))
        elif kind == 1:                                # upscale, up to 8x
            H, W = (int(v * rng.integers(1, 9)) for v in (h, w))
        else:                                          # anything
            H, W = (int(v) for v in rng.integers(1, 300, 2))
        pairs.append((h, w, H, W))
    return pairs


def test_oracle_equals_pillow_bicubic():
    rng = np.random.default_rng(7)
    for h, w, H, W in _size_pairs():
        img = rng.integers(0, 256, (h, w, 3), dtype=np.uint8)
        ref = np.asarray(Image.fromarray(img).resize((W, H), Image.BICUBIC))
        assert np.array_equal(O.resize(img, H, W), ref), (h, w, H, W)


def test_library_plans_equal_oracle():
    for h, w, H, W in _size_pairs()[:120]:
        for n_in, n_out in ((w, W), (h, H)):
            ax, bounds, coeffs = P.resample_plan(n_in, n_out)
            ob, oc = O.axis_plan(n_in, n_out)
            assert ax.taps == oc.shape[1] and np.array_equal(bounds, ob) and np.array_equal(coeffs, oc), (n_in, n_out)
            first, count = n_out // 3, max(1, n_out // 2)       # a window is the same rows of the whole plan
            ax, bounds, coeffs = P.resample_plan(n_in, n_out, first, count)
            assert np.array_equal(bounds, ob[first:first + count]) and np.array_equal(coeffs, oc[first:first + count])
            assert ax.span_first == ob[first, 0] and ax.span_first + ax.span_count == ob[first + count - 1].sum()


def test_value_table_equals_oracle():
    for args in ((None, None, None), (1 / 255, None, None), (None, PI.OPENAI_CLIP_MEAN, PI.OPENAI_CLIP_STD),
                 (1 / 255, PI.OPENAI_CLIP_MEAN, PI.OPENAI_CLIP_STD), (0.5, 0.5, 0.25)):
        a = P.value_table(*args)
        b = O.value_table(args[0], None if args[1] is None else np.broadcast_to(args[1], 3),
                          None if args[2] is None else np.broadcast_to(args[2], 3))
        assert a.dtype == np.float32 and a.shape == (3, 256) and np.array_equal(a.view(np.int32), b.view(np.int32))


def _clip_processor(se=336, crop=336):
    from transformers.models.clip.image_processing_pil_clip import CLIPImageProcessorPil
    return CLIPImageProcessorPil(size={"shortest_edge": se}, crop_size={"height": crop, "width": crop})


def _oracle_clip(proc_gpu, frames):
    T, H, W, _ = frames.shape
    resized, crop = proc_gpu.sizes(H, W)
    return O.clip_pixels(frames, resized, crop, proc_gpu.table)


@pytest.mark.parametrize("shape", [(1, 480, 640), (1, 90, 100), (2, 200, 120), (1, 336, 500)])
def test_oracle_clip_equals_transformers_pil_processor(shape):
    frames = PI.frames(sum(shape), shape)
    hf = _clip_processor()
    ref = hf.preprocess(list(frames), return_tensors="np")["pixel_values"]
    mine = _oracle_clip(P.CLIPFramePreprocessor(hf), frames)
    assert mine.shape == ref.shape and np.array_equal(mine.view(np.int32), ref.astype(np.float32).view(np.int32))


def test_oracle_equals_goldens():
    g = np.load(GOLDEN)
    for name, (seed, shape, se, crop) in PI.CLIP_CASES.items():
        f = PI.frames(seed, shape)
        assert zlib.crc32(f.tobytes()) == int(g[f"clip_{name}_crc"]), f"seeded frames of {name} changed"
        pix = _oracle_clip(P.CLIPFramePreprocessor(_clip_processor(se, crop)), f).astype(np.float16)
        assert np.array_equal(pix.view(np.int16), g[f"clip_{name}"].view(np.int16)), name
    for name, (seed, shape, mn, mx, pool) in PI.QWEN_CASES.items():
        f = PI.frames(seed, shape)
        assert zlib.crc32(f.tobytes()) == int(g[f"qwen_{name}_crc"]), f"seeded frames of {name} changed"
        q = P.Qwen2VLFramePreprocessor(mn, mx, pool)
        pix, grid = O.qwen_pixels(f, q.resized(*shape[1:]), q.table)
        assert grid == tuple(g[f"qwen_{name}_grid"]) == q.grid_thw(*shape), name
        assert np.array_equal(pix.view(np.int32), g[f"qwen_{name}"].view(np.int32)), name
        assert q.output_shape(*shape) == pix.shape


def test_size_restatements_equal_transformers():
    from transformers.image_transforms import center_crop, get_resize_output_image_size
    from transformers.models.qwen2_vl.image_processing_qwen2_vl import smart_resize
    rng = np.random.default_rng(3)
    for _ in range(300):
        h, w = (int(v) for v in rng.integers(1, 4000, 2))
        se = int(rng.choice([224, 336, 384, 17]))
        assert P.clip_resize_size(h, w, se) == get_resize_output_image_size(
            np.zeros((3, h, w), np.uint8), se, default_to_square=False, input_data_format="channels_first")
        if max(h, w) / min(h, w) <= 200:
            for factor in (28, 56, 84):
                for mn, mx in ((56 * 56, 28 * 28 * 1280), (112 * 112, 56 * 56 * 16), (4, 14 * 14 * 4 * 1280)):
                    assert P.smart_resize(h, w, factor, mn, mx) == smart_resize(h, w, factor, mn, mx), (h, w, factor)
    for h, w, ch, cw in ((100, 120, 84, 84), (101, 133, 84, 84), (336, 597, 336, 336), (597, 336, 336, 336), (7, 9, 2, 3)):
        idx = np.arange(h * w, dtype=np.int64).reshape(1, h, w)
        top, left = P.center_crop_offsets(h, w, ch, cw)
        assert np.array_equal(center_crop(idx, (ch, cw), input_data_format="channels_first"),
                              idx[:, top:top + ch, left:left + cw])


def test_clip_preprocessor_refuses_unsupported_knobs():
    with pytest.raises(NotImplementedError, match="resample"):
        P.CLIPFramePreprocessor(_clip_processor().__class__(resample=2))
    with pytest.raises(NotImplementedError, match="size"):
        P.CLIPFramePreprocessor(_clip_processor().__class__(size={"height": 336, "width": 336}))
    with pytest.raises(NotImplementedError, match="do_pad"):
        P.CLIPFramePreprocessor(_clip_processor().__class__(do_pad=True))


def _axis(in_size, out_size, first=0, count=None):
    ax, _, _ = P.resample_plan(in_size, out_size, first, count)
    ax.bounds, ax.coeffs = 64, 128            # never read: every call below is refused before a launch
    return ax


def test_malformed_calls_are_refused():
    lib = _lib.load()
    n0 = lib.fvs_launch_count()
    x, y = _axis(64, 56), _axis(48, 42)
    ws = lib.fvs_preprocess_workspace_bytes(C.byref(x), C.byref(y), 2)
    assert ws == 2 * 3 * y.span_count * 56
    good = dict(frames=256, T=2, H=48, W=64, C=3, x=x, y=y, table=512, layout=_lib.PRE_CLIP, pool=1, out=1024, ws=2048,
                wsb=ws)

    def call(**kw):
        a = dict(good, **kw)
        return lib.fvs_preprocess(a["frames"], a["T"], a["H"], a["W"], a["C"], C.byref(a["x"]), C.byref(a["y"]), a["table"],
                                  a["layout"], a["pool"], a["out"], a["ws"], a["wsb"], None)

    bad = [dict(frames=None), dict(table=None), dict(out=None), dict(ws=None), dict(C=4), dict(C=1), dict(T=0), dict(H=0),
           dict(W=0), dict(wsb=ws - 1), dict(layout=7), dict(W=65), dict(H=47),
           dict(layout=_lib.PRE_QWEN),                              # 42x56 is not a multiple of 28
           dict(x=_axis(64, 56), y=_axis(48, 56), layout=_lib.PRE_QWEN, T=3,
                wsb=1 << 20),                                       # an odd frame count > 1
           dict(x=_axis(64, 56), y=_axis(48, 56), layout=_lib.PRE_QWEN, pool=3, wsb=1 << 20),   # 56 is not a multiple of 28 * 3
           dict(x=_axis(64, 56, 0, 28), y=_axis(48, 56), layout=_lib.PRE_QWEN, wsb=1 << 20),   # a crop in the Qwen layout
           ]
    tampered = _axis(64, 56)
    tampered.taps += 1
    bad.append(dict(x=tampered))
    crop = _axis(64, 56, 10, 46)
    crop.count = 47                                                  # a crop window beyond the resized image
    bad.append(dict(x=crop))
    unaligned = _axis(64, 56)
    unaligned.bounds = 68
    bad.append(dict(x=unaligned))
    nulltab = _axis(64, 56)
    nulltab.coeffs = None
    bad.append(dict(x=nulltab))
    for kw in bad:
        assert call(**kw) == _lib.FVS_EINVAL, kw
    ax = _lib.ResampleAxis()
    for args in ((0, 5, 0, 5), (5, 0, 0, 1), (5, 8, -1, 3), (5, 8, 6, 3), (5, 8, 0, 0)):
        assert lib.fvs_resample_plan(*args, C.byref(ax), None, None) == _lib.FVS_EINVAL, args
    assert lib.fvs_resample_plan(5, 8, 0, 8, None, None, None) == _lib.FVS_EINVAL
    assert lib.fvs_launch_count() == n0


def test_frames_must_be_uint8_rgb():
    q = P.Qwen2VLFramePreprocessor()
    with pytest.raises(ValueError, match="uint8"):
        q(np.zeros((2, 56, 56, 3), np.float32))
    with pytest.raises(TypeError):
        q([np.zeros((56, 56, 3), np.uint8)])
