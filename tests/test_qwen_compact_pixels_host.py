"""CPU tests of 8-bit pixel codes for lazy and bank-less Qwen2-VL streams (DESIGN.md §3.20): the codes and their decode
restated in NumPy against the pre-processing oracle and its goldens, the codes layout's host plan, the knob's refusals,
the checkpoint's tensor set and the restore refusals that need no device, the new entry points' refusals (returned
before any CUDA call, nothing launched), and the resource use of the new and the unchanged kernels."""
import os
import re
import subprocess
import zlib

import numpy as np
import pytest
import torch

from flash_vstream_b200 import _lib as L
from flash_vstream_b200 import preprocess as P
from tests import preprocess_inputs as PI
from tests import preprocess_oracle as O
from tests.test_qwen_no_bank_host import _flash, _refused

GOLDEN = os.path.join(os.path.dirname(__file__), "golden", "preprocess.npz")
CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"
A = 0x10000          # a 16-byte aligned stand-in address: the refusals happen before anything is dereferenced


def np_codes(frames, resized):
    """uint8 [t*gh*gw, 1176]: the resized bytes in the Qwen2-VL patch layout (what FVS_PRE_QWEN_CODES writes)"""
    r = O.resize(frames, *resized)                               # [T, H, W, 3] uint8
    return O.qwen_patchify(np.ascontiguousarray(np.moveaxis(r, -1, 1)))[0]


def np_decode(codes, table):
    """fp32 table[column // 392][code], the row element the codes stand for"""
    ch = np.arange(codes.shape[1]) // 392
    return table[ch[None, :], codes]


def test_codes_are_the_resized_bytes_and_decode_to_the_goldens():
    g = np.load(GOLDEN)
    for name, (seed, shape, mn, mx, pool) in PI.QWEN_CASES.items():
        f = PI.frames(seed, shape)
        assert zlib.crc32(f.tobytes()) == int(g[f"qwen_{name}_crc"]), f"seeded frames of {name} changed"
        q = P.Qwen2VLFramePreprocessor(mn, mx, pool)
        codes = np_codes(f, q.resized(*shape[1:]))
        assert codes.dtype == np.uint8 and codes.shape == g[f"qwen_{name}"].shape == q.output_shape(*shape)
        fp32 = np_decode(codes, q.table)
        assert np.array_equal(fp32.view(np.int32), g[f"qwen_{name}"].view(np.int32)), name
        want = torch.from_numpy(g[f"qwen_{name}"])
        for dt in (torch.bfloat16, torch.float16):                # the cast of the fp32 rows, element by element
            assert torch.equal(torch.from_numpy(fp32).to(dt).view(torch.int16), want.type(dt).view(torch.int16))


def test_channel_of_column():
    ch = np.arange(1176) // 392
    p = np.arange(3 * 2 * 14 * 14).reshape(3, 2, 14, 14)          # ((c*2 + tp)*14 + py)*14 + px
    assert np.array_equal(ch, np.repeat(np.arange(3), 392)) and np.array_equal(p.reshape(-1) // 392, ch)
    assert all(len(set(ch[w * 8: w * 8 + 8])) == 1 for w in range(147))   # an 8-code word never spans two channels


def _jobs(shapes):
    q = P.Qwen2VLFramePreprocessor(max_pixels=336 * 504)
    jobs = (L.PreprocessJob * len(shapes))()
    for i, (T, H, W) in enumerate(shapes):
        (oh, _, _), (ow, _, _), _ = q._windows(H, W)
        x, _, _ = P.resample_plan(W, ow)
        y, _, _ = P.resample_plan(H, oh)
        jobs[i] = L.PreprocessJob(A, T, H, W, 3, x, y)
    return jobs


def test_codes_layout_plans_as_the_qwen_layout():
    import ctypes as C
    lib = L.load()
    rng = np.random.default_rng(3)
    shapes = [(int(rng.choice([1, 2, 4])), int(rng.integers(40, 400)), int(rng.integers(40, 400))) for _ in range(40)]
    for n in (1, 7, 33, 40):
        jobs = _jobs(shapes[:n])
        for a in jobs:                                        # fake device tables: the plan dereferences none
            a.x.bounds = a.x.coeffs = a.y.bounds = a.y.coeffs = A
        out = {}
        for layout in (L.PRE_QWEN, L.PRE_QWEN_CODES):
            plan, tot = (C.c_int64 * (4 * n))(), (C.c_int64 * 2)()
            r = lib.fvs_preprocess_plan(jobs, n, layout, 1, plan, tot)
            assert r == (n + 31) // 32, lib.fvs_last_error()
            out[layout] = (list(plan), list(tot))
        assert out[L.PRE_QWEN] == out[L.PRE_QWEN_CODES]
    plan, tot = (C.c_int64 * 4)(), (C.c_int64 * 2)()
    odd = _jobs([(3, 112, 112)])
    odd[0].x.bounds = odd[0].x.coeffs = odd[0].y.bounds = odd[0].y.coeffs = A
    assert lib.fvs_preprocess_plan(odd, 1, L.PRE_QWEN_CODES, 1, plan, tot) == L.FVS_EINVAL
    assert "1 or an even number" in lib.fvs_last_error().decode()


# ---------------------------------------------------------------------------------------------------------- knobs
def test_knob_refusals():
    from flash_vstream_b200.qwen.stream_state import QwenStreamState, check_compact_pixels
    with pytest.raises(ValueError, match="compact_pixels=True needs lazy_full_res=True"):
        QwenStreamState(_flash(), None, compact_pixels=True)
    for bad in (1, None, "yes"):
        with pytest.raises(ValueError, match="compact_pixels must be True or False"):
            QwenStreamState(_flash(), None, lazy_full_res=True, compact_pixels=bad)
    for fr in (True, False):
        st = QwenStreamState(_flash(), None, lazy_full_res=True, full_res_bank=fr, compact_pixels=True)
        assert st.compact_pixels and st.pixel_table is None
    assert not QwenStreamState(_flash(), None, lazy_full_res=True).compact_pixels          # the default is off
    assert check_compact_pixels(False, False) is False


def _pool(**kw):
    from flash_vstream_b200.qwen import QwenStreamPool
    from flash_vstream_b200.qwen.vision_tower import QwenVisionBlocksB200
    from flash_vstream_b200.qwen.vstream_qwen2vl_realtime import FlashMemory, VisualB200

    class Model:
        visual = VisualB200(FlashMemory(flash_memory_temporal_length=8, flash_memory_spatial_length=6), None,
                            encode_patches=QwenVisionBlocksB200.__new__(QwenVisionBlocksB200), device="cuda:0")
    return QwenStreamPool(Model(), **kw)


def test_pool_knob_refusals():
    import inspect
    from flash_vstream_b200.qwen import QwenStreamPool
    assert inspect.signature(QwenStreamPool).parameters["compact_pixels"].default is False
    with pytest.raises(ValueError, match="compact_pixels=True needs lazy_full_res=True"):
        _pool(compact_pixels=True, preprocess=P.Qwen2VLFramePreprocessor())
    with pytest.raises(ValueError, match="compact_pixels=True needs preprocess=Qwen2VLFramePreprocessor"):
        _pool(compact_pixels=True, lazy_full_res=True)
    with pytest.raises(ValueError, match="compact_pixels=True needs preprocess=Qwen2VLFramePreprocessor"):
        _pool(compact_pixels=True, lazy_full_res=True, full_res_bank=False, preprocess=object())
    pool = _pool(compact_pixels=True, lazy_full_res=True, full_res_bank=False, preprocess=P.Qwen2VLFramePreprocessor())
    assert pool.compact_pixels and not pool.full_res_bank


def test_pool_refuses_pixel_clips():
    """a compact pool takes uint8 frames only: a round of (pixels, grid) clips raises before anything is enqueued"""
    from flash_vstream_b200.qwen.multistream import _Stream
    from flash_vstream_b200.qwen.stream_state import QwenStreamState
    pool = _pool(compact_pixels=True, lazy_full_res=True, preprocess=P.Qwen2VLFramePreprocessor())
    calls = []
    pool.tower = pool._encode = lambda *a: calls.append(a)
    pool._streams = {0: _Stream(pool.visual, QwenStreamState(pool.flash, None, lazy_full_res=True, compact_pixels=True))}
    with pytest.raises(ValueError, match="compact_pixels pool keeps uint8 codes"):
        pool.step({0: (torch.zeros(64, 1176), torch.tensor([[1, 8, 8]]))})
    assert calls == [] and pool.state(0).n_frames == 0


# ---------------------------------------------------------------------------------------------------------- checkpoints
def _ckpt(compact, pix_frames=2, table=None):
    from flash_vstream_b200 import checkpoint as CK
    n, h, w, hs, ws, D = 4, 4, 4, 2, 2, 16
    cfg = {"flash": dict(_flash().config), "grid": [h, w], "small_grid": [hs, ws], "dtype": "bfloat16", "dim": D,
           "merger_dim": None}
    enc = torch.tensor([1] * (n - pix_frames) + [0] * pix_frames, dtype=torch.uint8)
    cnt = {"n_frames": n, "steps": n, "n_tem": 2, "n_spa": 2, "fast_steps": 0, "redone_steps": 0, "merged": 0,
           "tem_weights_dtype": "float32", "tem_timestamp_dtype": "float32", "pix_frames": pix_frames}
    bf = torch.bfloat16
    t = {"bank_x": torch.zeros(n, h * w, D, dtype=bf), "bank_small": torch.zeros(n, hs * ws, D, dtype=bf),
         "tem_x": torch.zeros(2 * hs * ws, D, dtype=bf), "tem_timestamp": torch.zeros(2), "tem_weights": torch.ones(2),
         "spa_positions": torch.zeros(2, dtype=torch.int64), "encoded": enc}
    if compact:
        cfg["compact_pixels"] = True
        t["pix_codes"] = torch.zeros(pix_frames, h * w * 1176, dtype=torch.uint8)
        t["pixel_table"] = torch.from_numpy(P.value_table(1 / 255, PI.OPENAI_CLIP_MEAN, PI.OPENAI_CLIP_STD)) \
            if table is None else table
    else:
        t["pixels"] = torch.zeros(pix_frames, h * w, 1176, dtype=bf)
    return CK.qwen(cfg, cnt, t, pin=False)


def test_checkpoint_tensor_set_and_refusals(tmp_path):
    from flash_vstream_b200 import checkpoint as CK
    ck = _ckpt(True)
    assert ck.config["compact_pixels"] is True and "pixels" not in ck.tensors
    assert ck.tensor("pix_codes").dtype == torch.uint8 and ck.tensor("pix_codes").shape == (2, 16 * 1176)
    assert ck.nbytes() < _ckpt(False).nbytes()
    assert "compact_pixels" not in _ckpt(False).config                   # other checkpoints are as before
    ck.save(tmp_path / "c.safetensors")
    back = CK.StreamCheckpoint.load(tmp_path / "c.safetensors", pin=False)
    assert back.config["compact_pixels"] and torch.equal(back.tensor("pix_codes"), ck.tensor("pix_codes"))
    for drop in ("pix_codes", "pixel_table"):
        with pytest.raises(ValueError, match=f"tensor '{drop}' is missing"):
            CK.StreamCheckpoint(CK.QWEN, ck.config, ck.counters, {k: v for k, v in ck.tensors.items() if k != drop})
    with pytest.raises(ValueError, match="'pix_codes' has dtype"):
        CK.StreamCheckpoint(CK.QWEN, ck.config, ck.counters, dict(ck.tensors, pix_codes=ck.tensor("pix_codes").float()))
    with pytest.raises(ValueError, match="'pixel_table' has shape"):
        CK.StreamCheckpoint(CK.QWEN, ck.config, ck.counters, dict(ck.tensors, pixel_table=torch.zeros(256, 3)))
    with pytest.raises(ValueError, match="unexpected tensors"):
        CK.StreamCheckpoint(CK.QWEN, ck.config, ck.counters, dict(ck.tensors, pixels=_ckpt(False).tensor("pixels")))


def test_restore_refusals():
    """refused before anything touches a device"""
    from flash_vstream_b200.qwen.stream_state import QwenStreamState
    fl = _flash()
    table = torch.from_numpy(P.value_table(1 / 255, PI.OPENAI_CLIP_MEAN, PI.OPENAI_CLIP_STD))
    with pytest.raises(NotImplementedError, match="compact_pixels=False"):     # tower-dtype rows -> codes
        QwenStreamState.restore(_ckpt(False), fl, None, "cuda:0", lazy_full_res=True, compact_pixels=True,
                                pixel_table=table)
    with pytest.raises(ValueError, match="pixel_table differs"):                # codes of another table
        QwenStreamState.restore(_ckpt(True), fl, None, "cuda:0", lazy_full_res=True, compact_pixels=True,
                                pixel_table=table + 1)
    with pytest.raises(ValueError, match="compact_pixels=True needs lazy_full_res=True"):
        QwenStreamState.restore(_ckpt(True), fl, None, "cuda:0", compact_pixels=True, pixel_table=table)
    with pytest.raises(NotImplementedError, match="lazy_full_res=True"):       # codes -> eager: today's rule
        QwenStreamState.restore(_ckpt(True), fl, None, "cuda:0")


# ---------------------------------------------------------------------------------------------------------- entry points
def test_code_symbols_exported():
    lib = L.load()
    for name in ("fvs_qwen_pixel_decode", "fvs_qwen_pixel_gather_multi"):
        assert hasattr(lib, name) and name in L.SIGNATURES


@pytest.mark.parametrize("args, msg", [
    ((None, 4, A, L.BF16, A), "null pointer"),
    ((A, 4, None, L.BF16, A), "null pointer"),
    ((A, 4, A, L.BF16, None), "null pointer"),
    ((A, 4, A, L.F32, A), "dtype must be f16 or bf16"),
    ((A, 0, A, L.BF16, A), "rows > 0"),
    ((A + 4, 4, A, L.BF16, A), "aligned"),
    ((A, 4, A, L.F16, A + 8), "aligned"),
])
def test_decode_refusals_launch_nothing(args, msg):
    lib = L.load()
    before = lib.fvs_launch_count()
    assert lib.fvs_qwen_pixel_decode(*args, None) == L.FVS_EINVAL
    assert msg in lib.fvs_last_error().decode()
    assert lib.fvs_launch_count() == before


def _codes_job(**kw):
    a = dict(plan=A, n=3, n_frames=10, base=2, host_chunks=A, chunk_frames=4, frame_elems=4 * 1176, table=A, out=A)
    a.update(kw)
    return L.QwenPixelJob(**a)


@pytest.mark.parametrize("kw, msg", [
    (dict(plan=None), "need a plan, a table, an output"),
    (dict(table=None), "need a plan, a table, an output"),
    (dict(out=None), "need a plan, a table, an output"),
    (dict(n=0), "0 < n <= 65535"),
    (dict(base=10), "0 <= base < n_frames"),
    (dict(host_chunks=None), "chunk table"),
    (dict(chunk_frames=0), "chunk table"),
    (dict(frame_elems=1175 * 4), "not whole rows of 1176 codes"),
    (dict(frame_elems=0), "not whole rows of 1176 codes"),
    (dict(out=A + 8), "misaligned"),
    (dict(plan=A + 4), "misaligned"),
])
def test_pixel_gather_of_codes_refusals_launch_nothing(kw, msg):
    arr = (L.QwenPixelJob * 3)(_codes_job(out=A << 8), _codes_job(**kw), _codes_job(out=A << 9))
    _refused("fvs_qwen_pixel_gather_multi", arr, 3, L.BF16, None, msg=msg)
    assert "fvs_qwen_pixel_gather_multi: job 1: " in L.load().fvs_last_error().decode()


def test_pixel_gather_of_codes_refuses_dtype_and_shared_outputs():
    arr = (L.QwenPixelJob * 2)(_codes_job(), _codes_job(out=A + 2 * 1176))
    _refused("fvs_qwen_pixel_gather_multi", arr, 2, L.F32, None, msg="dtype must be f16 or bf16")
    _refused("fvs_qwen_pixel_gather_multi", arr, 2, L.BF16, None, msg="jobs 0 and 1 share an output")


def test_pixel_gather_refuses_a_mix_of_codes_and_rows():
    """one call gathers tower-dtype rows (no table) or codes (a table in every job), never both"""
    for first, second in ((dict(table=None, frame_elems=4 * 1176), dict()), (dict(), dict(table=None))):
        arr = (L.QwenPixelJob * 2)(_codes_job(out=A << 8, **first), _codes_job(out=A << 9, **second))
        _refused("fvs_qwen_pixel_gather_multi", arr, 2, L.BF16, None, msg="job 1: need a plan, a table, an output")
        assert "code and row jobs do not mix" in L.load().fvs_last_error().decode()


# ---------------------------------------------------------------------------------------------------------- SASS
def _res_usage():
    """{mangled name: (registers, stack bytes, local bytes)} of every kernel in the built library"""
    from flash_vstream_b200 import _build
    _build.build()
    out = subprocess.run([CUOBJDUMP, "-res-usage", str(_build.LIB_PATH)], capture_output=True, text=True).stdout
    res, fn = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", line)
        if m and fn:
            res[fn] = tuple(int(v) for v in m.groups())
        fn = None
    return res


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_kernel_resources():
    res = _res_usage()

    def find(pat):
        hits = [r for k, r in res.items() if re.search(pat, k)]
        assert len(hits) == 1, (pat, hits)
        return hits[0]
    # the existing instantiations keep the registers, stack and local memory they had
    assert find(r"resample_cols_kernelILi0E") == (40, 0, 0)                 # FVS_PRE_CLIP
    assert find(r"resample_cols_kernelILi1E") == (32, 0, 0)                 # FVS_PRE_QWEN
    assert find(r"resample_rows_kernel") == (30, 0, 0)
    assert find(r"dam_gather_multi_kernelILi1E") == (38, 0, 0)              # also the pixel gather's of tower-dtype rows
    assert find(r"dam_gather_multi_kernelILi16E") == (32, 0, 0)
    # the new kernels use no stack or local memory
    new = [r for k, r in res.items() if re.search(r"resample_cols_kernelILi2E|pixel_decode_kernel|pixel_codes_gather_kernel", k)]
    assert len(new) == 1 + 2 + 4
    for reg, stack, local in new:
        assert stack == 0 and local == 0
