"""CPU tests of stream checkpoints: fvs_bank_restore refuses a bad state with FVS_EINVAL before any CUDA call (there is no
GPU here, so a CUDA call would fail differently) and leaves the bank's counters alone; the `.safetensors` format of
checkpoint.StreamCheckpoint round-trips host tensors, generator states and metadata, and refuses unknown versions and
families, missing tensors, shapes and dtypes that disagree with the counters, and configs that differ."""
import ctypes as C
import json
import random

import pytest
import torch

from flash_vstream_b200 import _lib as L
from flash_vstream_b200 import checkpoint as CK

CFG = L.StarConfig(1024, 24, 8, 4, 25, 25, 1, 3, 32, 0.2)


def fake_bank(*, chunk_cap=1, frames_cap=256):
    """a bank struct with dummy (never dereferenced) device pointers, holding some other stream's counters"""
    base = 1 << 32
    return L.Bank(base + 0x1000, base + 0x2000, base + 0x3000, base + 0x4000, base + 0x5000, frames_cap, chunk_cap,
                  7, 8, 2, 9, 9)


def counters(b):
    return (b.n_long, b.n_tur, b.n_cur, b.n_frames, b.step)


SRC = (0xA000, 0xB000, 0xC000, 0xD000)
GOOD = dict(n_tur=25, n_long=25, n_cur=4, n_frames=40, step=40)


def restore(bank, cfg=CFG, srcs=SRC, **kw):
    a = {**GOOD, **kw}
    return L.load().fvs_bank_restore(C.byref(cfg) if cfg is not None else None, C.byref(bank) if bank is not None else None,
                                     a["n_tur"], a["n_long"], a["n_cur"], a["n_frames"], a["step"], *srcs, None)


@pytest.mark.parametrize("case, message", [
    ("config", b"D (100)"), ("null_bank", b"null bank"), ("buffers", b"buffers missing"),
    ("n_long", b"n_long 26"), ("n_tur", b"n_tur 26"), ("n_cur", b"n_cur 5"), ("prefix_rows", b"prefix of"),
    ("frames_cap", b"frames_cap"), ("step0_frames", b"step 0 with 3"), ("frames0_step", b"step 4 with 0"),
    ("step0_rows", b"no memory rows"), ("prefix_src", b"prefix_src is null"), ("long_src", b"long_src is null"),
    ("tur_src", b"tur_src is null"), ("frames_src", b"frames_src is null"),
])
def test_bad_restore_is_refused_before_any_cuda_call(case, message):
    lib = L.load()
    bank = fake_bank()
    before = counters(bank)
    cfg, srcs, kw = CFG, SRC, {}
    target = bank
    if case == "config":
        cfg = L.StarConfig(100, 24, 8, 4, 25, 25, 1, 3, 32, 0.2)
    elif case == "null_bank":
        target = None
    elif case == "buffers":
        bank.header = None
    elif case == "n_long":
        kw = dict(n_long=26)                       # max(long_len, chunk_cap) = 25
    elif case == "n_tur":
        kw = dict(n_tur=26)
    elif case == "n_cur":
        kw = dict(n_cur=5)                         # key_len + cur_len = 4
    elif case == "prefix_rows":                    # cur_len 2 admits 5 key + current frames, a 1-frame bank holds 4
        cfg = L.StarConfig(1024, 24, 8, 4, 25, 25, 2, 3, 32, 0.2)
        kw = dict(n_cur=5)
    elif case == "frames_cap":
        kw = dict(n_frames=257, step=257)
    elif case == "step0_frames":
        kw = dict(n_tur=0, n_long=0, n_cur=0, n_frames=3, step=0)
    elif case == "frames0_step":
        kw = dict(n_tur=0, n_long=0, n_cur=0, n_frames=0, step=4)
    elif case == "step0_rows":
        kw = dict(n_tur=1, n_long=0, n_cur=0, n_frames=0, step=0)
    else:
        i = ("prefix_src", "long_src", "tur_src", "frames_src").index(case)
        srcs = tuple(None if j == i else s for j, s in enumerate(SRC))
    header_before = bank.header
    n0 = lib.fvs_launch_count()
    rc = restore(target, cfg, srcs, **kw)
    assert rc == L.FVS_EINVAL, (rc, lib.fvs_last_error())
    assert message in lib.fvs_last_error(), lib.fvs_last_error()
    assert counters(bank) == before and bank.header == header_before
    assert lib.fvs_launch_count() == n0


# ------------------------------------------------------------------------------------------------ the file format
def star_dict(cfg=CFG):
    return {k: getattr(cfg, k) for k in CK.STAR_FIELDS}


def llava_ckpt(n_tur=3, n_long=3, n_cur=2, n_frames=3, step=1, D=256, rng=True):
    g = torch.Generator().manual_seed(n_frames)
    cfg = {**star_dict(), "D": D}
    rows = n_tur + n_long * 16 + n_cur * 64
    f = lambda *s: torch.randn(*s, generator=g).half()
    r = None
    if rng:
        py = random.Random(5)
        py.random()
        r = {"cpu": torch.Generator().manual_seed(3).get_state(), "cuda": torch.arange(16, dtype=torch.uint8),
             "py": py.getstate()}
    return CK.llava(cfg, dict(n_tur=n_tur, n_long=n_long, n_cur=n_cur, n_frames=n_frames, step=step), f(rows, D),
                    f(n_long, 16, D), f(n_tur, 1, D), f(n_frames, 64, D), rng=r, pin=False)


def qwen_ckpt(n_frames=4, n_tem=2, n_spa=3, merged=True, dim=64, md=96):
    h, w, hs, ws = 8, 12, 4, 6
    dt = torch.bfloat16
    t = lambda *s: torch.randn(*s).to(dt)
    cfg = {"flash": {"flash_memory_temporal_length": 4, "flash_memory_spatial_length": 6,
                     "flash_memory_temporal_method": "kmeans_ordered"},
           "grid": [h, w], "small_grid": [hs, ws], "dtype": "bfloat16", "dim": dim, "merger_dim": md}
    cnt = {"n_frames": n_frames, "steps": 2, "n_tem": n_tem, "n_spa": n_spa, "fast_steps": 1, "redone_steps": 0,
           "merged": int(merged), "tem_weights_dtype": "float32", "tem_timestamp_dtype": "float32"}
    tensors = {"bank_x": t(n_frames, h * w, dim), "bank_small": t(n_frames, hs * ws, dim), "tem_x": t(n_tem * hs * ws, dim),
               "tem_weights": torch.rand(n_tem), "tem_timestamp": torch.rand(n_tem),
               "spa_positions": torch.arange(n_spa), "video_embeds": t(n_spa * h * w // 4 + n_tem * hs * ws // 4, md)}
    if merged:
        tensors["bank_merged"] = t(n_frames, h * w // 4, md)
    return CK.qwen(cfg, cnt, tensors, pin=False)


def same(a, b):
    assert a.family == b.family and a.version == b.version and a.config == b.config and a.counters == b.counters
    assert set(a.tensors) == set(b.tensors)
    for k in a.tensors:
        assert a.tensors[k].dtype == b.tensors[k].dtype and torch.equal(a.tensors[k], b.tensors[k]), k
    assert (a.rng is None) == (b.rng is None)
    if a.rng is not None:
        assert torch.equal(a.rng["cpu"], b.rng["cpu"]) and torch.equal(a.rng["cuda"], b.rng["cuda"])
        assert a.rng["py"] == b.rng["py"]
        r1, r2 = random.Random(), random.Random()
        r1.setstate(a.rng["py"])
        r2.setstate(b.rng["py"])
        assert [r1.random() for _ in range(5)] == [r2.random() for _ in range(5)]


@pytest.mark.parametrize("make", [llava_ckpt, lambda: llava_ckpt(rng=False), lambda: llava_ckpt(0, 0, 0, 0, 0),
                                  qwen_ckpt, lambda: qwen_ckpt(merged=False), lambda: qwen_ckpt(n_spa=0)])
def test_round_trip(tmp_path, make):
    ck = make()
    p = tmp_path / "s.safetensors"
    ck.save(p)
    back = CK.StreamCheckpoint.load(p, pin=False)
    same(ck, back)
    from safetensors import safe_open
    with safe_open(str(p), framework="pt") as f:
        meta = json.loads(f.metadata()["fvs_checkpoint"])
        assert meta["version"] == CK.FORMAT_VERSION and meta["family"] == ck.family
        if ck.rng is not None:
            assert f.get_tensor("rng.cpu").dtype == torch.uint8


def rewrite(src, dst, *, meta=None, drop=None, replace=None):
    """copy a checkpoint file with its metadata edited by `meta(dict)`, a tensor dropped or replaced"""
    from safetensors import safe_open
    from safetensors.torch import save_file
    with safe_open(str(src), framework="pt") as f:
        md = json.loads(f.metadata()["fvs_checkpoint"])
        tensors = {k: f.get_tensor(k) for k in f.keys()}
    if meta:
        meta(md)
    if drop:
        tensors.pop(drop)
    if replace:
        tensors.update(replace)
    save_file(tensors, str(dst), metadata={"fvs_checkpoint": json.dumps(md)})


@pytest.mark.parametrize("edit, message", [
    (dict(meta=lambda m: m.update(version=2)), "version 2"),
    (dict(meta=lambda m: m.update(family="llava-next")), "family 'llava-next'"),
    (dict(meta=lambda m: m.pop("counters")), "'counters'"),
    (dict(meta=lambda m: m["config"].pop("long_size")), "config.long_size"),
    (dict(meta=lambda m: m["counters"].update(n_frames=4)), "tensor 'frames' has shape"),
    (dict(meta=lambda m: m["counters"].update(n_long=2)), "tensor 'prefix' has shape"),
    (dict(drop="tur"), "tensor 'tur' is missing"),
    (dict(drop="rng.cpu"), "'rng.cpu' is missing"),
    (dict(replace={"long": torch.zeros(3, 16, 256, dtype=torch.float32)}), "tensor 'long' has dtype"),
    (dict(replace={"extra": torch.zeros(1)}), "unexpected tensors"),
])
def test_load_refuses(tmp_path, edit, message):
    p, q = tmp_path / "a.safetensors", tmp_path / "b.safetensors"
    llava_ckpt().save(p)
    rewrite(p, q, **edit)
    with pytest.raises(ValueError, match=message.replace("(", r"\(").replace(")", r"\)")):
        CK.StreamCheckpoint.load(q, pin=False)


def test_qwen_load_refuses(tmp_path):
    p, q = tmp_path / "a.safetensors", tmp_path / "b.safetensors"
    qwen_ckpt().save(p)
    rewrite(p, q, meta=lambda m: m["counters"].update(n_spa=2))
    with pytest.raises(ValueError, match="'spa_positions' has shape"):
        CK.StreamCheckpoint.load(q, pin=False)
    rewrite(p, q, drop="bank_merged")
    with pytest.raises(ValueError, match="'bank_merged' is missing"):
        CK.StreamCheckpoint.load(q, pin=False)
    rewrite(p, q, meta=lambda m: m["config"].update(dtype="float8"))
    with pytest.raises(ValueError, match="config.dtype"):
        CK.StreamCheckpoint.load(q, pin=False)


def test_config_mismatch_is_named():
    ck = llava_ckpt(D=1024)
    CK.check_star(ck, CFG, "t")                                     # the float32 ratio compares equal
    CK.check_star(ck, {**star_dict(), "ratio": 0.2}, "t")           # a dict's ratio is rounded like the struct's
    with pytest.raises(ValueError, match="config.long_len"):
        CK.check_star(ck, L.StarConfig(1024, 24, 8, 4, 24, 25, 1, 3, 32, 0.2), "t")
    with pytest.raises(ValueError, match="config.ratio"):
        CK.check_star(ck, {**star_dict(), "ratio": 0.3}, "t")
    with pytest.raises(ValueError, match="not a LLaVA"):
        CK.check_star(qwen_ckpt(), CFG, "t")
