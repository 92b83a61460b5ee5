"""Stream checkpoints: the state a streaming step reads, on the host, in one `.safetensors` file.

A stream's state is device-resident (DESIGN.md §2), so a stream that has started is tied to its GPU and its process.  A
`StreamCheckpoint` is a copy of exactly what the next step reads — nothing that is rebuilt from it — held in (pinned)
host memory, so the stream can be parked in host memory, moved to another GPU or process, or written to disk, and then
continue bit for bit as if it had never stopped (DESIGN.md §3.12):

  * "llava-star" (ops.StreamBank, multistream.StreamPool, the single-stream LLaVA model):
      prefix  f16 [n_tur + n_long*long_size^2 + n_cur*cur_size^2, D]   the published [Turing | long | key + current]
      long    f16 [n_long, long_size^2, D]                              the long working set between steps
      tur     f16 [n_tur, 1, D]                                         the Turing working set between steps
      frames  f16 [n_frames, cur_size^2, D]                             the whole frame buffer
    counters n_tur, n_long, n_cur, n_frames, step; config = the STAR knobs (D, grid, cur_size, ...).
  * "qwen2vl-flash" (qwen.stream_state.QwenStreamState):
      bank_x [n_frames, h*w, D], bank_small [n_frames, hs*ws, D], bank_merged [n_frames, h*w/4, merger_dim] (when the
      state has one), tem_x [n_tem*hs*ws, D], tem_weights / tem_timestamp [n_tem], spa_positions int64 [n_spa],
      video_embeds [n_spa*h*w/4 + n_tem*hs*ws/4, merger_dim] (with a merger);
    counters n_frames, steps, n_tem, n_spa, fast_steps, redone_steps and the dtypes of the two CSM vectors; config = the
    FlashMemory config, grid, small_grid, dtype, dim, merger_dim.
    A lazy_full_res state adds counters.pix_frames, encoded uint8 [n_frames] and pixels [pix_frames, h*w, 1176] (the
    frames with pixel rows only).  A state without a full-resolution bank also adds counters.bank_frames: bank_x and
    bank_merged then hold its base bank [bank_frames, ...], its mask bytes are 2 for a stored frame, and spa_x
    [n_spa, h*w, D] carries the DAM's rows.  A compact_pixels state (config.compact_pixels true) carries its pixel rows
    as pix_codes uint8 [pix_frames, h*w*1176] and their value table pixel_table float32 [3, 256] in place of pixels.
  * `rng`: the draw source a StreamPool stream owns (draws.DrawSource): torch CPU and CUDA generator states (uint8 tensors
    "rng.cpu" / "rng.cuda") and the `random.Random` state.  Streams that draw from the global generators carry none.

The file holds the tensors under their names and one string metadata entry, "fvs_checkpoint", with the JSON of
{version, family, config, counters, rng: {py, cuda}}.  `load` refuses, with ValueError naming the field, an unknown version
or family, a missing tensor and a tensor whose shape or dtype disagrees with the counters.  This module is the only one
that knows the layout: the stream classes build checkpoints through `llava` / `qwen` and read them through `tensor`.
"""
from __future__ import annotations

import json
from typing import Optional

import torch

FORMAT_VERSION = 1
LLAVA, QWEN = "llava-star", "qwen2vl-flash"
FAMILIES = (LLAVA, QWEN)
STAR_FIELDS = ("D", "grid", "cur_size", "long_size", "long_len", "tur_len", "cur_len", "key_len", "ntm_dim", "ratio")
LLAVA_COUNTERS = ("n_tur", "n_long", "n_cur", "n_frames", "step")
QWEN_COUNTERS = ("n_frames", "steps", "n_tem", "n_spa", "fast_steps", "redone_steps")
_META_KEY = "fvs_checkpoint"

_DTYPES = {"float16": torch.float16, "bfloat16": torch.bfloat16, "float32": torch.float32, "int32": torch.int32,
           "int64": torch.int64, "uint8": torch.uint8}


def dtype_name(dt: torch.dtype) -> str:
    return str(dt).replace("torch.", "")


def _dtype(name: str, field: str) -> torch.dtype:
    if name not in _DTYPES:
        raise ValueError(f"stream checkpoint: {field} has unsupported dtype {name!r}")
    return _DTYPES[name]


def _host(t: torch.Tensor, pin: bool) -> torch.Tensor:
    """a host copy of `t` (pinned when asked); a device source is copied asynchronously on the current stream"""
    out = torch.empty(tuple(t.shape), dtype=t.dtype, pin_memory=pin)
    out.copy_(t, non_blocking=t.is_cuda and pin)
    return out


def _pin_default() -> bool:
    return torch.cuda.is_available()


class StreamCheckpoint:
    """family, version, config (dict), counters (dict), rng (dict or None: {"cpu", "cuda", "py"}), tensors (name -> host
    tensor).  Build one with `llava` / `qwen` or `load`; the constructor checks every tensor against the counters."""

    def __init__(self, family: str, config: dict, counters: dict, tensors: dict, rng: Optional[dict] = None,
                 version: int = FORMAT_VERSION):
        if version != FORMAT_VERSION:
            raise ValueError(f"stream checkpoint: version {version!r} is not supported (this build reads {FORMAT_VERSION})")
        if family not in FAMILIES:
            raise ValueError(f"stream checkpoint: family {family!r} is not one of {FAMILIES}")
        self.family, self.version = family, version
        self.config, self.counters, self.tensors, self.rng = dict(config), dict(counters), dict(tensors), rng
        self._check()

    # ---- layout -----------------------------------------------------------------------------------------------------
    def layout(self) -> dict:
        """name -> (shape, dtype) of every tensor the counters call for"""
        c, n = self.config, self.counters
        if self.family == LLAVA:
            for k in STAR_FIELDS:
                if k not in c:
                    raise ValueError(f"stream checkpoint: config.{k} is missing")
            for k in LLAVA_COUNTERS:
                if k not in n:
                    raise ValueError(f"stream checkpoint: counters.{k} is missing")
            D, a2, b2 = int(c["D"]), int(c["cur_size"]) ** 2, int(c["long_size"]) ** 2
            f16 = torch.float16
            return {"prefix": ((n["n_tur"] + n["n_long"] * b2 + n["n_cur"] * a2, D), f16),
                    "long": ((n["n_long"], b2, D), f16), "tur": ((n["n_tur"], 1, D), f16),
                    "frames": ((n["n_frames"], a2, D), f16)}
        for k in ("flash", "grid", "small_grid", "dtype", "dim", "merger_dim"):
            if k not in c:
                raise ValueError(f"stream checkpoint: config.{k} is missing")
        for k in QWEN_COUNTERS + ("merged", "tem_weights_dtype", "tem_timestamp_dtype"):
            if k not in n:
                raise ValueError(f"stream checkpoint: counters.{k} is missing")
        if n["n_frames"] == 0:
            return {}
        (h, w), (hs, ws) = c["grid"], c["small_grid"]
        D, md, dt = int(c["dim"]), c["merger_dim"], _dtype(c["dtype"], "config.dtype")
        nb = n.get("bank_frames", n["n_frames"])      # frames with stored full-resolution rows (a stream without a bank: its base)
        if not 0 <= nb <= n["n_frames"]:
            raise ValueError(f"stream checkpoint: counters.bank_frames ({nb}) is outside [0, n_frames]")
        out = {"bank_x": ((nb, h * w, D), dt), "bank_small": ((n["n_frames"], hs * ws, D), dt),
               "tem_x": ((n["n_tem"] * hs * ws, D), dt),
               "tem_timestamp": ((n["n_tem"],), _dtype(n["tem_timestamp_dtype"], "counters.tem_timestamp_dtype")),
               "spa_positions": ((n["n_spa"],), torch.int64)}
        if n["tem_weights_dtype"] is not None:       # temporal_method 'sample' keeps no weights
            out["tem_weights"] = ((n["n_tem"],), _dtype(n["tem_weights_dtype"], "counters.tem_weights_dtype"))
        if n["merged"]:
            out["bank_merged"] = ((nb, h * w // 4, md), dt)
        if md is not None:
            out["video_embeds"] = ((n["n_spa"] * h * w // 4 + n["n_tem"] * hs * ws // 4, md), dt)
        if "pix_frames" in n:                         # a lazy_full_res stream: its mask, the pixel rows of its frames not yet encoded
            out["encoded"] = ((n["n_frames"],), torch.uint8)
            if c.get("compact_pixels"):               # 8-bit codes and the table they decode through
                out["pix_codes"] = ((n["pix_frames"], h * w * 3 * 2 * 14 * 14), torch.uint8)
                out["pixel_table"] = ((3, 256), torch.float32)
            else:
                out["pixels"] = ((n["pix_frames"], h * w, 3 * 2 * 14 * 14), dt)
        if "bank_frames" in n:                        # no full-resolution bank: the DAM's rows, which no bank can rebuild
            out["spa_x"] = ((n["n_spa"], h * w, D), dt)
        return out

    def _check(self):
        want = self.layout()
        for name, (shape, dt) in want.items():
            t = self.tensors.get(name)
            if t is None:
                raise ValueError(f"stream checkpoint: tensor {name!r} is missing")
            if tuple(t.shape) != tuple(int(v) for v in shape):
                raise ValueError(f"stream checkpoint: tensor {name!r} has shape {tuple(t.shape)}, the counters call for "
                                 f"{tuple(shape)}")
            if t.dtype != dt:
                raise ValueError(f"stream checkpoint: tensor {name!r} has dtype {t.dtype}, expected {dt}")
        extra = set(self.tensors) - set(want)
        if extra:
            raise ValueError(f"stream checkpoint: unexpected tensors {sorted(extra)}")
        if self.rng is not None:
            for k in ("cpu", "py"):
                if self.rng.get(k) is None:
                    raise ValueError(f"stream checkpoint: rng.{k} is missing")
            for k in ("cpu", "cuda"):
                if self.rng.get(k) is not None and self.rng[k].dtype != torch.uint8:
                    raise ValueError(f"stream checkpoint: rng.{k} must be a uint8 tensor")

    def tensor(self, name: str) -> torch.Tensor:
        return self.tensors[name]

    def nbytes(self) -> int:
        return sum(t.numel() * t.element_size() for t in self.tensors.values())

    # ---- file -------------------------------------------------------------------------------------------------------
    def save(self, path) -> None:
        """one .safetensors file: the tensors, the torch RNG states as uint8 tensors "rng.cpu" / "rng.cuda", and the rest
        as JSON in the string metadata"""
        from safetensors.torch import save_file
        tensors = {k: v.contiguous() for k, v in self.tensors.items()}
        rng = None
        if self.rng is not None:
            tensors["rng.cpu"] = self.rng["cpu"].contiguous()
            if self.rng.get("cuda") is not None:
                tensors["rng.cuda"] = self.rng["cuda"].contiguous()
            v, internal, gauss = self.rng["py"]
            rng = {"py": [v, list(internal), gauss], "cuda": self.rng.get("cuda") is not None}
        meta = {"version": self.version, "family": self.family, "config": self.config, "counters": self.counters, "rng": rng}
        save_file(tensors, str(path), metadata={_META_KEY: json.dumps(meta)})

    @classmethod
    def load(cls, path, *, pin: Optional[bool] = None) -> "StreamCheckpoint":
        from safetensors import safe_open
        with safe_open(str(path), framework="pt") as f:
            md = f.metadata() or {}
            if _META_KEY not in md:
                raise ValueError(f"stream checkpoint: {path} has no {_META_KEY!r} metadata")
            meta = json.loads(md[_META_KEY])
            raw = {k: f.get_tensor(k) for k in f.keys()}
        for k in ("version", "family", "config", "counters"):
            if k not in meta:
                raise ValueError(f"stream checkpoint: metadata field {k!r} is missing")
        if meta["version"] != FORMAT_VERSION:
            raise ValueError(f"stream checkpoint: version {meta['version']!r} is not supported (this build reads "
                             f"{FORMAT_VERSION})")
        pin = _pin_default() if pin is None else pin
        rng = None
        if meta.get("rng") is not None:
            if "rng.cpu" not in raw:
                raise ValueError("stream checkpoint: tensor 'rng.cpu' is missing")
            v, internal, gauss = meta["rng"]["py"]
            rng = {"cpu": raw.pop("rng.cpu"), "cuda": raw.pop("rng.cuda", None), "py": (v, tuple(internal), gauss)}
            if meta["rng"].get("cuda") and rng["cuda"] is None:
                raise ValueError("stream checkpoint: tensor 'rng.cuda' is missing")
        tensors = {k: (v.pin_memory() if pin else v) for k, v in raw.items()}
        return cls(meta["family"], meta["config"], meta["counters"], tensors, rng=rng, version=meta["version"])


# ---------------------------------------------------------------------------------------------------- builders
def llava(config: dict, counters: dict, prefix, long, tur, frames, rng: Optional[dict] = None,
          pin: Optional[bool] = None, owned: Optional[dict] = None) -> StreamCheckpoint:
    """A "llava-star" checkpoint from a bank's views (device or host; device sources are copied asynchronously on the
    current stream — synchronise it before reading the tensors).  `owned`: host tensors made for this checkpoint alone,
    taken without another copy (their views above are then None)."""
    pin = _pin_default() if pin is None else pin
    cfg = {k: config[k] for k in STAR_FIELDS}
    cnt = {k: int(counters[k]) for k in LLAVA_COUNTERS}
    views = {"prefix": prefix, "long": long, "tur": tur, "frames": frames}
    tensors = {k: _host(v, pin) for k, v in views.items() if v is not None}
    return StreamCheckpoint(LLAVA, cfg, cnt, {**tensors, **(owned or {})}, rng=rng)


def qwen(config: dict, counters: dict, tensors: dict, pin: Optional[bool] = None,
         owned: Optional[dict] = None) -> StreamCheckpoint:
    """A "qwen2vl-flash" checkpoint; `tensors` as listed in the module docstring (device views are copied asynchronously
    on the current stream).  `owned`: host tensors made for this checkpoint alone, taken without another copy."""
    pin = _pin_default() if pin is None else pin
    return StreamCheckpoint(QWEN, config, counters, {**{k: _host(v, pin) for k, v in tensors.items()}, **(owned or {})})


def star_config(cfg) -> dict:
    """the STAR knobs of an L.StarConfig (or of a dict, with `ratio` rounded to float32 like the library's struct) as
    the dict a checkpoint stores"""
    if isinstance(cfg, dict):
        out = {k: cfg[k] for k in STAR_FIELDS}
        out["ratio"] = float(torch.tensor(float(cfg["ratio"]), dtype=torch.float32))
        return out
    return {k: getattr(cfg, k) for k in STAR_FIELDS}


def check_star(ckpt: StreamCheckpoint, cfg, who: str) -> None:
    """ValueError naming the first STAR knob in which `ckpt` differs from `cfg` (an L.StarConfig or a dict)"""
    if ckpt.family != LLAVA:
        raise ValueError(f"{who}: a {ckpt.family!r} checkpoint is not a LLaVA stream's")
    mine = star_config(cfg)
    for k in STAR_FIELDS:
        if ckpt.config[k] != mine[k]:
            raise ValueError(f"{who}: config.{k} of the checkpoint ({ckpt.config[k]}) differs from this one's ({mine[k]})")


def rng_state(source) -> dict:
    """the generator states of an owned draws.DrawSource (settle it first)"""
    return {"cpu": source.cpu.clone(), "cuda": None if source.cuda is None else source.cuda.clone(),
            "py": source.py.getstate()}
