"""Seeded cases for the alternate temporal compressors at the shapes and magnitudes a video produces, shared by
tests/golden/make_golden_alt_shapes.py (REFERENCE side), tests/test_alt_shapes_host.py and tests/test_alt_shapes_gpu.py.

Magnitude profiles of the features:
  unit        piecewise-stationary scenes plus noise, RMS ~ 1;
  clip        the unit profile x 2.5 (RMS 2.5) with three channels of every patch in the hundreds, like CLIP layer -2
              outliers.  A pooled long row of 16 x 1024 then has f16(sum f16(v^2)) = +inf, so kmeans_feature's cdist
              runs with every |x|^2 saturated (alternates_oracle.cdist16);
  duplicates  runs of bit-identical frames (a static scene): exact similarity ties that the argmaxes resolve to the first
              index, across warps in the all-pairs variants.
Every draw is explicit and comes from the case seed: the coin flips of the drop variants and kmeans' init_idx /
refill_idx, as the reference would draw them after `random.seed(seed); torch.manual_seed(seed)` (randint per step,
torch.randperm(T) on the CPU).
"""
from __future__ import annotations

import random

import numpy as np
import torch

from tests.golden_inputs import _gen, checksum  # noqa: F401

MAX_ITER = 10
D = 1024                      # channels of a CLIP ViT-L row; P = PD / 1024 patches
OUTLIER_DIMS = (17, 300, 777)


def _real():
    """T0 = 25 (video_long_memory_length) on long rows of 16 x 1024 (compress_long_memory_size 4) and 64 x 1024 (8)"""
    out = {}
    for fn, short in (("drop_feature", "drop"), ("merge_feature", "merge"), ("k_drop_feature", "kdrop"),
                      ("k_merge_feature", "kmerge")):
        for i, (PD, T, prof) in enumerate(((16384, 26, "unit"), (16384, 33, "clip"), (16384, 200, "duplicates"),
                                           (65536, 33, "duplicates"), (65536, 200, "clip"))):
            out[f"{short}_{PD // 1024}k_{T}_{prof}"] = dict(fn=fn, T=T, T0=25, PD=PD, seed=1000 + 10 * len(out) + i,
                                                            profile=prof)
    for fn, short in (("drop_feature", "drop"), ("merge_feature", "merge"), ("k_drop_feature", "kdrop")):
        out[f"{short}_16k_1000_unit"] = dict(fn=fn, T=1000, T0=25, PD=16384, seed=1500 + len(out), profile="unit")
    out["drop_16k_33_simin"] = dict(fn="drop_feature", T=33, T0=25, PD=16384, seed=1601, profile="unit", sim_in=True)
    out["merge_16k_33_simin"] = dict(fn="merge_feature", T=33, T0=25, PD=16384, seed=1602, profile="duplicates",
                                     sim_in=True)
    return out


def _kmeans():
    return {
        "kmeans_16k_60_unit": dict(fn="kmeans_feature", T=60, T0=25, PD=16384, seed=1701, profile="unit"),
        "kmeans_16k_120_duplicates": dict(fn="kmeans_feature", T=120, T0=25, PD=16384, seed=1702, profile="duplicates"),
        "kmeans_16k_200_clip": dict(fn="kmeans_feature", T=200, T0=25, PD=16384, seed=1703, profile="clip"),
        "kmeans_16k_500_unit": dict(fn="kmeans_feature", T=500, T0=25, PD=16384, seed=1704, profile="unit"),
        # a row holding +inf: (-2x).c = -inf against |x|^2 = inf is NaN, which torch.cdist's matmul form keeps
        # (clamp_min).  T = 30 > 25 selects that form, as every real k-means does (the direct form, for at most 25 rows on
        # both sides, gives inf there instead).
        "kmeans_1k_30_nan": dict(fn="kmeans_feature", T=30, T0=3, PD=1024, seed=1880, profile="nan"),
    }


def _limits():
    """T0 = 2 and 1023 (the kernels' range; 255 in between) on one 1024-slice, T = T0 + 1 (one step) and T0 + 8;
    PD = 2^20 (the 1024 slice partials of SeqShared::scratch)"""
    out = {}
    profs = ("unit", "duplicates", "clip")
    for fn, short in (("drop_feature", "drop"), ("merge_feature", "merge"), ("k_drop_feature", "kdrop"),
                      ("k_merge_feature", "kmerge")):
        for T0 in (2, 255, 1023):
            for dT in (1, 8):
                prof = profs[len(out) % 3]
                out[f"{short}_t0{T0}_{T0 + dT}_{prof}"] = dict(fn=fn, T=T0 + dT, T0=T0, PD=1024, seed=2000 + len(out),
                                                              profile=prof)
        out[f"{short}_1m_6_unit"] = dict(fn=fn, T=6, T0=2, PD=1 << 20, seed=2100 + len(out), profile="unit")
    return out


CASES = {**_real(), **_kmeans(), **_limits()}

# moderate cases recorded from the reference (tests/golden/alt_shapes.npz): the clip and duplicates profiles, T0 = 2 and
# every k-means case up to T = 200 (the inf regime and the NaN case among them), at PD <= 16384.  Not
# drop_16k_200_duplicates: its argmaxes fall between the self-similarities of different static runs, 1.0 or 0.9995
# depending on the fp32 summation order (ATen's or the canonical one), the one-ulp near-tie alternates_oracle documents.
GOLDEN = [n for n, c in CASES.items() if c["PD"] <= 16384 and c["T"] <= 200 and n != "drop_16k_200_duplicates"
          and (c["profile"] in ("clip", "duplicates") or c["T0"] == 2 or c["fn"] == "kmeans_feature")]


# model-level glue: (long-memory rows T, video_long_memory_length T0) of the reference's key retrieval records
GLUE_SHAPES = ((8, 4), (4, 4), (3, 2), (30, 25))


def glue_features(T, T0):
    return torch.randn(T, 16, D, generator=_gen(T + 100 * T0)).half()


def _unit(T, P, g):
    scenes = torch.randn(8, P, D, generator=g)
    which = torch.sort(torch.randint(0, 8, (T,), generator=g)).values
    return 0.8 * scenes[which] + 0.6 * torch.randn(T, P, D, generator=g)


def features(name: str) -> torch.Tensor:
    """[T, P, D] float16 of case `name`"""
    c = CASES[name]
    T, P = c["T"], c["PD"] // D
    g = _gen(c["seed"])
    prof = c["profile"]
    if prof == "nan":
        x = torch.randn(T, P, D, generator=g)
        x[0] = 0.5                  # |x|^2 = 256 exactly: distance 0 to itself, ahead of the NaN of the +inf centroid
        x[2, 0, 5] = float("inf")
        return x.half()
    x = _unit(T, P, g)
    if prof == "clip":
        x = 2.5 * x
        for d in OUTLIER_DIMS:      # |v| in [100, 400), sign per frame and patch
            sign = torch.where(torch.rand(T, P, generator=g) < 0.5, -1.0, 1.0)
            x[:, :, d] = sign * (100.0 + 300.0 * torch.rand(T, P, generator=g))
    elif prof == "duplicates":
        t = 0
        while t < T:
            run = int(torch.randint(1, 7, (1,), generator=g))
            x[t:t + run] = x[t]
            t += run
    return x.half()


def coins(name: str) -> list:
    """random.randint(0, 1) per incoming frame of a drop variant (compress_functions.py:38, :194); the others draw none"""
    c = CASES[name]
    if c["fn"] not in ("drop_feature", "k_drop_feature"):
        return []
    r = random.Random(c["seed"])
    return [r.randint(0, 1) for _ in range(max(0, c["T"] - c["T0"]))]


def kmeans_draws(name: str):
    """(init_idx, refill_idx): torch.randperm(T)[:T0] on the CPU generator (:93) and MAX_ITER * T0 random.randint(0, T-1)
    refill candidates (:107), int32"""
    c = CASES[name]
    T, T0 = c["T"], c["T0"]
    if c["profile"] == "nan":
        init = np.array([0, 1, 2], np.int32)                   # the 0.5 row, a plain row, the +inf row
    else:
        init = torch.randperm(T, generator=_gen(c["seed"]))[:T0].numpy().astype(np.int32)
    r = random.Random(c["seed"])
    return init, np.array([r.randint(0, T - 1) for _ in range(MAX_ITER * T0)], np.int32)


def sim_in(name: str):
    """the img_similarity given to drop / merge, or None: values in [-1, 1] on a 1/64 grid, so some of them tie"""
    c = CASES[name]
    if not c.get("sim_in"):
        return None
    v = torch.randint(-64, 65, (c["T0"] + 3,), generator=_gen(c["seed"] + 7)) / 64.0
    return v.half()
