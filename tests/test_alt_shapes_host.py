"""The alternate temporal compressors at the shapes and magnitudes a video produces, on the CPU: the oracle against the
goldens recorded from the reference (tests/golden/alt_shapes.npz), the case table itself, the refusals decided on the
host, and the model-level glue (compressor -> weight -> argsort -> key retrieval) on the oracle side."""
from __future__ import annotations

import functools
import os
import random

import numpy as np
import pytest
import torch

from oracle import alternates_oracle as AO
from oracle import fvs_oracle as O
from tests import alt_shapes_inputs as AS
from tests.test_alt_oracle_golden import ulp16

G = np.load(os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "alt_shapes.npz"))
ALT_NAMES = ("drop", "merge", "kmeans", "kdrop", "kmerge", "uni_kmerge", "both_kmerge", "split_kmerge")
OFFLINE_NAMES = ALT_NAMES[:5]


def unflatten(name):
    n_rows, n_mem, mem = G[name + "_n_rows"], G[name + "_n_mem"], G[name + "_mem"]
    steps, r, p = [], 0, 0
    for nr in n_rows:
        st = []
        for _ in range(nr):
            st.append(mem[p:p + n_mem[r]].tolist())
            p += n_mem[r]
            r += 1
        steps.append(st)
    return steps


@functools.lru_cache(maxsize=None)
def run_oracle(name):
    """(feat, sim, steps, kmeans result dict) of the oracle on case `name`, once per process"""
    c = AS.CASES[name]
    x = AS.features(name).numpy()
    res = {}
    if c["fn"] == "kmeans_feature":
        init, refill = AS.kmeans_draws(name)
        feat, sim, steps = AO.kmeans_feature(x, c["T0"], init_idx=init, refill_idx=refill, result=res)
    elif c["fn"] in ("drop_feature", "k_drop_feature"):
        s = AS.sim_in(name)
        args = () if c["fn"] == "k_drop_feature" else (None if s is None else s.numpy(),)
        feat, sim, steps = getattr(AO, c["fn"])(x, c["T0"], *args, coins=AS.coins(name))
    else:
        s = AS.sim_in(name)
        feat, sim, steps = getattr(AO, c["fn"])(x, c["T0"], None if s is None else s.numpy())
    return feat, sim, steps, res


# ------------------------------------------------------------------------------------------------ the oracle vs the reference
@pytest.mark.parametrize("name", AS.GOLDEN)
def test_oracle_matches_reference(name):
    c = AS.CASES[name]
    feat, sim, steps, res = run_oracle(name)
    assert steps == unflatten(name)                                   # every per-step member list, exactly
    got = np.asarray(feat, np.float16).reshape(c["T0"], -1)[:, ::61]
    want = G[name + "_feat"].view(np.float16)
    if c["fn"] in ("drop_feature", "k_drop_feature"):
        assert np.array_equal(got.view(np.int16), want.view(np.int16))       # a pure selection of input frames
    else:                                                                      # averages: one f16 step at most
        nan = np.isnan(want)
        assert np.array_equal(np.isnan(got), nan)
        assert ulp16(got[~nan], want[~nan]) <= 1
    if c["fn"] == "kmeans_feature":
        assert res["refills"] == int(G[name + "_refills"])               # the empty clusters of every iteration
    ws = G[name + "_sim"].view(np.float16)
    if ws.size:
        s = np.asarray(sim, np.float16)
        assert s.shape == ws.shape
        off = ~np.isclose(ws.astype(np.float32), -100.0)
        assert np.abs(s.astype(np.float32) - ws.astype(np.float32))[off].max() <= 2e-3
    else:
        assert sim is None


# ------------------------------------------------------------------------------------------------ the case table
def test_case_table_inputs_and_draws():
    for name, c in AS.CASES.items():
        x = AS.features(name)
        assert tuple(x.shape) == (c["T"], c["PD"] // AS.D, AS.D) and x.dtype == torch.float16
        assert (AS.checksum(x) == G[name + "_chk"]).all(), f"{name}: seeded input drifted"
        if c["fn"] == "kmeans_feature":
            init, refill = AS.kmeans_draws(name)
            assert len(set(init.tolist())) == c["T0"] and init.max() < c["T"] and refill.max() < c["T"]
            assert len(refill) == AS.MAX_ITER * c["T0"]
        else:
            coins = AS.coins(name)
            drops = c["fn"] in ("drop_feature", "k_drop_feature")
            assert len(coins) == (c["T"] - c["T0"] if drops else 0) and set(coins) <= {0, 1}
        assert 2 <= c["T0"] < c["T"]
    # the kernels' limits are all in the table
    shapes = {(c["T0"], c["PD"], c["T"]) for c in AS.CASES.values() if c["fn"] != "kmeans_feature"}
    for T0 in (2, 255, 1023):
        assert {(T0, 1024, T0 + 1), (T0, 1024, T0 + 8)} <= shapes
    assert (2, 1 << 20, 6) in shapes and (25, 65536, 200) in shapes


def test_clip_profile_saturates_the_kmeans_norms():
    """|x|^2 = f16(sum f16(v^2)) is +inf for every row of the clip profile (the kmeans inf regime), finite for the unit one"""
    for name, c in AS.CASES.items():
        if c["PD"] != 16384:
            continue
        X = AS.features(name).numpy().reshape(c["T"], -1)
        frac = []
        AO.cdist16(X, X[:1], stats=frac)
        if c["profile"] == "clip":
            assert frac == [1.0], name
        elif c["profile"] in ("unit", "duplicates"):
            assert frac == [0.0], name


def test_duplicates_profile_has_identical_runs():
    for name, c in AS.CASES.items():
        if c["profile"] != "duplicates":
            continue
        X = AS.features(name).reshape(c["T"], -1)
        same = [torch.equal(X[t], X[t + 1]) for t in range(c["T"] - 1)]
        assert sum(same) >= (c["T"] - 1) // 4, name


def test_kmeans_nan_case_diverges_without_nan_propagation(monkeypatch):
    """A distance that is NaN (-inf + inf) stays NaN under clamp_min and is the smallest for argmin; a clamp that maps it to
    0 instead (fmaxf) ties it with a true 0.  The 0.5 row is at distance 0 from itself and NaN from the +inf centroid, so
    the two clamps assign it differently at the first step, and the case's outputs (refills, centroids) differ too."""
    name = "kmeans_1k_30_nan"
    X = AS.features(name).numpy().reshape(30, -1)
    init, refill = AS.kmeans_draws(name)
    d = AO.cdist16(X, X[init])
    assert np.isnan(d[0, 2]) and d[0, 0] == 0
    assert O.argmin_first_nan(d, axis=1)[0] == 2
    assert O.argmin_first_nan(np.where(np.isnan(d), 0, d), axis=1)[0] == 0
    _, _, _, res = run_oracle(name)
    assert all(res["dist_nan"])
    cdist = AO.cdist16
    monkeypatch.setattr(AO, "cdist16", lambda X, C, stats=None: np.where(np.isnan(d := cdist(X, C, stats)), 0, d))
    other = {}
    C2, _, _ = AO.kmeans_feature(AS.features(name).numpy(), 3, init_idx=init, refill_idx=refill, result=other)
    C1 = run_oracle(name)[0]
    assert other["refills"] != res["refills"] or not np.array_equal(C1.view(np.int16), C2.view(np.int16))


# ------------------------------------------------------------------------------------------------ host-side refusals
def test_argsort_desc_refuses_what_is_not_a_weight_vector():
    from flash_vstream_b200 import ops
    with pytest.raises(ValueError, match="1-D"):
        ops.argsort_desc(torch.zeros(25, 25, dtype=torch.float16))
    with pytest.raises(TypeError):
        ops.argsort_desc(None)


def host_model(name, **cfg):
    """a model whose long and Turing rows are already 4 x 4 (nothing to pool), on the CPU: every refusal below is decided
    before anything reaches a kernel"""
    from flash_vstream_b200.vstream_arch import FlashVStreamB200, NeuralTuringMachine
    base = dict(video_sample_type=name, compress_size=4, compress_long_memory_size=4, compress_Turing_memory_size=4)
    base.update(cfg)
    return FlashVStreamB200(None, NeuralTuringMachine(1024, 32).half(), **base)


def expected_exception(name, T, T0):
    """what the reference's key retrieval raises on T long rows, None when it runs (see test_oracle_glue_vs_reference)"""
    if name in ("kdrop", "kmeans") or T <= T0:
        return TypeError
    return RuntimeError if name.endswith("kmerge") else None


def coin_count(name, T, T0):
    """the coin flips the reference's compressor draws for T long rows: one per incoming frame for drop and kdrop (kdrop
    draws them before its key retrieval raises), none for the others.  A refused kmeans draws nothing in the product (its
    reference draws depend on a Lloyd loop that would have to run) and is never asked for draws here."""
    return T - T0 if name in ("drop", "kdrop") and T > T0 else 0


def advanced(state, n):
    """the `random` state after n more random.randint(0, 1) draws from `state`"""
    r = random.Random()
    r.setstate(state)
    for _ in range(n):
        r.randint(0, 1)
    return r.getstate()


def oracle_compressor(name, T0, coins=()):
    """the alternates_oracle function of `video_sample_type` name with its draws bound: the coin flips of drop / kdrop; for
    kmeans placeholder draws (every configuration that reaches kmeans raises at its weight before they matter)"""
    fn = {"drop": AO.drop_feature, "merge": AO.merge_feature, "kmeans": AO.kmeans_feature,
          "kdrop": AO.k_drop_feature}.get(name, AO.k_merge_feature)
    if name == "kmeans":
        return functools.partial(fn, init_idx=list(range(T0)), refill_idx=[0] * (AS.MAX_ITER * T0))
    return functools.partial(fn, coins=list(coins)) if name in ("drop", "kdrop") else fn


@pytest.fixture
def no_retrieval(monkeypatch):
    from flash_vstream_b200 import ops

    def stub(*a, **k):
        raise AssertionError("key_retrieve reached with a weight the reference cannot sort")
    monkeypatch.setattr(ops, "key_retrieve", stub)


@pytest.mark.parametrize("name", OFFLINE_NAMES)
def test_offline_refusals_on_host(name, no_retrieval):
    feats = torch.randn(30, 16, 1024, generator=torch.Generator().manual_seed(3)).half()
    for T in (30, 26, 12):          # long memory of T - 1 rows against video_long_memory_length 25
        want = expected_exception(name, T - 1, 25)
        if want is None:
            continue                # drop / merge with T - 1 > 25 run: covered on the GPU
        state = random.getstate()
        with pytest.raises(want):
            host_model(name).compress_temporal_features([feats[:T]])
        assert random.getstate() == advanced(state, coin_count(name, T - 1, 25))   # the reference's draws, no more


@pytest.mark.parametrize("name", ALT_NAMES)
def test_streaming_refusals_on_host(name, no_retrieval):
    feats = torch.randn(8, 16, 1024, generator=torch.Generator().manual_seed(4)).half()
    for long_len in (25, 4):
        want = expected_exception(name, 8, long_len)
        if want is None:
            continue
        m = host_model(name, video_long_memory_length=long_len)
        m.consolidate_streaming(feats[:4])                 # the first call only publishes
        first = list(m.video_embedding_memory)
        state = random.getstate()
        with pytest.raises(want):
            m.consolidate_streaming(feats[4:])
        assert all(a is b for a, b in zip(first, m.video_embedding_memory))      # the stream is as it was
        assert m.__dict__["_fvs_buf"]["n"] == 4                                 # the refused chunk is not buffered
        assert random.getstate() == advanced(state, coin_count(name, 8, long_len))


# ------------------------------------------------------------------------------------------------ the oracle's glue
def seeded_coins(name, T, T0, seed):
    """the coins the reference's compressor draws for T long rows after random.seed(seed)"""
    r = random.Random(seed)
    return [r.randint(0, 1) for _ in range(coin_count(name, T, T0))]


@pytest.mark.parametrize("fn", ["drop_feature", "merge_feature", "k_drop_feature", "k_merge_feature"])
def test_oracle_glue_vs_reference(fn):
    """the extended oracle's compress_temporal_features raises what the reference's composition raised, or retrieves the
    key frames it retrieved"""
    name = {"drop_feature": "drop", "merge_feature": "merge", "k_drop_feature": "kdrop", "k_merge_feature": "kmerge"}[fn]
    for T, T0 in AS.GLUE_SHAPES:
        key = f"glue_{fn}_{T}_{T0}"
        x = AS.glue_features(T, T0).numpy()
        cfg = O.StarConfig(cur_len=0, long_len=T0, long_size=4, tur_len=0)
        comp = oracle_compressor(name, T0, seeded_coins(name, T, T0, T))
        exc = str(G[key + "_exc"])
        want = expected_exception(name, T, T0)
        assert exc == ("ok" if want is None else want.__name__), key
        if want is None:
            _, dbg = O.compress_temporal_features(x, cfg, None, compressor=comp)
            assert np.array_equal(dbg["key_idx"], G[key + "_idx"]), key
        else:
            with pytest.raises(want):
                O.compress_temporal_features(x, cfg, None, compressor=comp)


def test_oracle_glue_kmeans_and_streaming():
    x = torch.randn(12, 16, 1024, generator=torch.Generator().manual_seed(6)).half().numpy()
    for T, T0 in ((12, 4), (4, 4)):     # kmeans_feature returns img_similarity (None) as its weight
        with pytest.raises(TypeError):
            O.compress_temporal_features(x[:T], O.StarConfig(cur_len=0, long_len=T0, long_size=4, tur_len=0), None,
                                         compressor=oracle_compressor("kmeans", T0))
    # streaming, long 4 / chunk 4: drop and merge run on every call; the others raise on the second
    for name in ALT_NAMES:
        cfg = O.StarConfig(cur_len=1, cur_size=4, long_len=4, long_size=4, tur_len=25, tur_size=4)
        st = O.StreamState()
        st, _ = O.stream_step(st, x[:4], cfg, None, compressor=oracle_compressor(name, 4))
        want = expected_exception(name, 8, 4)
        if want is None:
            O.stream_step(st, x[4:8], cfg, None, compressor=oracle_compressor(name, 4, seeded_coins(name, 8, 4, 1)))
            assert st.long.shape == (4, 16, 1024) and st.cur.shape == (4, 16, 1024)
        else:
            before = (st.cur, st.long, st.buf)
            with pytest.raises(want):
                O.stream_step(st, x[4:8], cfg, None, compressor=oracle_compressor(name, 4, seeded_coins(name, 8, 4, 1)))
            assert all(a is b for a, b in zip((st.cur, st.long, st.buf), before))
