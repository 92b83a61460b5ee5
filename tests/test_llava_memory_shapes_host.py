"""The LLaVA streaming memory at every STAR configuration the fused step admits, up to its limits (CPU half).

consolidate_kernel (csrc/stream_kernels.cu) runs the whole LLaVA memory update, out of the per-unit functions of
csrc/mem_device.cuh.  Before this file every oracle comparison used the default 681-token config; the op-by-op path,
the other check, calls the same units, so a wrong unit is wrong in both.  This file holds the case table that
test_llava_memory_shapes_gpu.py runs on the GPU: every admitted compress_size at grid 24, the 256-token bank of bench.py,
the kernel's declared limits (kMaxT 192 working-set rows, kMaxK 64 clusters, kMaxS 32 slices, kMaxKey 8 key frames, 64
Turing rows of width 64), current-memory lengths 0 / 3 / 5, one-row Turing memories that fold 32 chunks a step, duplicate
frames that empty clusters, and features large enough to saturate the f16 distances.  It pins each case's seeded inputs
by checksum and proves, from the config arithmetic of prepare_job and from the oracle's trace, that each case reaches
what it names — so an RNG or torch change that moves a case off its branch fails here, on any machine."""
import functools

import numpy as np
import pytest
import torch

from oracle import fvs_oracle as O
from tests import golden_inputs as GI
from tests import llava_abstract as LA

GRID = 24
RATIO = 0.2

# name -> config (D, cur_size a, long_size b, long_len, tur_len, cur_len, key_len, ntm_dim), clip sizes, data, seed,
# the ways the GPU file runs it ("bank", "pool", "op", "capped"; "waves": the pool also with max_blocks forcing several
# cooperative launches), whether the CPU half runs the oracle ("light"), and the branches the case must reach.
# data: "scene" (randn scenes + 0.15 noise), "dup" (4 distinct frames, repeated exactly), "sat" (scenes x 16: every f16
# k-means and key distance between different frames is inf), "overflow" (20000 + 3000 x scenes: distances saturate as in
# "sat", so every row that is not a seed joins cluster 0 by first index, and that cluster's f16 sum overflows to inf)
CASES = {
    "default_d1024_clip32": dict(D=1024, a=8, b=4, long_len=25, tur_len=25, cur_len=1, key_len=3, ntm_dim=32,
                                 chunks=[32, 32, 32], data="scene", seed=9101, ways=("bank", "pool", "op", "capped"),
                                 light=True, branches=("first_clip_over_bank", "T57", "T64", "ragged7")),
    "bank256_d1024": dict(D=1024, a=8, b=4, long_len=0, tur_len=64, cur_len=3, key_len=3, ntm_dim=32,
                          chunks=[40, 40, 40], data="scene", seed=9102, ways=("bank", "pool", "op", "capped"), light=True,
                          branches=("no_long", "chunk_over_32")),
    "limits_d2048": dict(D=2048, a=8, b=4, long_len=64, tur_len=64, cur_len=1, key_len=8, ntm_dim=64,
                         chunks=[96, 96], data="scene", seed=9103, ways=("bank", "pool", "waves"), light=False,
                         branches=("T192", "K64", "S32", "key8", "tur64_h64", "chunk_over_32")),
    "a2_b1_d1024": dict(D=1024, a=2, b=1, long_len=25, tur_len=25, cur_len=1, key_len=3, ntm_dim=32,
                        chunks=[1, 1, 8, 8, 8, 4], data="scene", seed=9104, ways=("bank", "op"), light=True,
                        branches=("S1", "kl_warmup", "kmeans")),
    "a3_b1_d1024": dict(D=1024, a=3, b=1, long_len=25, tur_len=25, cur_len=1, key_len=3, ntm_dim=32,
                        chunks=[1, 1, 8, 8, 8, 4], data="scene", seed=9105, ways=("bank", "pool", "op"), light=True,
                        branches=("S1", "kl_warmup", "kmeans")),
    "a4_b2_d256": dict(D=256, a=4, b=2, long_len=25, tur_len=25, cur_len=1, key_len=3, ntm_dim=32,
                       chunks=[1, 1, 8, 8, 8, 4], data="scene", seed=9106, ways=("bank", "op"), light=True,
                       branches=("S1", "kl_warmup", "kmeans")),
    "a4_b1_d1024": dict(D=1024, a=4, b=1, long_len=25, tur_len=25, cur_len=1, key_len=3, ntm_dim=32,
                        chunks=[1, 1, 8, 8, 8, 4], data="scene", seed=9107, ways=("bank", "op"), light=True,
                        branches=("S1", "kl_warmup", "kmeans")),
    "a6_b3_d1024": dict(D=1024, a=6, b=3, long_len=25, tur_len=25, cur_len=1, key_len=3, ntm_dim=32,
                        chunks=[1, 1, 8, 8, 8, 4], data="scene", seed=9108, ways=("bank", "op"), light=True,
                        branches=("S9", "kl_warmup", "kmeans")),
    "a6_b2_d256": dict(D=256, a=6, b=2, long_len=25, tur_len=25, cur_len=1, key_len=3, ntm_dim=32,
                       chunks=[1, 1, 8, 8, 8, 4], data="scene", seed=9109, ways=("bank", "op"), light=True,
                       branches=("S1", "kl_warmup", "kmeans")),
    "a8_b2_d1024": dict(D=1024, a=8, b=2, long_len=25, tur_len=25, cur_len=1, key_len=3, ntm_dim=32,
                        chunks=[1, 1, 8, 8, 8, 4], data="scene", seed=9110, ways=("bank", "op"), light=True,
                        branches=("kl_warmup", "kmeans")),
    "cur0_d256": dict(D=256, a=8, b=4, long_len=25, tur_len=25, cur_len=0, key_len=3, ntm_dim=32,
                      chunks=[1, 4, 8, 8, 8, 3], data="scene", seed=9111, ways=("bank", "op"), light=True,
                      branches=("cur_none", "kmeans")),
    "cur3_single_d256": dict(D=256, a=8, b=4, long_len=25, tur_len=25, cur_len=3, key_len=3, ntm_dim=32,
                             chunks=[1] * 30, data="scene", seed=9112, ways=("bank", "op", "capped"), light=True,
                             branches=("cur_all_of_clip", "kmeans")),
    "cur5_d256": dict(D=256, a=8, b=4, long_len=25, tur_len=25, cur_len=5, key_len=3, ntm_dim=32,
                      chunks=[4, 8, 3, 8, 8, 8], data="scene", seed=9113, ways=("bank", "pool", "op", "capped"),
                      light=True, branches=("cur_all_of_clip", "cur_clip_end", "kmeans")),
    "tur1_h1_d256": dict(D=256, a=8, b=4, long_len=25, tur_len=1, cur_len=1, key_len=3, ntm_dim=1,
                         chunks=[32, 32, 32], data="scene", seed=9114, ways=("bank", "op", "capped"), light=True,
                         branches=("many_chunks", "mbuf_both")),
    "dup_d1024": dict(D=1024, a=8, b=4, long_len=25, tur_len=25, cur_len=1, key_len=3, ntm_dim=32,
                      chunks=[32, 32, 32], data="dup", seed=9115, ways=("bank", "op"), light=True,
                      branches=("refill2", "kmeans")),
    "sat_d1024": dict(D=1024, a=8, b=4, long_len=25, tur_len=25, cur_len=1, key_len=3, ntm_dim=32,
                      chunks=[16, 16, 16], data="sat", seed=9116, ways=("bank", "op"), light=True,
                      branches=("dist_inf", "key_inf")),
    "overflow_d1024": dict(D=1024, a=8, b=4, long_len=25, tur_len=25, cur_len=1, key_len=3, ntm_dim=32,
                           chunks=[16, 16, 16], data="overflow", seed=9117, ways=("bank", "op"), light=True,
                           branches=("dist_inf", "c_inf", "diff_nan")),
}


def star_dict(c):
    """the ops.StreamBank config of a case"""
    return dict(D=c["D"], grid=GRID, cur_size=c["a"], long_size=c["b"], long_len=c["long_len"], tur_len=c["tur_len"],
                cur_len=c["cur_len"], key_len=c["key_len"], ntm_dim=c["ntm_dim"], ratio=RATIO)


def star_oracle(c):
    return O.StarConfig(cur_len=c["cur_len"], cur_size=c["a"], long_len=c["long_len"], long_size=c["b"],
                        tur_len=c["tur_len"], key_length=c["key_len"], update_ratio=RATIO)


@functools.lru_cache(maxsize=2)
def case_features(name):
    """[frames, 576, D] f16 ViT features of the case (what the bank pools)"""
    c = CASES[name]
    g = GI._gen(c["seed"])
    N, D, P = sum(c["chunks"]), c["D"], GRID * GRID
    out = torch.empty(N, P, D, dtype=torch.float16)
    scale, offset = {"scene": (1.0, 0.0), "dup": (1.0, 0.0), "sat": (16.0, 0.0), "overflow": (3000.0, 20000.0)}[c["data"]]
    if c["data"] == "dup":
        base = torch.randn(4, P, D, generator=g).half()
        which = torch.randint(0, 4, (N,), generator=g)
        out.copy_(base[which])
        return out
    t = 0
    while t < N:
        n = int(torch.randint(3, 10, (1,), generator=g))
        scene = torch.randn(P, D, generator=g)
        for _ in range(min(n, N - t)):
            out[t] = ((scene + 0.15 * torch.randn(P, D, generator=g)) * scale + offset).half()
            t += 1
    return out


@functools.lru_cache(maxsize=None)
def case_ntm(name):
    """(q_w, q_b, k_w, k_b) f16 torch tensors.  Scaled features get weights scaled down by the same factor, so that the
    Turing projections stay finite (their saturation is not what those cases are about)."""
    c = CASES[name]
    w = GI.ntm_weights(c["D"], c["ntm_dim"], c["seed"])
    s = {"sat": 1 / 16, "overflow": 1 / 20000}.get(c["data"], 1.0)
    return tuple((w[k].float() * s).half() if k.endswith("_w") else w[k] for k in ("q_w", "q_b", "k_w", "k_b"))


def case_draws(name, step, T, K):
    """the k-means draws of step `step` (init_idx [K], refill_idx [10 K] int32 numpy)"""
    return GI.kmeans_draws(T, K, CASES[name]["seed"] * 100 + step)


def plan(c):
    """the per-step shapes prepare_job derives (csrc/stream_kernels.cu) -> list of dicts T, K, S, kl, kmeans, chunks,
    n_long, n_tur, n_cur, cur_start"""
    out, n_long, n_tur = [], 0, 0
    S = c["b"] * c["b"] * c["D"] // 1024
    for s, t in enumerate(c["chunks"]):
        mem = s > 0
        T = (n_long if mem else 0) + t
        K = c["long_len"]
        km = mem and K > 0 and T > K
        kl = min(c["key_len"], K if km else T) if mem and K > 0 else 0
        n_in = (n_tur if mem else 0) + t
        T1 = c["tur_len"]
        n_ch = -(-(n_in - T1) // T1) if mem and n_in > T1 else 0
        chunks = [min(T1, n_in - T1 - i * T1) for i in range(n_ch)]
        n_long = 0 if K == 0 else (K if km else T)
        n_tur = T1 if n_ch else n_in
        cur_start = min(c["cur_len"], t)
        # (long_len 0: the kernel's long working set still takes the clip's level-b rows, which no step reads: T = 0)
        out.append(dict(T=T if K > 0 else 0, K=K, S=S, kl=kl, kmeans=km, chunks=chunks, n_long=n_long, n_tur=n_tur,
                        n_cur=kl + cur_start, cur_start=cur_start))
    return out


@functools.lru_cache(maxsize=1)
def oracle_run(name):
    """the oracle over the whole case -> per step: dict(cur, long, key_idx, labels, exit_step, refills, converged, wsum,
    trace, tur_new [t, 1, D] f16).  The Turing rows the oracle keeps are its fp64-accurate ones; the GPU file holds the
    device's Turing rows to tests.llava_abstract instead."""
    c = CASES[name]
    feats = case_features(name).numpy()
    ntm = tuple(x.numpy() for x in case_ntm(name))
    cfg = star_oracle(c)
    st, out, pos, n_long = O.StreamState(), [], 0, 0
    for s, t in enumerate(c["chunks"]):
        fa = O.spatial_pool(feats[pos:pos + t], c["a"])
        pos += t
        T = n_long + t
        dn = case_draws(name, s, T, c["long_len"]) if s > 0 and 0 < c["long_len"] < T else (None, None)
        tr = []
        st, dbg = O.stream_step(st, fa, cfg, ntm, init_idx=dn[0], refill_idx=dn[1], trace=tr)
        n_long = st.long.shape[0]
        out.append(dict(cur=st.cur.copy(), long=st.long.copy(), key_idx=dbg.get("key_idx", np.zeros(0, np.int64)),
                        labels=dbg.get("labels"), exit_step=dbg.get("exit_step"), refills=dbg.get("refills"),
                        wsum=dbg.get("weight") if "labels" in dbg else None, trace=tr[0],
                        tur_new=O.spatial_pool(fa, 1), n_frames=pos))
    return out


# ------------------------------------------------------------------------------------------------ the proofs
def test_every_case_is_admitted_by_the_fused_step():
    """the host-side checks of check_config / _fused_reject, restated: every case runs on the fused kernel"""
    for name, c in CASES.items():
        D, a, b = c["D"], c["a"], c["b"]
        assert GRID % a == 0 and a != GRID and a * a <= 64 and b > 0 and a % b == 0 and a != b, name
        assert D % 256 == 0 and (b * b * D) % 1024 == 0, name
        assert 0 <= c["long_len"] <= 64 and 0 < c["tur_len"] <= 64 and 0 < c["ntm_dim"] <= 64, name
        assert 0 <= c["key_len"] <= 8 and c["cur_len"] >= 0, name
        for p in plan(c):
            assert p["T"] <= 192 and p["S"] <= 32, (name, p)


def test_admitted_compress_sizes_are_all_covered():
    """every compress_size the fused step admits at grid 24 (a proper long size exists for a > 1), at D 256 and 1024"""
    admitted = {a for a in range(1, GRID) if GRID % a == 0 and a * a <= 64 and any(a % b == 0 and b != a
                                                                                     for b in range(1, a + 1))}
    assert admitted == {2, 3, 4, 6, 8}
    assert admitted <= {c["a"] for c in CASES.values()}
    assert {256, 1024} <= {c["D"] for c in CASES.values() if c["a"] != 8 or c["b"] != 4}
    S = {c["b"] * c["b"] * c["D"] // 1024 for c in CASES.values()}
    assert 1 in S and max(S) == 32 and any(s >= 9 for s in S if s < 32)


@pytest.mark.parametrize("name", list(CASES))
def test_inputs_are_pinned(name):
    """the seeded inputs of every case, by checksum; the table at the end of this file was recorded with torch's CPU
    generator (an RNG change that moves them fails here first)"""
    got = int(GI.checksum(case_features(name)).sum()) + sum(int(GI.checksum(w).sum()) for w in case_ntm(name))
    assert got == PINNED[name], (name, got)


@pytest.mark.parametrize("name", list(CASES))
def test_case_reaches_its_branches(name):
    c = CASES[name]
    P = plan(c)
    br = set(c["branches"])
    if "first_clip_over_bank" in br:
        assert P[0]["n_long"] == 32 > c["long_len"] and P[0]["n_tur"] == 32 > c["tur_len"]
    if "T57" in br:
        assert 57 in [p["T"] for p in P if p["kmeans"]]
    if "T64" in br:
        assert 64 in [p["T"] for p in P if p["kmeans"]]
    if "ragged7" in br:
        assert [25, 7] in [p["chunks"] for p in P]
    if "no_long" in br:
        assert all(p["n_long"] == 0 and p["kl"] == 0 and not p["kmeans"] for p in P)
        assert all(p["n_cur"] == p["cur_start"] for p in P)
    if "chunk_over_32" in br:
        assert any(ch > 32 for p in P for ch in p["chunks"])
    if "T192" in br:
        assert max(p["T"] for p in P) == 192
    if "K64" in br:
        assert any(p["kmeans"] and p["K"] == 64 for p in P)
    if "S32" in br:
        assert P[0]["S"] == 32
    if "key8" in br:
        assert any(p["kl"] == 8 for p in P)
    if "tur64_h64" in br:
        assert c["tur_len"] == 64 and c["ntm_dim"] == 64 and any(p["chunks"] == [64, 64] for p in P)
    if "S1" in br:
        assert P[0]["S"] == 1
    if "S9" in br:
        assert P[0]["S"] == 9
    if "kl_warmup" in br:
        assert any(0 < p["kl"] < c["key_len"] for p in P)
    if "kmeans" in br:
        assert any(p["kmeans"] for p in P)
    if "cur_none" in br:
        assert all(p["cur_start"] == 0 for p in P)
    if "cur_all_of_clip" in br:
        assert any(0 < p["cur_start"] == t for p, t in zip(P, c["chunks"]))
    if "cur_clip_end" in br:
        assert any(p["cur_start"] < t for p, t in zip(P, c["chunks"]))
    if "many_chunks" in br:
        assert max(len(p["chunks"]) for p in P) >= 32
    if "mbuf_both" in br:
        assert {len(p["chunks"]) % 2 for p in P if p["chunks"]} == {0, 1}
    if not c["light"]:
        return
    R = oracle_run(name)
    for s, (p, r) in enumerate(zip(P, R)):
        tr = r["trace"]
        assert (tr["T"], tr["K"], tr["S"], tr["kl"], tr["kmeans"], tr["chunks"]) == \
            (p["T"], p["K"], p["S"], p["kl"], p["kmeans"], p["chunks"]), (name, s, tr, p)
        assert r["long"].shape[0] == p["n_long"] and r["cur"].shape[0] == p["n_cur"], (name, s)
    iters = [it for r in R for it in r["trace"]["iters"]]
    if "refill2" in br:
        assert sum(1 for it in iters if it["refills"] > 0) >= 2
        assert any(r["refills"] and r["refills"] > 0 for r in R)
    if "dist_inf" in br:
        assert any(it["dist_inf"] for it in iters)
    if "key_inf" in br:
        # the key distances of the first key frames: inf against every frame of another scene (its per-patch sums are
        # finite, their f16 total is not), finite only within the key frame's own scene
        c_ = CASES[name]
        feats = case_features(name).numpy()
        lng = O.spatial_pool(O.spatial_pool(feats[:c_["chunks"][0]], c_["a"]), c_["b"])
        terms = O._sqdiff_f16(lng[:, None], lng[None, :2])
        tot = O._seq_sum(O._lane_sum(terms).astype(O.F16).astype(O.F32), -1).astype(O.F16)
        off = ~np.eye(lng.shape[0], 2, dtype=bool)
        with np.errstate(over="ignore"):
            per_patch = O._lane_sum(terms).astype(O.F16).astype(O.F32)
        assert np.isfinite(per_patch).all() and np.isinf(tot.astype(np.float32)[off]).mean() > 0.8
    if "c_inf" in br:
        assert any(it["c_inf"] for it in iters)
        # every distance of a row that is not the seed of a finite centroid is inf: the tie goes to cluster 0, the first
        # index (finite features never give a NaN distance, so NaN reaches the convergence diff, not the labels).  At the
        # first k-means step every working-set row is a distinct frame; later ones also hold copies of refilled rows.
        r = R[1]
        init = case_draws(name, 1, len(r["labels"]), c["long_len"])[0]
        rest = np.setdiff1d(np.arange(len(r["labels"])), init[1:])
        assert (r["labels"][rest] == 0).all() and len(rest) > 1
    if "diff_nan" in br:
        assert any(np.isnan(it["diff"]) for it in iters)


def test_long_len_zero_is_no_long_memory_from_the_first_step():
    """the oracle's long_len == 0: no long rows and no key frames from the first step on (the op-by-op path and the fused
    kernel do the same; DESIGN.md §6)"""
    c = dict(CASES["bank256_d1024"], D=256, chunks=[5, 3, 70])
    feats = GI.scene_features(78, 64, 256, 7)
    w = GI.ntm_weights(256, 32, 7)
    ntm = tuple(w[k].numpy() for k in ("q_w", "q_b", "k_w", "k_b"))
    st, pos = O.StreamState(), 0
    for s, t in enumerate(c["chunks"]):
        tr = []
        st, dbg = O.stream_step(st, feats[pos:pos + t].numpy(), star_oracle(c), ntm, trace=tr)
        pos += t
        assert st.long.shape == (0, 16, 256) and len(dbg.get("key_idx", [])) == 0
        assert np.array_equal(st.cur.view(np.int16), feats[pos - min(3, t):pos].numpy().view(np.int16))
        assert tr[0]["kmeans"] is False and tr[0]["kl"] == 0
    assert st.prefix().shape == (64 + 3 * 64, 256)


@pytest.mark.parametrize("name", list(GI.abstract_cases()))
def test_kernel_order_abstract_update_vs_oracle_and_golden(name):
    """tests.llava_abstract (the kernel's order, exp correctly rounded) against oracle.abstract_update within its 4 ulp,
    and against the reference golden at that golden's bar; its candidate set holds the nominal result"""
    from tests.test_oracle_golden import load, same_inputs, ulp_diff_f16
    z = load("abstract.npz")
    M, F, seed = GI.abstract_cases()[name]
    same_inputs(z, f"{name}_in_sum", M, F)
    w = GI.ntm_weights(M.shape[1], 32, seed)
    a = [w[k].numpy() for k in ("q_w", "q_b", "k_w", "k_b")]
    nom = LA.update_nominal(M.numpy(), [F.numpy()], *a, 0.2)
    assert ulp_diff_f16(nom, O.abstract_update(M.numpy(), F.numpy(), *a, 0.2)).max() <= 4
    ref = z[f"{name}_out"]
    rel = np.linalg.norm(nom.astype(np.float32) - ref.astype(np.float32)) / np.linalg.norm(ref.astype(np.float32))
    assert rel < 1e-3 and ulp_diff_f16(nom, ref).max() <= 4
    cands, _ = LA.update_candidates(M.numpy(), [F.numpy()], *a, 0.2)
    LA.check_rows(nom, cands)


def test_kernel_order_restatement_sees_a_dropped_rounding():
    """the restatement is sharp: dropping the f16 rounding of 1 - decay moves some element of a 25 x 1024 update"""
    M, F, seed = GI.abstract_cases()["chunk"]
    w = GI.ntm_weights(1024, 32, seed)
    a = [w[k].numpy() for k in ("q_w", "q_b", "k_w", "k_b")]
    cands, _ = LA.update_candidates(M.numpy(), [F.numpy()], *a, 0.2)
    q, k = LA.proj(M.numpy(), a[0], a[1]), LA.proj(F.numpy(), a[2], a[3])
    wt, _, _ = LA.weights(q, k, 0.2)
    decay = LA._rh(LA.lane_strided_sum(wt))
    acc = np.zeros((25, 1024), np.float32)
    for j in range(25):
        acc = acc + wt[:, j:j + 1] * F.numpy()[j].astype(np.float32)[None]
    keep = LA._rh(M.numpy().astype(np.float32) * (np.float32(1) - decay)[:, None])
    bad = (keep + LA._rh(acc)).astype(np.float16)
    with pytest.raises(AssertionError):
        LA.check_rows(bad, cands)


PINNED = {
    "default_d1024_clip32": 1752000532407,
    "bank256_d1024": 2189955445209,
    "limits_d2048": 7008511624256,
    "a2_b1_d1024": 548738569448,
    "a3_b1_d1024": 548921381864,
    "a4_b2_d256": 137209491887,
    "a4_b1_d1024": 548847157812,
    "a6_b3_d1024": 548672077721,
    "a6_b2_d256": 137111098511,
    "a8_b2_d1024": 548828893289,
    "cur0_d256": 146313181948,
    "cur3_single_d256": 137237343248,
    "cur5_d256": 178177880003,
    "tur1_h1_d256": 437434274410,
    "dup_d1024": 1751872239058,
    "sat_d1024": 934273120680,
    "overflow_d1024": 868004135691,
}
