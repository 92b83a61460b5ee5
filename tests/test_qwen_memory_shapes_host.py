"""The Qwen2-VL Flash Memory kernels at the shapes a real stream runs (CPU half).

csrc/qwen_kernels.cu is bit-exact against oracle/qwen_oracle.py, but most of its code only runs past the toy shapes of
test_qwen_gpu_parity.py: the 2-stage cp.async ring of KO_KC = 8 centroid slices (K > 8), the 32-partial chains of
seq_reduce / ko_converge (S >= 33 slices: two passes), the incremental Lloyd loop (dirty / refilled
clusters, a change list that shrinks, no commit on a tolerance stop), the klarge row groups and the f16 overflow to
inf / NaN, and lex_compare's 1024-element chunks.  This file holds the case table that
test_qwen_memory_shapes_gpu.py runs on the GPU, pins its seeded generators, and proves with the oracle's trace that each
case reaches the branch it names — so an RNG or torch change that moves a case off its branch fails here, on any
machine, instead of passing quietly on the GPU."""
import numpy as np
import pytest
import torch

from oracle import qwen_oracle as QO
from tests.golden_inputs import _gen, checksum
from tests.qwen_inputs import DT

SLICE = 1024
KO_KC = 8          # centroid slices per cp.async stage of ko_partial
PD_REAL = 184320   # 12x12 half-resolution tokens x 1280 (336 px)
NEVER = 0.0        # tol that never stops the loop (diff < 0 is never true)

# ------------------------------------------------------------------------------------------------ ordered k-means
# name -> K, S (slices of 1024), T, x dtype, data ("iid" / "scene" / "stream"), weights, max_iter, tol, seed, and the
# branches the case must reach (checked below from the oracle's trace).  The hex tol values are the fp32 just above the
# trace's diff at the iteration that must stop the loop (0-based, the `exit_step` of kmeans_ordered_core) while that diff
# is still > 0: the new centroids differ from the old ones and must not be committed.
KMEANS_CASES = {
    "k8_s1_stop_it0": dict(K=8, S=1, T=9, dtype="bf16", data="scene", weights="ones", max_iter=10, tol=1e6, seed=701,
                           branches=("stop_it0",)),
    "k9_s33_f16_iid": dict(K=9, S=33, T=61, dtype="f16", data="iid", weights="rand", max_iter=10,
                           tol=float.fromhex("0x1.7dcb28p+6"), seed=702,
                           branches=("chunks", "two_passes", "t_ragged", "stop_it1", "stop_dirty", "skip")),
    "k17_s33_f32_iid": dict(K=17, S=33, T=56, dtype="f32", data="iid", weights="ints", max_iter=10, tol=NEVER, seed=703,
                            branches=("chunks", "two_passes", "never", "subset", "skip", "idle")),
    "k60_s1_half0": dict(K=60, S=1, T=61, dtype="bf16", data="scene", weights="half0", max_iter=10, tol=NEVER, seed=704,
                         branches=("chunks", "t_ragged", "never", "refill2", "re_refill", "subset", "skip")),
    "k8_s180_bf16_iid": dict(K=8, S=180, T=29, dtype="bf16", data="iid", weights="ones", max_iter=10, tol=1e-4, seed=705,
                             branches=("two_passes", "t_ragged", "stop_it1")),
    "k9_s270_f32": dict(K=9, S=270, T=10, dtype="f32", data="scene", weights="ones", max_iter=10, tol=NEVER, seed=706,
                        branches=("chunks", "two_passes", "t_ragged", "never")),
    "k17_s33_f16_maxiter0": dict(K=17, S=33, T=61, dtype="f16", data="scene", weights="ones", max_iter=0, tol=1e-4,
                                 seed=707, branches=("chunks", "two_passes", "t_ragged", "degenerate")),
    "k60_s1_f32_iid": dict(K=60, S=1, T=185, dtype="f32", data="iid", weights="rand", max_iter=10,
                           tol=float.fromhex("0x1.2be064p+0"), seed=708,
                           branches=("chunks", "t_ragged", "stop_it2_4", "stop_dirty", "moving", "subset", "skip")),
    "k17_s180_f16_half0": dict(K=17, S=180, T=18, dtype="f16", data="scene", weights="half0", max_iter=10, tol=NEVER,
                               seed=709, branches=("chunks", "two_passes", "refill2", "subset", "skip")),
    "k8_s270_bf16_ints": dict(K=8, S=270, T=61, dtype="bf16", data="scene", weights="ints", max_iter=10, tol=1e-4,
                              seed=710, branches=("two_passes", "t_ragged", "stop_it2_4", "subset", "skip")),
    "k9_s1_bf16_iid": dict(K=9, S=1, T=32, dtype="bf16", data="iid", weights="half0", max_iter=10, tol=NEVER, seed=711,
                           branches=("chunks", "never", "moving", "refill2", "subset", "skip")),
    "k60_s33_f16_ints": dict(K=60, S=33, T=61, dtype="f16", data="stream", weights="ints", max_iter=10, tol=1e-4, seed=712,
                             branches=("chunks", "two_passes", "t_ragged", "stop_it2_4", "subset", "skip")),
    # one full BASELINE CSM update: 61 half-resolution frames of 144 tokens x 1280 -> 60 centroids, reference tol
    "k60_s180_bf16_baseline": dict(K=60, S=180, T=61, dtype="bf16", data="stream", weights="ones", max_iter=10, tol=1e-4,
                                   seed=713, branches=("chunks", "two_passes", "t_ragged", "subset", "skip")),
}


def kmeans_input(c):
    """-> X [T, S*1024] in the case's dtype, weights fp32 [T], init rows int32 [K] (distinct), refill rows int32"""
    g = _gen(c["seed"])
    T, K, PD = c["T"], c["K"], c["S"] * SLICE
    if c["data"] == "iid":
        x = torch.randn(T, PD, generator=g)
    else:      # "scene": a few shots of a slowly changing video; "stream": 40 scenes over 61 frames (the BASELINE stream)
        n, noise = (40, 0.3) if c["data"] == "stream" else (max(2, (2 * K) // 3), 0.2)
        scenes = torch.randn(n, PD, generator=g)
        which = torch.sort(torch.randint(0, n, (T,), generator=g)).values
        x = scenes[which] + noise * torch.randn(T, PD, generator=g)
    x = x.to(DT[c["dtype"]])
    if c["weights"] == "ones":
        w = torch.ones(T)
    elif c["weights"] == "ints":             # the carried CSM weights of a stream: small integer member counts
        w = torch.randint(1, 5, (T,), generator=g).float()
    elif c["weights"] == "rand":
        w = torch.rand(T, generator=g) * 3 + 0.25
    else:                                    # "half0": half the rows weightless -> clusters empty out and are refilled
        w = torch.rand(T, generator=g) + 0.5
        w[torch.randperm(T, generator=g)[: T // 2]] = 0.0
    init = torch.randperm(T, generator=g)[:K].to(torch.int32)
    refill = torch.randint(0, T, (max(1, c["max_iter"] * K),), generator=g, dtype=torch.int32)
    return x, w, init, refill


def kmeans_oracle(c):
    """-> (C fp32 [K, PD], labels int32 [T], wsum fp32 [K] or None, info [last iteration, refills consumed, converged],
    trace).  max_iter == 0 is the degenerate branch: one assignment to the seed rows, nothing updated."""
    x, w, init, refill = kmeans_input(c)
    X = QO._f32(x)
    if c["max_iter"] == 0:
        C = X[init.long().numpy()].copy()
        labels = QO.argmin_first_nan(QO.efficient_euclidean_distance(X, C), axis=1).astype(np.int32)
        return C, labels, None, [0, 0, 0], []
    trace = []
    tol = c["tol"]
    C, labels, wsum, it, used = QO.kmeans_ordered_core(X, w.numpy(), init.numpy(), refill.numpy(), c["K"], c["max_iter"],
                                                       tol, trace=trace)
    converged = int(bool(trace[-1]["diff"] < np.float32(tol)))
    return C, labels, wsum, [it, used, converged], trace


def dirty(trace, i):
    """clusters that gained or lost a row between iterations i-1 and i (ko_assign's dirty flags)"""
    a, b = trace[i - 1]["labels"], trace[i]["labels"]
    m = a != b
    return set(a[m].tolist()) | set(b[m].tolist())


def reached(c, trace):
    """the branches of KMEANS_CASES' vocabulary that this case's run reaches"""
    K, S, T = c["K"], c["S"], c["T"]
    got = set()
    if K > KO_KC and K % KO_KC:
        got.add("chunks")                    # more than one stage of the ring, and a partial last stage
    if S >= 33:
        got.add("two_passes")                # seq_reduce / ko_converge chain over two 32-partial passes
    if T % 8:
        got.add("t_ragged")                  # the last 8-row block of ko_partial is partial
    if c["max_iter"] == 0:
        got.add("degenerate")
        return got
    tol = np.float32(c["tol"])
    last = len(trace) - 1
    if trace[last]["diff"] < tol:
        if last == 0:
            got.add("stop_it0")              # nothing is ever committed
        elif last == 1:
            got.add("stop_it1")
        elif 2 <= last <= 4:
            got.add("stop_it2_4")
        if last > 0 and trace[last]["diff"] > 0:
            got.add("stop_dirty")            # stopped while a centroid still changed: ko_commit must not run
    elif len(trace) == c["max_iter"]:
        got.add("never")
    if sum(1 for r in trace[1:4] if r["moved"] > 0) == 3:
        got.add("moving")                    # labels still move in iterations 1, 2 and 3
    for i in range(1, len(trace)):
        sweep = trace[i - 1]["changed"]      # the change list ko_partial sweeps in iteration i
        if 0 < len(sweep) < K:
            got.add("subset")
        if not sweep:
            got.add("idle")                  # nothing changed: ko_partial and ko_commit have nothing to do
        clean = set(range(K)) - dirty(trace, i) - set(trace[i - 1]["refilled"])
        if clean:
            got.add("skip")                  # ko_update skips an unchanged cluster
        if set(trace[i - 1]["refilled"]) - dirty(trace, i):
            got.add("re_refill")             # refilled, no row moved, and still re-drawn: only wprev says so
    if sum(1 for r in trace if r["refilled"]) >= 2:
        got.add("refill2")
    return got


# ------------------------------------------------------------------------------------------------ klarge retrieval
# name -> metric, dtype, PD, k (centroids retrieved), t (bank frames), data, seed, branches.  "order" data puts two
# equal-and-opposite 1024-element blocks 40 slices apart on top of small values, so every similarity is a cancellation
# whose bits depend on the order in which the slice partials are added.
KLARGE_CASES = {
    "kl_eu_bf16_real": dict(metric="euclidean", dtype="bf16", PD=PD_REAL, k=30, t=250, data="near", seed=801, branches=()),
    "kl_eu_f16_overflow": dict(metric="euclidean", dtype="f16", PD=PD_REAL, k=30, t=17, data="near", seed=802,
                               branches=("inf", "nan", "nan_wins")),
    "kl_eu_f16_k64": dict(metric="euclidean", dtype="f16", PD=PD_REAL, k=64, t=17, data="small", seed=803, branches=()),
    "kl_eu_bf16_k1_t1": dict(metric="euclidean", dtype="bf16", PD=276480, k=1, t=1, data="near", seed=804, branches=()),
    "kl_eu_bf16_26x46": dict(metric="euclidean", dtype="bf16", PD=1530880, k=31, t=2, data="near", seed=805, branches=()),
    "kl_cos_f16_order": dict(metric="cosine", dtype="f16", PD=PD_REAL, k=31, t=33, data="order", seed=806,
                             branches=("order",)),
    "kl_cos_bf16_order": dict(metric="cosine", dtype="bf16", PD=276480, k=64, t=2, data="order", seed=807,
                              branches=("order",)),
    "kl_cos_f16_zero_row": dict(metric="cosine", dtype="f16", PD=276480, k=1, t=250, data="zero_row", seed=808,
                                branches=("nan", "nan_wins")),
}


def klarge_input(c):
    """-> (tem_x [k+3, PD], klarge_idx int64 [k], bank [t, PD]) in the case's dtype"""
    g = _gen(c["seed"])
    k, t, PD = c["k"], c["t"], c["PD"]
    st = k + 3
    scale = {"near": 1.0, "small": 0.03, "order": 0.05, "zero_row": 0.5}[c["data"]]
    bank = torch.randn(t, PD, generator=g) * scale
    tem = torch.randn(st, PD, generator=g) * scale
    src = torch.randint(0, t, (st,), generator=g)
    near = torch.rand(st, generator=g) < 0.5        # half the centroids are noisy copies of a bank frame
    tem[near] = bank[src[near]] + 0.1 * scale * torch.randn(int(near.sum()), PD, generator=g)
    if c["data"] == "order":
        v = 16.0 * torch.rand(SLICE, generator=g) + 1.0
        for a in (tem, bank):
            a[:, :SLICE] = v
        tem[:, 40 * SLICE: 41 * SLICE] = v
        bank[:, 40 * SLICE: 41 * SLICE] = -v
    if c["data"] == "zero_row":
        bank[t // 3] = 0.0                              # |b| = 0: every similarity with it is 0/0 = NaN
    kidx = torch.randperm(st, generator=g)[:k]
    dt = DT[c["dtype"]]
    return tem.to(dt), kidx, bank.to(dt)


def klarge_oracle(c):
    tem, kidx, bank = klarge_input(c)
    f = QO.klarge_cosine if c["metric"] == "cosine" else QO.klarge_distances
    d = f(tem[kidx], bank)
    return d, QO.argmin_first_nan(d, axis=1)


# ------------------------------------------------------------------------------------------------ pinned generators
CHECKSUMS = {
    "k8_s1_stop_it0": [2313753, 290599425, 1719, 33228, 36, 492, 334, 34500],
    "k9_s33_f16_iid": [501630591, 63193252246, 26311, 3177514, 267, 4383, 2641, 253716],
    "k17_s33_f32_iid": [955092211, 120335983102, 8373, 965272, 556, 16552, 4750, 567466],
    "k60_s1_half0": [15651844, 1973717386, 14549, 1652883, 1815, 211651, 17938, 2227446],
    "k8_s180_bf16_iid": [1335914412, 168308128044, 5539, 328628, 118, 1810, 1033, 108956],
    "k9_s270_f32": [1394746934, 175748068860, 1910, 40740, 41, 693, 387, 38668],
    "k17_s33_f16_maxiter0": [501424191, 63179335301, 11651, 1436916, 477, 16173, 10, 10],
    "k60_s1_f32_iid": [95568338, 12042651346, 79633, 9665837, 5945, 705685, 55643, 6778051],
    "k17_s180_f16_half0": [807381331, 101735403113, 4533, 173973, 151, 5627, 1600, 186116],
    "k8_s270_bf16_ints": [4216301105, 531209723001, 8310, 991836, 234, 3266, 2552, 257661],
    "k9_s1_bf16_iid": [8184042, 1031018045, 6281, 414391, 191, 3383, 1322, 142843],
    "k60_s33_f16_ints": [502132010, 63266282133, 8372, 1020808, 1793, 229273, 17930, 2211704],
    "k60_s180_bf16_baseline": [2812375913, 354341395735, 11651, 1436916, 1815, 213035, 18312, 2315298],
    "kl_eu_bf16_real": [1520283881, 191571125771, 520, 59336, 11516157704, 1451070092905],
    "kl_eu_f16_overflow": [1480137372, 186510009693, 489, 58921, 762388158, 96041657024],
    "kl_eu_f16_k64": [2755531197, 347170256498, 2104, 266758, 698945917, 88067096489],
    "kl_eu_bf16_k1_t1": [276380219, 34814587399, 0, 0, 69091255, 8705879093],
    "kl_eu_bf16_26x46": [13009601138, 1639320627684, 515, 66267, 765212516, 96399669902],
    "kl_cos_f16_order": [1414406188, 178234575652, 503, 61271, 1377264749, 173540433044],
    "kl_cos_bf16_order": [4533656996, 571208522287, 2173, 267698, 135607005, 17093860816],
    "kl_cos_f16_zero_row": [264636836, 33329129469, 2, 2, 16476933810, 2076104116456],
}


def _chk(*ts):
    return [int(v) for t in ts for v in checksum(t)]


@pytest.mark.parametrize("name", list(KMEANS_CASES))
def test_kmeans_inputs_are_pinned(name):
    c = KMEANS_CASES[name]
    x, w, init, refill = kmeans_input(c)
    assert x.shape == (c["T"], c["S"] * SLICE) and x.dtype == DT[c["dtype"]]
    assert len(set(init.tolist())) == c["K"] and int(refill.max()) < c["T"]
    assert _chk(x, w, init, refill) == CHECKSUMS[name], "seeded input drifted"


@pytest.mark.parametrize("name", list(KLARGE_CASES))
def test_klarge_inputs_are_pinned(name):
    c = KLARGE_CASES[name]
    tem, kidx, bank = klarge_input(c)
    assert bank.shape == (c["t"], c["PD"]) and kidx.numel() == c["k"]
    assert _chk(tem, kidx, bank) == CHECKSUMS[name], "seeded input drifted"


# ------------------------------------------------------------------------------------------------ branches reached
@pytest.mark.parametrize("name", list(KMEANS_CASES))
def test_kmeans_case_reaches_its_branches(name):
    c = KMEANS_CASES[name]
    C, labels, wsum, info, trace = kmeans_oracle(c)
    got = reached(c, trace)
    missing = set(c["branches"]) - got
    assert not missing, f"{name} no longer reaches {sorted(missing)} (reaches {sorted(got)})"
    if c["max_iter"]:
        assert info[0] == len(trace) - 1 and info[1] == sum(len(r["refilled"]) for r in trace)


def test_kmeans_table_covers_the_grid():
    """every value the issue's grid names appears, and every branch is reached by some case"""
    cs = KMEANS_CASES.values()
    assert {8, 9, 17, 60} <= {c["K"] for c in cs}
    assert {1, 33, 180, 270} <= {c["S"] for c in cs}
    assert {"bf16", "f16", "f32"} <= {c["dtype"] for c in cs}
    assert {"ones", "ints", "rand", "half0"} <= {c["weights"] for c in cs}
    Ts = {(c["K"], c["T"]) for c in cs}
    assert any(T == K + 1 for K, T in Ts) and any(T == 61 for K, T in Ts) and any(T == 3 * K + 5 for K, T in Ts)
    assert any(c["K"] == 60 and c["S"] == 180 and c["T"] == 61 and c["dtype"] == "bf16" for c in cs)
    every = {"chunks", "two_passes", "t_ragged", "subset", "skip", "idle", "refill2", "re_refill", "moving", "stop_it0",
             "stop_it1", "stop_it2_4", "stop_dirty", "never", "degenerate"}
    assert every == {b for c in cs for b in c["branches"]}


@pytest.mark.parametrize("name", list(KLARGE_CASES))
def test_klarge_case_reaches_its_branches(name):
    c = KLARGE_CASES[name]
    d, idx = klarge_oracle(c)
    got = set()
    if np.isinf(d).any():
        got.add("inf")
    if np.isnan(d).any():
        got.add("nan")
        if all(np.isnan(d[i, idx[i]]) for i in range(len(idx)) if np.isnan(d[i]).any()):
            got.add("nan_wins")
    if c["data"] == "order":
        # the cancellation: most similarities are far smaller than the two blocks' partials, so the rounding of adding the
        # other slices next to a partial of ~0.5 (in fp32) shows in their 16-bit bits, and a different slice order moves them
        tem, kidx, bank = klarge_input(c)
        an = QO._round(QO._f32(tem[kidx][:, :SLICE]) / QO.row_norm(tem[kidx])[:, None], tem.dtype)
        bn = QO._round(QO._f32(bank[:, :SLICE]) / QO.row_norm(bank)[:, None], bank.dtype)
        block = an @ bn.T
        if np.median(np.abs(d) / block) < 1e-4:
            got.add("order")
    missing = set(c["branches"]) - got
    assert not missing, f"{name} no longer reaches {sorted(missing)}"
    if c["metric"] == "euclidean" and c["dtype"] == "bf16":
        assert np.isfinite(d).all()


def test_klarge_table_covers_the_grid():
    cs = KLARGE_CASES.values()
    assert {PD_REAL, 276480, 1530880} <= {c["PD"] for c in cs}
    assert {1, 30, 31, 64} <= {c["k"] for c in cs}
    assert {1, 2, 17, 33, 250} <= {c["t"] for c in cs}
    assert {(m, d) for m in ("euclidean", "cosine") for d in ("bf16", "f16")} <= {(c["metric"], c["dtype"]) for c in cs}
