"""GPU tests of the CSM chain of many Qwen2-VL streams in one launch per kernel (DESIGN.md §3.17).

ABI level: random jobs of different T, K, PD, dtypes, draws, iteration caps and tolerances go once through each
fvs_qwen_*_multi entry point and once through the single-stream calls; every output must be torch.equal, whatever the
budget (down to one job per launch group).  Pool level: QwenStreamPool against the same streams stepped alone through
QwenStreamState, and against a pool whose BATCH_MIN_JOBS is above its stream count (every k-means stream steps its
memory in a one-item call), bit for bit after every round."""
import random

import pytest
import torch

from tests.qwen_mem_multi_inputs import Alone, clip, host_for, merger, rt, run, tower  # noqa: F401  (module fixtures)

pytestmark = pytest.mark.gpu


def make_job(seed, T, K, P, dtype, dup=0, clustered=False, max_iter=10, tol=1e-4, order=False):
    """inputs of one k-means job: X [T, P*1024], weights, draws (init from the unique rows, refills over T)"""
    g = torch.Generator().manual_seed(seed)
    PD = P * 1024
    if clustered:                                   # a few well-separated centres: the loop meets the tolerance early
        cent = torch.randn(3, PD, generator=g) * 4
        X = cent[torch.arange(T) % 3] + 1e-3 * torch.randn(T, PD, generator=g)
    else:
        X = torch.randn(T, PD, generator=g)
    for d in range(dup):                            # duplicate rows: fewer unique rows than T
        X[T - 1 - d] = X[d]
    X = X.to(dtype).cuda()
    w = (torch.rand(T, generator=g) + 0.5).cuda()
    init = torch.randperm(T - dup, generator=g)[:K].to(torch.int32).cuda()
    refill = torch.randint(0, T, (max(1, max_iter * K),), generator=g).to(torch.int32).cuda()
    o = torch.randperm(K, generator=g).cuda() if order else None
    return dict(X=X, w=w, init=init, refill=refill, K=K, max_iter=max_iter, tol=tol, order=o)


def single(j):
    from flash_vstream_b200.qwen import ops as Q
    uniq, nu = Q.unique_rows(j["X"])
    C, wsum, labels, info = Q.kmeans_ordered(j["X"], j["w"], uniq, j["init"], j["refill"], j["K"], j["max_iter"], j["tol"])
    sidx, ts, ws, flags = Q.kmeans_finalize(labels, wsum, j["order"])
    out = Q.gather_rows_cast(C, sidx, j["X"].dtype)
    return dict(uniq=uniq.clone(), nu=nu, C=C, wsum=wsum, labels=labels, info=info, sidx=sidx, ts=ts, ws=ws, flags=flags,
                out=out)


def multi(js, budget):
    from flash_vstream_b200 import _lib as L
    from flash_vstream_b200.qwen import ops as Q
    lib = L.load()
    res, jobs = [], []
    for j in js:
        T, PD = j["X"].shape
        K = j["K"]
        d = "cuda"
        r = dict(uniq=torch.zeros(T, dtype=torch.int32, device=d), nu=torch.empty(1, dtype=torch.int32, device=d),
                 C=torch.empty(K, PD, device=d), wsum=torch.empty(K, device=d),
                 labels=torch.empty(T, dtype=torch.int32, device=d), info=torch.empty(4, dtype=torch.int32, device=d),
                 sidx=torch.empty(K, dtype=torch.int64, device=d), ts=torch.empty(K, device=d), ws=torch.empty(K, device=d),
                 flags=torch.empty(1, dtype=torch.int32, device=d), out=torch.empty(K, PD, dtype=j["X"].dtype, device=d),
                 uws=torch.empty(lib.fvs_qwen_unique_workspace_bytes(T), dtype=torch.uint8, device=d),
                 kws=torch.empty(lib.fvs_qwen_kmeans_workspace_bytes(T, K, PD), dtype=torch.uint8, device=d))
        jobs.append(Q.mem_job(j["X"], K, w=j["w"], init_idx=j["init"], refill_idx=j["refill"], max_iter=j["max_iter"],
                              tol=j["tol"], uniq_idx=r["uniq"], n_unique=r["nu"], uniq_ws=r["uws"], C=r["C"], wsum=r["wsum"],
                              labels=r["labels"], info=r["info"], km_ws=r["kws"], order=j["order"], sorted_idx=r["sidx"],
                              ts=r["ts"], w_sorted=r["ws"], flags=r["flags"], out=r["out"]))
        res.append(r)
    arr = Q.mem_jobs(jobs)
    n0 = lib.fvs_launch_count()
    Q.unique_rows_multi(arr, budget)
    Q.kmeans_multi(arr, budget)
    Q.kmeans_finalize_multi(arr, budget)
    Q.gather_rows_cast_multi(arr, budget)
    return res, lib.fvs_launch_count() - n0, Q.mem_plan(arr, budget)[2]


def equal(a, b):
    if a.dtype in (torch.float16, torch.bfloat16):
        a, b = a.view(torch.int16), b.view(torch.int16)
    elif a.dtype == torch.float32:
        a, b = a.view(torch.int32), b.view(torch.int32)
    return torch.equal(a, b)


@pytest.fixture(scope="module")
def lib(rt):  # noqa: F811
    from flash_vstream_b200 import _lib as L
    return L.load(build_if_missing=False)


@pytest.mark.parametrize("budget", [0, 600, 1])
def test_multi_equals_single_calls(lib, budget):
    r = random.Random(budget)
    dts = [torch.bfloat16, torch.float16, torch.float32]
    js = []
    for i in range(19):                              # more jobs than one launch group takes
        T = r.choice([5, 9, 17, 33, 61])
        K = r.randint(1, min(T - 3, 12))
        js.append(make_job(100 + i, T, K, r.choice([1, 2, 3]), dts[i % 3], dup=2 if i % 5 == 0 else 0,
                           clustered=i % 4 == 1, max_iter=[10, 3, 0, 10][i % 4] if i % 5 else 10,
                           tol=1e9 if i % 7 == 3 else 1e-4, order=i % 6 == 2))
    got, launches, groups = multi(js, budget)
    for i, j in enumerate(js):
        ref = single(j)
        for k, v in ref.items():
            if j["max_iter"] == 0 and k in ("wsum", "ws"):
                continue                             # the degenerate branch computes no weight sums (its caller uses ones)
            assert equal(got[i][k], v), (budget, i, k)
    exits = {int(g["info"][0]) for g in got}
    assert len(exits) > 2, exits                     # the jobs stopped at different iterations
    assert groups == (2 if budget == 0 else len(js) if budget == 1 else groups)
    assert groups >= 2 and launches > 0


def test_one_job_alone_and_next_to_others(lib):
    """a job's bits do not depend on its neighbours: the same job in three different tables"""
    a = make_job(7, 61, 30, 2, torch.bfloat16)
    others = [make_job(8 + i, 9 + 4 * i, 4, 1, torch.float16, clustered=True) for i in range(5)]
    outs = [multi([a], 0)[0][0], multi(others[:2] + [a] + others[2:], 0)[0][2], multi(others + [a], 3)[0][5]]
    for o in outs[1:]:
        for k in o:
            if k not in ("uws", "kws"):
                assert equal(o[k], outs[0][k]), k


def test_refused_table_launches_nothing(lib):
    from flash_vstream_b200.qwen import ops as Q
    js = [make_job(1, 9, 4, 1, torch.bfloat16), make_job(2, 9, 4, 1, torch.bfloat16)]
    res, _, _ = multi(js, 0)
    C = res[0]["C"]
    bad = Q.mem_job(js[1]["X"], 4, w=js[1]["w"], init_idx=js[1]["init"], refill_idx=js[1]["refill"],
                    uniq_idx=res[1]["uniq"], n_unique=res[1]["nu"], uniq_ws=res[1]["uws"], C=C, wsum=res[1]["wsum"],
                    labels=res[1]["labels"], info=res[1]["info"], km_ws=res[1]["kws"])
    good = Q.mem_job(js[0]["X"], 4, w=js[0]["w"], init_idx=js[0]["init"], refill_idx=js[0]["refill"],
                     uniq_idx=res[0]["uniq"], n_unique=res[0]["nu"], uniq_ws=res[0]["uws"], C=C, wsum=res[0]["wsum"],
                     labels=res[0]["labels"], info=res[0]["info"], km_ws=res[0]["kws"])
    n0 = lib.fvs_launch_count()
    with pytest.raises(ValueError, match="share an output"):
        Q.kmeans_multi([good, bad])
    assert lib.fvs_launch_count() == n0


def launches(lib, fn):
    n0 = lib.fvs_launch_count()
    fn()
    return lib.fvs_launch_count() - n0


@pytest.mark.parametrize("call, max_iter, want", [("unique", 10, 2), ("kmeans", 10, 3 + 6 * 10 + 1),
                                                  ("kmeans", 3, 3 + 6 * 3 + 1), ("kmeans", 0, 7), ("finalize", 10, 1),
                                                  ("gather", 10, 1)])
def test_single_call_launch_counts(lib, call, max_iter, want):
    """a single call is the one-job table: the launches of its stage sequence, one per stage and iteration"""
    from flash_vstream_b200.qwen import ops as Q
    j = make_job(3, 33, 8, 2, torch.bfloat16, max_iter=max_iter)
    uniq, _ = Q.unique_rows(j["X"])
    kmeans = lambda: Q.kmeans_ordered(j["X"], j["w"], uniq, j["init"], j["refill"], j["K"], j["max_iter"], j["tol"])  # noqa: E731
    C, wsum, labels, _ = kmeans()
    sidx = Q.kmeans_finalize(labels, wsum)[0]
    fns = dict(unique=lambda: Q.unique_rows(j["X"]), kmeans=kmeans, finalize=lambda: Q.kmeans_finalize(labels, wsum),
               gather=lambda: Q.gather_rows_cast(C, sidx, torch.bfloat16))
    assert launches(lib, fns[call]) == want


@pytest.mark.parametrize("n_dev", [11, 5, 0])
@pytest.mark.parametrize("metric, sweeps", [("euclidean", 1), ("cosine", 2)])
def test_klarge_launch_counts(lib, metric, sweeps, n_dev):
    """3 (Euclidean) or 6 (cosine) launches, plus one per extra tier of a bank with host rows in each sweep"""
    from flash_vstream_b200.qwen import ops as Q
    from tests.test_qwen_small_tier_gpu import _tiered
    g = torch.Generator().manual_seed(5)
    t, F = 11, 4
    bank = torch.randn(t, 2048, generator=g).bfloat16().cuda()
    tem_x = torch.randn(40, 2048, generator=g).bfloat16().cuda()
    kidx = torch.randperm(40, generator=g)[:30].cuda()
    tb, chunks = _tiered(bank, n_dev, F)
    want = (3 if metric == "euclidean" else 6) + sweeps * (len(Q.klarge_plan(t, n_dev, F)) - 1)
    assert launches(lib, lambda: Q.klarge_retrieve(tem_x, kidx, tb, metric=metric)) == want
    if n_dev == t:
        assert launches(lib, lambda: Q.klarge_retrieve(tem_x, kidx, bank, metric=metric)) == want
    torch.cuda.synchronize()


@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_klarge_retrieve_multi_equals_single_calls(lib, metric, dtype):
    """jobs of different k, bank lengths t_total (rows split across several blocks) and PD, in more than one launch"""
    from flash_vstream_b200.qwen import ops as Q
    r = random.Random(hash((metric, str(dtype))) & 0xffff)
    items = []
    for i in range(19):
        g = torch.Generator().manual_seed(300 + i)
        PD, st, t = 1024 * r.choice([1, 2, 3]), r.randint(4, 70), r.choice([1, 7, 31, 33, 100, 250])
        k = r.randint(1, min(st, 64))
        tem_x = torch.randn(st, PD, generator=g).to(dtype).cuda()
        bank = torch.randn(t, PD, generator=g).to(dtype).cuda()
        if i % 4 == 0:
            bank[t // 2] = 0                                 # a zero row: NaN from the cosine metric, which wins
        items.append((tem_x, torch.randperm(st, generator=g)[:k].cuda(), bank))
    got = Q.klarge_retrieve_multi(items, metric, want_dist=True)
    for i, (tem_x, idx, bank) in enumerate(items):
        ri, rd = Q.klarge_retrieve(tem_x, idx, bank, want_dist=True, metric=metric)
        assert torch.equal(got[i][0], ri) and equal(got[i][1], rd), (metric, dtype, i)


def test_dam_gather_multi_equals_one_job_tables(lib):
    """per job: its own device tier, host chunks (some picks read there), previous DAM and host_fetches counter"""
    from flash_vstream_b200.qwen import ops as Q
    calls, refs = [], []
    for i in range(18):
        g = torch.Generator().manual_seed(500 + i)
        fx, fm, n_frames = 64 * (1 + i % 3), 32 * (1 + i % 2), 12 + i
        n_dev, cf = (n_frames if i % 3 == 0 else 5 + i % 4), 4
        x = torch.randn(n_frames, fx, generator=g).bfloat16()
        mg = torch.randn(n_frames, fm, generator=g).bfloat16()
        chunks, ptrs = [], []
        for c in range(-(-(n_frames - n_dev) // cf)):
            buf = torch.empty(cf * (fx + fm), dtype=torch.bfloat16).pin_memory()
            lo, hi = n_dev + c * cf, min(n_frames, n_dev + (c + 1) * cf)
            buf[: (hi - lo) * fx].copy_(x[lo:hi].reshape(-1))
            buf[cf * fx: cf * fx + (hi - lo) * fm].copy_(mg[lo:hi].reshape(-1))
            chunks.append(buf)
            ptrs.append(Q.host_device_ptr(buf))
        table = torch.tensor(ptrs or [0], dtype=torch.int64).cuda()
        picks = torch.randint(0, n_frames, (1 + i % 6,), generator=g).cuda()
        prev_p = torch.randint(0, n_frames, (3,), generator=g).cuda() if i % 2 else None
        prev = None if prev_p is None else (prev_p, x[prev_p.cpu()].cuda(), mg[prev_p.cpu()].cuda())
        for dst in (calls, refs):
            dst.append(dict(picks=picks, n_frames=n_frames, dev_x=x[:n_dev].cuda() if n_dev else None,
                            dev_merged=mg[:n_dev].cuda() if n_dev else None, n_dev=n_dev, chunks=table, chunk_frames=cf,
                            x_frame_elems=fx, merged_frame_elems=fm, prev=prev,
                            spa_x_out=torch.empty(picks.numel(), fx, dtype=torch.bfloat16, device="cuda"),
                            merged_out=torch.empty(picks.numel(), fm, dtype=torch.bfloat16, device="cuda"),
                            host_fetches=torch.zeros(1, dtype=torch.int64, device="cuda"), _keep=chunks))
    strip = lambda a: {k: v for k, v in a.items() if k != "_keep"}
    Q.dam_gather_multi([strip(a) for a in calls])
    for a in refs:
        Q.dam_gather_multi([strip(a)])
    torch.cuda.synchronize()
    fetched = 0
    for a, b in zip(calls, refs):
        for k in ("spa_x_out", "merged_out", "host_fetches"):
            assert equal(a[k], b[k]), k
        fetched += int(a["host_fetches"])
    assert fetched > 0


# ---- pool level --------------------------------------------------------------------------------------------------------
def pool_run(rt, tower, merger, S, rounds_n=8, method="klarge_retrieve", ts=(1, 2, 8), caps=None, grids=None, seed=0,  # noqa: F811
             temporal_method=None, **kw):
    """S streams opened over the first rounds (half at round 0, the rest at round 3) in a batched and a per-stream
    pool (BATCH_MIN_JOBS above S: one-item calls only), random clip lengths, some streams sitting rounds out; caps:
    small_device_frames per stream (cycled)"""
    from flash_vstream_b200.qwen import QwenStreamPool
    host = host_for(rt, tower, merger, method=method)
    if temporal_method is not None:
        host.visual.flash_memory.temporal_method = temporal_method
    pool, per_stream = QwenStreamPool(host, **kw), QwenStreamPool(host, **kw)
    pool.BATCH_MIN_JOBS = 2                                       # job tables from two k-means streams on
    per_stream.BATCH_MIN_JOBS = S + 1                             # every k-means stream alone
    r = random.Random(seed)
    alone = {}
    for k in range(rounds_n):
        while len(alone) < (max(1, S // 2) if k < 3 else S):
            i = len(alone)
            cap = kw.get("small_device_frames") if caps is None else caps[i % len(caps)]
            for p in (pool, per_stream):
                assert p.open(seed=1000 + i) == i
                p.state(i).small_device_frames = cap
            alone[i] = Alone(host, 1000 + i, device_frames=kw.get("device_frames"), small_device_frames=cap)
        listed = [s for s in alone if r.random() < 0.85] or [0]
        rnd = {s: clip(100 * k + s, r.choice(ts), *(grids[s % len(grids)] if grids else (8, 8))) for s in listed}
        run(pool, alone, [rnd], (S, k), others=(per_stream,))
    return pool, list(alone)


@pytest.mark.parametrize("S", [1, 2, 5, 16, 32])
def test_pool_memory_equals_streams_alone(rt, tower, merger, S):  # noqa: F811
    from flash_vstream_b200.qwen import stream_state as SS
    calls = {"kmeans": 0, "retrieve": 0, "gather": 0}               # calls with more than one job
    orig = (SS.CF.ordered_kmeans_enqueue_multi, SS.Q.klarge_retrieve_multi, SS.Q.dam_gather_multi)

    def spy(name, fn):
        def f(jobs, *a, **k):
            calls[name] += len(jobs) > 1
            return fn(jobs, *a, **k)
        return f
    SS.CF.ordered_kmeans_enqueue_multi = spy("kmeans", orig[0])
    SS.Q.klarge_retrieve_multi = spy("retrieve", orig[1])
    SS.Q.dam_gather_multi = spy("gather", orig[2])
    try:
        pool, sids = pool_run(rt, tower, merger, S, rounds_n=9 if S < 32 else 7)
    finally:
        SS.CF.ordered_kmeans_enqueue_multi, SS.Q.klarge_retrieve_multi, SS.Q.dam_gather_multi = orig
    assert any(pool.state(s).fast_steps for s in sids)
    if S >= 5:                                                    # the job tables ran, not only the one-item calls
        assert min(calls.values()) > 0, calls


@pytest.mark.parametrize("method", ["klarge_retrieve", "klarge_retrieve_cos"])
def test_pool_memory_methods_grids_and_clip_lengths(rt, tower, merger, method):  # noqa: F811
    pool_run(rt, tower, merger, 5, method=method, ts=(1, 8), grids=[(8, 8), (8, 16)], seed=3)


def test_pool_memory_fast_kmeans_and_capped_banks(rt, tower, merger):  # noqa: F811
    pool, sids = pool_run(rt, tower, merger, 4, rounds_n=8, seed=5, temporal_method="fast_kmeans_ordered", device_frames=0,
                          caps=[None, 2])
    assert any(pool.state(s).n_small_host for s in sids) and not all(pool.state(s).n_small_host for s in sids)


def test_pool_memory_duplicate_rows_redo(rt, tower, merger):  # noqa: F811
    from flash_vstream_b200.qwen import QwenStreamPool
    host = host_for(rt, tower, merger)
    pool = QwenStreamPool(host)
    pool.BATCH_MIN_JOBS = 2                                       # the redo next to streams of one job table
    alone = {pool.open(seed=s): Alone(host, s) for s in range(3)}
    rounds = [{s: clip(10 * k + s, 2) for s in alone} for k in range(4)]
    rounds.append({0: clip(91, 2), 1: clip(92, 2, repeat=True), 2: clip(93, 8)})
    rounds.append({s: clip(95 + s, 1) for s in alone})
    run(pool, alone, rounds, "redo")
    assert pool.state(1).redone_steps == 1 and pool.state(0).redone_steps == 0


def test_pool_memory_real_tower_336(rt, merger):  # noqa: F811
    """the 32-layer tower at 336 px and the default memory (CSM 60, DAM 30): 3 streams past the CSM length"""
    from flash_vstream_b200.qwen import QwenStreamPool
    from flash_vstream_b200.qwen.vision_tower import QwenVisionBlocksB200
    from tests import qwen_rt_inputs as RI
    from tests import qwen_vit_inputs as VI
    tw = QwenVisionBlocksB200(VI.state_dict(dict(depth=32, embed=1280, heads=16, seed=5), "bf16"), depth=32, heads=16,
                              dtype=torch.bfloat16)
    try:
        mg = rt.PatchMerger.from_weights({k: v.cuda() for k, v in RI.merger_weights(1280, 3584, "bf16", 7).items()})
        host = rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(rt.FlashMemory(), mg, encode_patches=tw))
        pool = QwenStreamPool(host)
        pool.BATCH_MIN_JOBS = 2
        alone = {pool.open(seed=s): Alone(host, s) for s in range(3)}
        rounds = [{s: clip(7 * k + s, 8 if k < 8 else 1, 24, 24) for s in alone if k < 8 or (k + s) % 4} for k in range(11)]
        run(pool, alone, rounds, "336")
        assert all(pool.state(s).fast_steps >= 2 for s in alone)
    finally:
        tw.close()
