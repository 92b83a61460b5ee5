"""CPU tests of the many-stream CSM chain (DESIGN.md §3.17): the launch plan fvs_qwen_mem_plan, the refusals of the
fvs_qwen_*_multi entry points (validated before any CUDA call, so no device is needed), and the host side of a batched
round: what QwenStreamState.complete does with each stream's read-back row (valid, empty cluster, duplicate-rows redo)
and the one round error naming the failing streams."""
import ctypes as C

import pytest
import torch

from flash_vstream_b200 import _lib as L
from flash_vstream_b200.qwen import ops as Q

FAKE = 1 << 40                      # never dereferenced: every call below is refused before it launches


@pytest.fixture(scope="module")
def lib():
    return L.load()


def job(T=61, K=60, PD=184320, base=0):
    """a fvs_qwen_mem_job whose pointers are distinct fake addresses (2^44 bytes apart per field, 2^50 per job)"""
    j = L.QwenMemJob(T=T, K=K, PD=PD, x_dtype=L.BF16, max_iter=10, tol=1e-4, out_dtype=L.BF16,
                     uniq_workspace_bytes=1 << 30, km_workspace_bytes=1 << 40)
    a = FAKE + base * (1 << 50)
    for i, (name, _) in enumerate(L.QwenMemJob._fields_):
        if _ is C.c_void_p and name != "order_in":
            setattr(j, name, a + i * (1 << 44))
    return j


def expected_groups(blocks, budget):
    groups, g, n, s = [], 0, 0, 0
    for b in blocks:
        if n and (n == L.QWEN_MEM_JOBS_PER_LAUNCH or (budget > 0 and s + b > budget)):
            g, n, s = g + 1, 0, 0
        groups.append(g)
        n, s = n + 1, s + b
    return groups


@pytest.mark.parametrize("n", [1, 2, 5, 32, 64])
@pytest.mark.parametrize("budget", [0, 1, 1500, 10000, 1 << 30])
def test_plan(lib, n, budget):
    jobs = [job(T=5 + 7 * (i % 9), K=4, PD=1024 * (1 + i % 3), base=i) for i in range(n)]
    blocks, groups, launches = Q.mem_plan(jobs, budget)
    assert blocks == [((j.T + 7) // 8) * (j.PD // 1024) for j in jobs] and min(blocks) >= 1
    assert groups == expected_groups(blocks, budget) and launches == groups[-1] + 1
    for g in range(launches):                    # at most 16 jobs, and within the budget unless a job is alone
        members = [b for b, gg in zip(blocks, groups) if gg == g]
        assert 1 <= len(members) <= L.QWEN_MEM_JOBS_PER_LAUNCH
        assert budget == 0 or len(members) == 1 or sum(members) <= budget
    if budget == 0:
        assert launches == -(-n // L.QWEN_MEM_JOBS_PER_LAUNCH)
    if budget == 1:
        assert launches == n


def test_plan_refusals(lib):
    for bad in (job(T=4097, K=4), job(T=9, K=10), job(PD=1000), job(T=0)):
        with pytest.raises(ValueError, match="fvs_qwen_mem_plan"):
            Q.mem_plan([job(), bad])
    with pytest.raises(ValueError):
        Q.mem_plan([job()], -1)


CALLS = ("fvs_qwen_unique_rows_multi", "fvs_qwen_kmeans_multi", "fvs_qwen_kmeans_finalize_multi",
         "fvs_gather_rows_cast_multi")


@pytest.mark.parametrize("call", CALLS)
def test_refusals_launch_nothing(lib, call):
    def fn(jobs):                                # the C entry point itself, on the default stream
        arr = jobs if isinstance(jobs, C.Array) else Q.mem_jobs(jobs)
        L.check(getattr(lib, call)(arr, len(arr), 0, None), call)
    n0 = lib.fvs_launch_count()
    with pytest.raises(ValueError, match="T <= 4096"):
        fn([job(base=0), job(T=4097, base=1)])
    with pytest.raises(ValueError, match="PD"):
        fn([job(base=0), job(PD=1536, base=1)])
    shared = job(base=1)
    for name in ("uniq_idx", "C", "sorted_idx", "out"):        # one output of each call, shared with job 0
        setattr(shared, name, getattr(job(base=0), name) + 64)
    with pytest.raises(ValueError, match="jobs 0 and 1 share an output"):
        fn([job(base=0), shared])
    nul = job(base=1)
    for name in ("uniq_idx", "labels", "flags", "out"):
        setattr(nul, name, None)
    with pytest.raises(ValueError, match="job 1: null"):
        fn([job(base=0), nul])
    small = job(base=1)
    small.uniq_workspace_bytes = small.km_workspace_bytes = 16
    if call in ("fvs_qwen_unique_rows_multi", "fvs_qwen_kmeans_multi"):
        with pytest.raises(ValueError, match="workspace too small"):
            fn([job(base=0), small])
    with pytest.raises(ValueError, match="n_jobs > 0"):
        fn(Q.mem_jobs([]))
    assert lib.fvs_launch_count() == n0


# ---- the host side of a batched round ----------------------------------------------------------------------------------
class FakeRng:
    def __init__(self):
        self.log = []

    def consume(self, T, n):
        self.log.append(("consume", T, n))

    def rewind(self, snap):
        self.log.append(("rewind", snap))


def state_with(readback, T=61, snap="s0", own_refills=True):
    from flash_vstream_b200.qwen.multistream import _Stream
    from flash_vstream_b200.qwen.stream_state import QwenStreamState

    class Flash:
        temporal_length = 60
    st = QwenStreamState(Flash(), None)
    st.rng = FakeRng()
    st.redo = []
    st._compress_sync = lambda *a: st.redo.append(a)
    st._pending = dict(cand="cand", cand_w="w", T=T, d={}, start_idx=0, t=1, snap=snap, own_refills=own_refills,
                       readback=torch.tensor(readback + [0] * (8 - len(readback)), dtype=torch.int32))
    return _Stream(None, st)


def test_complete_reads_its_own_row():
    ok = state_with([61, 4, 7, 0, 0, 0]).stream_state
    ok.complete()
    assert ok.rng.log == [("consume", 61, 7)] and ok.fast_steps == 1 and ok.steps == 1 and not ok.redo
    replay = state_with([61, 4, 7, 0, 0, 0], snap=None, own_refills=False).stream_state
    replay.complete()
    assert replay.rng.log == [] and replay.fast_steps == 1


def test_complete_redo_rewinds_only_that_stream():
    dup = state_with([59, 0, 0, 0, 0, 0]).stream_state          # duplicate rows: n_unique < T
    other = state_with([61, 9, 3, 1, 0, 0]).stream_state
    dup.complete()
    other.complete()
    assert dup.rng.log == [("rewind", "s0")] and dup.redone_steps == 1 and len(dup.redo) == 1
    assert other.rng.log == [("consume", 61, 3)] and other.redone_steps == 0 and not other.redo


def test_empty_cluster_raises_and_round_names_sids():
    from flash_vstream_b200.qwen.multistream import QwenStreamPool
    pool = QwenStreamPool.__new__(QwenStreamPool)
    pool._streams = {0: state_with([61, 1, 0, 1, 0, 0]), 1: state_with([61, 1, 0, 1, 0, 2]),
                     2: state_with([61, 1, 0, 1, 0, 0]), 3: state_with([61, 1, 0, 1, 0, 1])}
    with pytest.raises(ZeroDivisionError) as e:
        pool._complete([0, 1, 2, 3])
    assert sorted(e.value.errors) == [1, 3] and "[1, 3]" in str(e.value)
    assert pool._streams[0].stream_state.steps == 1 and pool._streams[2].stream_state.steps == 1
    assert pool._streams[1].stream_state.steps == 0


def test_retrieve_multi_refuses_host_tier_and_shared_outputs(lib):
    def rjob(base, **kw):
        a = FAKE + base * (1 << 50)
        j = L.QwenRetrieveJob(tem_x=a, klarge_idx=a + (1 << 44), bank=a + 2 * (1 << 44), k=30, t_total=100, n_dev=100,
                              PD=184320, idx_out=a + 3 * (1 << 44), dist_out=None, workspace=a + 4 * (1 << 44),
                              workspace_bytes=1 << 40)
        for k, v in kw.items():
            setattr(j, k, v)
        return j

    def call(jobs, metric=L.KLARGE_EUCLIDEAN):
        arr = (L.QwenRetrieveJob * len(jobs))(*jobs)
        L.check(lib.fvs_qwen_klarge_retrieve_multi(arr, len(arr), L.BF16, metric, None), "fvs_qwen_klarge_retrieve_multi")
    n0 = lib.fvs_launch_count()
    with pytest.raises(ValueError, match="job 1: 40 of its 100 bank rows are in host memory"):
        call([rjob(0), rjob(1, n_dev=60)], L.KLARGE_COSINE)
    with pytest.raises(ValueError, match="jobs 0 and 1 share an output"):
        call([rjob(0), rjob(1, idx_out=FAKE + 3 * (1 << 44) + 8)])
    with pytest.raises(ValueError, match="job 1: need 0 < k <= 64"):
        call([rjob(0), rjob(1, k=65)])
    with pytest.raises(ValueError, match="PD"):
        call([rjob(0), rjob(1, PD=1000)])
    with pytest.raises(ValueError, match="unknown metric"):
        call([rjob(0)], 7)
    assert lib.fvs_launch_count() == n0


def test_gather_table_refuses_shared_counters(lib):
    def gjob(base, **kw):
        a = FAKE + base * (1 << 50)
        j = L.QwenGatherJob(picks=a, n=30, n_frames=100, n_base=100, dev_x=a + (1 << 44), dev_merged=a + 2 * (1 << 44),
                            n_dev=100, x_frame_elems=576 * 1280, merged_frame_elems=144 * 512, spa_x_out=a + 3 * (1 << 44),
                            merged_out=a + 4 * (1 << 44), host_fetches=a + 5 * (1 << 44))
        for k, v in kw.items():
            setattr(j, k, v)
        return j
    n0 = lib.fvs_launch_count()
    for bad, msg in ((gjob(1, host_fetches=FAKE + 5 * (1 << 44)), "jobs 0 and 1 share an output"),
                     (gjob(1, n_dev=50), "host frames without a chunk table"), (gjob(1, n=0), "0 < n <= 65535")):
        arr = (L.QwenGatherJob * 2)(gjob(0), bad)
        with pytest.raises(ValueError, match=msg):
            L.check(lib.fvs_qwen_dam_gather_multi(arr, 2, L.BF16, None), "fvs_qwen_dam_gather_multi")
    assert lib.fvs_launch_count() == n0


# ---- the pool's job collection ----------------------------------------------------------------------------------------
class FakeState:
    """a stream whose enqueue_input asks for the k-means when `full` (else runs its pass-through), or raises"""

    def __init__(self, full, fail=False):
        self.full, self.fail, self._pending, self.n_frames = full, fail, None, 5

    def enqueue_input(self, *a, draws=None, merged=None):
        if self.fail:
            raise RuntimeError("enqueue_input failed")
        self._pending = {}
        return (None, None), (dict(me=self) if self.full else None)


def fake_pool(monkeypatch, states, min_jobs=4):
    """a pool of FakeStates whose enqueue_csm calls are recorded as ([state, ...], readbacks)"""
    from flash_vstream_b200.qwen import multistream as MS
    pool = MS.QwenStreamPool.__new__(MS.QwenStreamPool)
    pool.BATCH_MIN_JOBS = min_jobs
    pool._streams = {i: MS._Stream(None, st) for i, st in enumerate(states)}
    pool._readbacks = torch.zeros(8, 8, dtype=torch.int32)     # pinned in a real pool; large enough not to grow here
    pool.calls = []
    monkeypatch.setattr(MS, "enqueue_csm", lambda items, rb: pool.calls.append(([r["me"] for _, r in items], rb)))
    return pool


def args(n):
    return list(range(n)), [(None, 1, 8, 8)] * n, [(None, None)] * n, [None] * n, {}


def test_pool_enqueues_only_streams_past_the_csm_length(monkeypatch):
    states = [FakeState(full=f) for f in (True, False, True, True, False, True)]
    pool = fake_pool(monkeypatch, states)
    assert pool._enqueue_memory(*args(6))
    assert len(pool.calls) == 1 and pool.calls[0][0] == [states[0], states[2], states[3], states[5]]
    assert pool.calls[0][1] is pool._readbacks


def test_small_rounds_make_one_item_calls(monkeypatch):
    """under BATCH_MIN_JOBS k-means streams: one one-item call per stream, the call a stream stepped alone makes"""
    states = [FakeState(full=f) for f in (True, False, True)]
    pool = fake_pool(monkeypatch, states)
    pool._enqueue_memory(*args(3))
    assert [c[0] for c in pool.calls] == [[states[0]], [states[2]]]
    for i, (_, rb) in enumerate(pool.calls):                     # each stream its own row of the round's read-backs
        assert rb.shape == (1, 8) and rb.data_ptr() == pool._readbacks[i].data_ptr()


def test_a_failing_stream_still_enqueues_the_collected_ones(monkeypatch):
    states = [FakeState(full=True), FakeState(full=True), FakeState(full=True, fail=True), FakeState(full=True)]
    pool = fake_pool(monkeypatch, states, min_jobs=1)
    with pytest.raises(RuntimeError, match="enqueue_input failed"):
        pool._enqueue_memory(*args(4))
    assert [c[0] for c in pool.calls] == [[states[0], states[1]]]   # the streams before the failing one
