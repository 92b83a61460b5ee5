"""GPU tests of the pool serve loops (serve.pool_memory_manager, qwen.serve.pool_memory_manager) fed decoded uint8 frames
from producer threads: every stream ends bit-identical to its twin, the same frames through the single-stream
frame_memory_manager with the same preprocessor under the seed contract of DESIGN.md §3.9 — with streams at several
source resolutions, uneven clip counts, clip lengths and end times; a stream that ends early does not stop the others;
readers attached before the first frame read consistent snapshots while the loop runs; the LLaVA step reads the
pre-processing output in place (no concatenation)."""
import queue
import random
import threading

import pytest
import torch

from flash_vstream_b200 import preprocess as P
from flash_vstream_b200.draws import GLOBAL
from tests import preprocess_inputs as PI
from tests.test_gpu_parity import fvs, make_model  # noqa: F401  (fvs is a fixture)
from tests.test_multistream_gpu import assert_same_stream
from tests.test_preprocess_host import _clip_processor
from tests.test_stream_step_gpu import small_tower

pytestmark = pytest.mark.gpu

STAR = dict(compress_size=4, compress_long_memory_size=2)


def _schedule(n, sizes, lengths, seed):
    """per stream: its clips (uint8 [t, H, W, 3] host arrays) — uneven counts and lengths, one source size per stream"""
    r = random.Random(seed)
    out = []
    for s in range(n):
        H, W = sizes[s % len(sizes)]
        count = r.randint(2, 12) if s else 2                      # stream 0 ends early
        out.append([PI.frames(1000 * seed + 100 * s + k, (r.choice(lengths), H, W)) for k in range(count)])
    return out


def _produce(q, clips, seed):
    """a camera thread: its clips at uneven intervals, then None"""
    r = random.Random(seed)

    def run():
        for c in clips:
            threading.Event().wait(r.random() * 0.02)
            q.put(torch.from_numpy(c))
        q.put(None)
    t = threading.Thread(target=run)
    t.start()
    return t


def _serve(pool, manager, sids, schedule, readers_check, on_round=None):
    queues = {sid: queue.Queue() for sid in sids}
    stop = threading.Event()
    reads = []

    def read_loop():
        with torch.cuda.stream(torch.cuda.Stream()):
            while not stop.is_set():
                reads.append(readers_check())
    reader = threading.Thread(target=read_loop)
    reader.start()
    producers = [_produce(queues[sid], clips, 7 + i) for i, (sid, clips) in enumerate(zip(sids, schedule))]
    meters = {}
    try:
        counts = manager(pool, queues, time_meter=meters, on_round=on_round)
    finally:
        stop.set()
        reader.join()
        for p in producers:
            p.join()
    assert counts == {sid: sum(c.shape[0] for c in clips) for sid, clips in zip(sids, schedule)}
    for sid, clips in zip(sids, schedule):
        assert meters[sid]._get("memory_latency")._count == len(clips) - 1
    for t in threading.enumerate():                        # the queue threads end with their queue's None
        if t.name.startswith("pool-queue-"):
            t.join(5)
            assert not t.is_alive(), t.name
    return reads


# ---- LLaVA -----------------------------------------------------------------------------------------------------------
def test_llava_pool_serve_equals_single_stream_loops(fvs):
    pkg, ops = fvs
    from flash_vstream_b200.serve import MemoryReader, export_bank, frame_memory_manager, pool_memory_manager
    cfg, tower = small_tower(pkg)
    D, seed = cfg.hidden, 33
    proc = P.CLIPFramePreprocessor(_clip_processor(112, 112))
    schedule = _schedule(6, [(240, 320), (360, 640), (480, 270)], (1, 2, 3, 5, 8), 1)
    pool = pkg.StreamPool(make_model(D, seed, pkg, tower=tower, **STAR), chunk_cap=8, preprocess=proc)
    sids = [pool.open(seed=500 + i) for i in range(6)]
    readers = {sid: MemoryReader(*export_bank(pool.bank(sid))) for sid in sids}     # attached before the first frame
    seen = {sid: {} for sid in sids}                                                  # step -> prefix, from the writer

    def on_round(counts):
        for sid in sids:
            b = pool.bank(sid)
            seen[sid].setdefault(int(b.bank.step), b.prefix().clone())

    def read_all():
        return {sid: tuple(x.clone() if torch.is_tensor(x) else dict(x) for x in r.read()) for sid, r in readers.items()}
    on_round(None)
    reads = _serve(pool, pool_memory_manager, sids, schedule, read_all, on_round)
    assert len(reads) > 1
    for snap in reads:                                         # every snapshot is the prefix of some finished step
        for sid, (prefix, meta) in snap.items():
            want = seen[sid][meta["step"]]
            assert torch.equal(bits_t(prefix), bits_t(want)), (sid, meta["step"])
    for i, (sid, clips) in enumerate(zip(sids, schedule)):
        GLOBAL.settle()
        torch.manual_seed(500 + i)
        random.seed(500 + i)
        twin = make_model(D, seed, pkg, tower=tower, **STAR)
        q = queue.Queue()
        for c in clips:
            q.put(torch.from_numpy(c))
        q.put(None)
        assert frame_memory_manager(twin, q, preprocess=proc) == sum(c.shape[0] for c in clips)
        assert_same_stream(pool.bank(sid), twin, ("llava", sid))
    assert max(pool.bank(s).bank.n_frames for s in sids) > 25                          # past the warm-up


def bits_t(t):
    return t.cpu().view(torch.int16)


def test_llava_uint8_step_reads_the_preprocessed_pixels_in_place(fvs):
    pkg, ops = fvs
    cfg, tower = small_tower(pkg)
    proc = P.CLIPFramePreprocessor(_clip_processor(112, 112))
    pool = pkg.StreamPool(make_model(cfg.hidden, 5, pkg, tower=tower, **STAR), chunk_cap=8, preprocess=proc)
    sids = [pool.open(seed=i) for i in range(3)]
    made, read = [], []

    class Spy:
        def __init__(self, pre):
            self.pre = pre

        def many(self, clips):
            res = self.pre.many(clips)
            made.append(res[0].data_ptr())
            return res

    class Lib:
        def __init__(self, lib):
            self.lib = lib

        def __getattr__(self, name):
            fn = getattr(self.lib, name)
            if name != "fvs_stream_step_multi":
                return fn
            return lambda *a: (read.append(a[4]), fn(*a))[1]
    pool.preprocess = Spy(proc)
    for sid in sids:
        pool.bank(sid).lib = Lib(pool.bank(sid).lib)
    clips = {sid: PI.frames(sid, (t, 240 + 120 * sid, 320)) for sid, t in zip(sids, (1, 3, 2))}
    pool.step(clips)
    assert made and read == made                         # the step's input pointer is the pre-processing output
    # and the round equals the pixels path
    ref = pkg.StreamPool(make_model(cfg.hidden, 5, pkg, tower=tower, **STAR), chunk_cap=8)
    rs = [ref.open(seed=i) for i in range(3)]
    ref.step({r: proc(clips[s]).unsqueeze(0) for r, s in zip(rs, sids)})
    for r, s in zip(rs, sids):
        assert torch.equal(bits_t(ref.prefix(r)), bits_t(pool.prefix(s)))


def test_llava_round_mixing_frames_and_pixels_is_refused(fvs):
    pkg, ops = fvs
    cfg, tower = small_tower(pkg)
    proc = P.CLIPFramePreprocessor(_clip_processor(112, 112))
    pool = pkg.StreamPool(make_model(cfg.hidden, 5, pkg, tower=tower, **STAR), chunk_cap=8, preprocess=proc)
    a, b = pool.open(seed=1), pool.open(seed=2)
    f = PI.frames(3, (2, 240, 320))
    pixels = proc(f)
    lib = ops.L.load()
    torch.cuda.synchronize()
    n0 = lib.fvs_launch_count()
    with pytest.raises(ValueError, match="not a mix"):
        pool.step({a: f, b: pixels})
    bad = torch.zeros(2, 240, 320, 4, dtype=torch.uint8)          # a refused pre-processing call: nothing moves
    with pytest.raises(ValueError, match="job 1"):
        pool.step({a: f, b: bad})
    torch.cuda.synchronize()
    assert lib.fvs_launch_count() == n0
    assert pool.bank(a).bank.step == pool.bank(b).bank.step == 0
    pool.step({a: f, b: f})
    assert pool.bank(a).bank.step == pool.bank(b).bank.step == 1


# ---- Qwen2-VL --------------------------------------------------------------------------------------------------------
@pytest.fixture(scope="module")
def qwen_side():
    from tests.test_qwen_multistream_gpu import D, DM
    from tests import qwen_rt_inputs as RI
    from tests import qwen_vit_inputs as VI
    import flash_vstream_b200.qwen.vstream_qwen2vl_realtime as rt
    from flash_vstream_b200.qwen.vision_tower import QwenVisionBlocksB200
    torch.set_grad_enabled(False)
    tower = QwenVisionBlocksB200(VI.state_dict(dict(depth=2, embed=D, heads=16, seed=5), "bf16"), depth=2, heads=16,
                                 dtype=torch.bfloat16)
    merger = rt.PatchMerger.from_weights({k: v.cuda() for k, v in RI.merger_weights(D, DM, "bf16", 7).items()})

    def host():
        flash = rt.FlashMemory(flash_memory_temporal_length=8, flash_memory_spatial_length=6)
        return rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(flash, merger, encode_patches=tower))
    yield host
    tower.close()


def test_qwen_pool_serve_equals_single_stream_loops(fvs, qwen_side):
    from flash_vstream_b200.qwen import QwenStreamPool
    from flash_vstream_b200.qwen.serve import QwenMemoryReader, export_qwen_memory, frame_memory_manager, pool_memory_manager
    from tests.test_qwen_multistream_gpu import same
    # three source sizes -> grids 8x8, 8x12 and 12x4 (pool 2 resizes to multiples of 56)
    proc = P.Qwen2VLFramePreprocessor(max_pixels=112 * 168, additional_pool_size=2)
    sizes = [(100, 120), (120, 180), (200, 100)]
    schedule = _schedule(6, sizes, (1, 2, 4), 2)
    pool = QwenStreamPool(qwen_side(), preprocess=proc)
    sids = [pool.open(seed=700 + i) for i in range(6)]
    readers = {sid: QwenMemoryReader(*export_qwen_memory(pool.stream(sid), grid=proc.grid_thw(1, *sizes[i % 3])[1:]))
               for i, sid in enumerate(sids)}
    seen = {sid: {0: None} for sid in sids}

    def on_round(counts):
        for sid in sids:
            st = pool.state(sid)
            if st.n_frames:
                seen[sid].setdefault(st.steps, st.video_embeds.clone())

    def read_all():
        out = {}
        for sid, r in readers.items():
            ve, meta = r.read()
            out[sid] = (ve.clone(), meta["clips"], meta["n_frames"])
        return out
    reads = _serve(pool, pool_memory_manager, sids, schedule, read_all, on_round)
    assert len(reads) > 1
    for snap in reads:
        for sid, (ve, clips, n) in snap.items():
            want = seen[sid][clips]
            assert (ve.numel() == 0) if want is None else same(ve, want), (sid, clips)
    for i, (sid, clips) in enumerate(zip(sids, schedule)):
        GLOBAL.settle()
        torch.manual_seed(700 + i)
        random.seed(700 + i)
        twin = qwen_side()
        q = queue.Queue()
        for c in clips:
            q.put(torch.from_numpy(c))
        q.put(None)
        assert frame_memory_manager(twin, q, preprocess=proc) == sum(c.shape[0] for c in clips)
        a, b = pool.state(sid), twin.stream_state
        for k in ("n_frames", "steps", "fast_steps", "redone_steps", "n_tem", "grid", "small_grid"):
            assert getattr(a, k) == getattr(b, k), (sid, k)
        for j, (u, v) in enumerate(zip(pool.as_list(sid), b.as_list())):
            assert same(u, v), (sid, j)
        assert same(a.video_embeds, b.video_embeds) and same(a.spa_positions, b.spa_positions), sid
    assert any(pool.state(s).fast_steps for s in sids)


def test_qwen_round_mixing_frames_and_pixels_is_refused(fvs, qwen_side):
    from flash_vstream_b200.qwen import QwenStreamPool
    proc = P.Qwen2VLFramePreprocessor(max_pixels=112 * 168, additional_pool_size=2)
    pool = QwenStreamPool(qwen_side(), preprocess=proc)
    a, b = pool.open(seed=1), pool.open(seed=2)
    f = PI.frames(4, (2, 100, 120))
    x = proc(f)
    with pytest.raises(ValueError, match="not a mix"):
        pool.step({a: f, b: (x["pixel_values_videos"], x["video_grid_thw"])})
    with pytest.raises(ValueError, match="job 1"):
        pool.step({a: f, b: PI.frames(4, (3, 100, 120))})
    assert pool.state(a).n_frames == pool.state(b).n_frames == 0
    pool.step({a: f, b: f})
    assert pool.state(a).steps == pool.state(b).steps == 1
