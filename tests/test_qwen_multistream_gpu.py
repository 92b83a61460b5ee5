"""GPU tests of QwenStreamPool (DESIGN.md §3.15): every pool stream, after every round, is bit-identical to the same stream
stepped alone through QwenStreamState with the same seeds — the 13-item list, video_embeds, counters and the position of
each of its generators — whatever the round's composition: 1 to 16 streams, clips of 1, 2 and 8 temporal patches, streams
filling, crossing and past the CSM length, opened mid-way or left out of a round, several camera grids, rounds split over
several tower calls, a duplicate-rows redo next to fast-path streams, refused rounds, checkpoints, capped banks and a
reader of the publication."""
import random

import pytest
import torch

from tests import qwen_rt_inputs as RI
from tests import qwen_vit_inputs as VI

pytestmark = pytest.mark.gpu
D, DM = 1280, 512


@pytest.fixture(scope="module")
def rt():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    from flash_vstream_b200 import _lib
    _lib.load(build_if_missing=False)
    torch.set_grad_enabled(False)
    import flash_vstream_b200.qwen.vstream_qwen2vl_realtime as m
    return m


@pytest.fixture(scope="module")
def tower(rt):
    from flash_vstream_b200.qwen.vision_tower import QwenVisionBlocksB200
    t = QwenVisionBlocksB200(VI.state_dict(dict(depth=2, embed=D, heads=16, seed=5), "bf16"), depth=2, heads=16,
                             dtype=torch.bfloat16)
    yield t
    t.close()


@pytest.fixture(scope="module")
def merger(rt):
    return rt.PatchMerger.from_weights({k: v.cuda() for k, v in RI.merger_weights(D, DM, "bf16", 7).items()})


def host_for(rt, tower, merger, T=8, S=6, method="klarge_retrieve"):
    flash = rt.FlashMemory(flash_memory_temporal_length=T, flash_memory_spatial_length=S, flash_memory_spatial_method=method)
    return rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(flash, merger, encode_patches=tower))


def clip(seed, t, h=8, w=8, repeat=False, device="cuda:0"):
    """patch rows [t*h*w, 1176] (bf16, device) and the grid; `repeat`: the second temporal patch repeats the first (the
    clip's half-resolution frames are then duplicate CSM rows)"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(t, h * w, 1176, generator=g)
    if repeat:
        x[1] = x[0]
    return x.reshape(-1, 1176).bfloat16().to(device), torch.tensor([[t, h, w]])


class Alone:
    """one stream stepped alone: the host's own tower pass (forward_simple_not_merge) and QwenStreamState.step"""

    def __init__(self, host, seed, device_frames=None):
        from flash_vstream_b200.draws import DrawSource
        from flash_vstream_b200.qwen.stream_state import QwenStreamState
        v = host.visual
        self.visual = v
        self.st = QwenStreamState(v.flash_memory, v.merger, device_frames=device_frames)
        self.st.rng = DrawSource(seed, "cuda")

    def step(self, c, draws=None):
        pix, thw = c
        t, h, w = (int(v) for v in thw[0])
        feats, _, _ = self.visual.forward_simple_not_merge(pix, thw)
        n = t * h * w
        self.st.step(feats[:n], feats[n: n + n // 4], t, (h, w), (h // 2, w // 2), self.st.n_frames, draws=draws)


def bits(t):
    t = t.cpu()
    return t.view(torch.int16) if t.dtype in (torch.bfloat16, torch.float16) else t


def same(a, b):
    if a is None or b is None:
        return a is None and b is None
    if not torch.is_tensor(a):
        return a == b
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(bits(a), bits(b))


def same_rng(a, b):
    a.settle()
    b.settle()
    return torch.equal(a.cpu, b.cpu) and torch.equal(a.cuda, b.cuda) and a.py.getstate() == b.py.getstate()


def check(pool, sid, alone, tag):
    a, b = pool.state(sid), alone.st
    for k in ("n_frames", "steps", "fast_steps", "redone_steps", "n_tem", "grid", "small_grid", "n_host"):
        assert getattr(a, k) == getattr(b, k), (tag, sid, k)
    assert same_rng(a.rng, b.rng), (tag, sid)
    if a.n_frames == 0:
        return
    for i, (u, v) in enumerate(zip(pool.as_list(sid), b.as_list())):
        assert same(u, v), (tag, sid, i)
    assert same(a.video_embeds, b.video_embeds) and same(a.spa_positions, b.spa_positions), (tag, sid)


def run(pool, alone, rounds, tag):
    """rounds: [{sid: clip}]; every stream of the pool is checked after every round"""
    for r, rnd in enumerate(rounds):
        pool.step(rnd)
        for sid, c in rnd.items():
            alone[sid].step(c)
        for sid in alone:
            check(pool, sid, alone[sid], (tag, r))


@pytest.mark.parametrize("S", [1, 2, 5, 16])
def test_pool_equals_streams_alone(rt, tower, merger, S):
    from flash_vstream_b200.draws import GLOBAL
    from flash_vstream_b200.qwen import QwenStreamPool
    host = host_for(rt, tower, merger)
    pool = QwenStreamPool(host)
    sids, alone = [], {}
    g0 = (torch.get_rng_state(), torch.cuda.get_rng_state(), random.getstate())
    r = random.Random(S)
    rounds = []
    for k in range(9):
        while len(sids) < (max(1, S // 2) if k < 3 else S):             # half the streams open at round 3
            sid = pool.open(seed=1000 + len(sids))
            sids.append(sid)
            alone[sid] = Alone(host, 1000 + sid)
        listed = [s for s in sids if r.random() < 0.8] or sids[:1]   # some streams sit a round out
        rounds.append({s: clip(100 * k + s, r.choice([1, 2, 8])) for s in listed})
        run(pool, alone, rounds[-1:], ("S", S, k))
    states = [pool.state(s) for s in sids]
    assert max(st.n_frames for st in states) > 2 * 4 and any(st.fast_steps for st in states)   # past T0 = 4 frames
    assert (torch.equal(g0[0], torch.get_rng_state()) and torch.equal(g0[1], torch.cuda.get_rng_state())
            and g0[2] == random.getstate() and not GLOBAL._pending)            # the global generators never moved


def test_grids_and_split_tower_calls(rt, tower, merger):
    from flash_vstream_b200.qwen import QwenStreamPool
    from flash_vstream_b200.qwen.multistream import plan_tower_calls
    host = host_for(rt, tower, merger)
    grids = [(8, 8 * k) for k in range(1, 10)]                      # 9 cameras: 18 distinct (h, w) -> 2 tower calls
    segs = [[(1, h, w), (1, h // 2, w // 2)] for h, w in grids]
    assert len(plan_tower_calls(segs, QwenStreamPool.TOWER_ROWS)) == 2
    pools = {"grids": QwenStreamPool(host), "rows": QwenStreamPool(host)}
    pools["rows"].TOWER_ROWS = 300                                   # and a row budget that splits almost every clip off
    for name, pool in pools.items():
        alone = {}
        for i in range(len(grids)):
            alone[pool.open(seed=i)] = Alone(host, i)
        rounds = [{s: clip(10 * k + s, (1, 2, 8)[(k + s) % 3], *grids[s]) for s in alone} for k in range(6)]
        rounds.insert(2, {0: clip(77, 2, *grids[0]), 3: clip(78, 1, *grids[3])})         # two grids in one round
        run(pool, alone, rounds, name)


def test_duplicate_rows_redo_next_to_fast_streams(rt, tower, merger):
    from flash_vstream_b200.qwen import QwenStreamPool
    host = host_for(rt, tower, merger)
    pool = QwenStreamPool(host)
    alone = {pool.open(seed=s): Alone(host, s) for s in range(3)}
    rounds = [{s: clip(10 * k + s, 2) for s in alone} for k in range(4)]
    rounds.append({0: clip(91, 2), 1: clip(92, 2, repeat=True), 2: clip(93, 8)})
    rounds.append({s: clip(95 + s, 1) for s in alone})
    fast0 = None
    for k, rnd in enumerate(rounds):
        if k == 4:
            fast0 = [pool.state(s).fast_steps for s in alone]
        run(pool, alone, [rnd], ("redo", k))
    assert pool.state(1).redone_steps == 1 and pool.state(1).fast_steps == fast0[1] + 1
    assert pool.state(0).fast_steps == fast0[0] + 2 and pool.state(2).redone_steps == 0


def test_refused_round_moves_nothing(rt, tower, merger):
    from flash_vstream_b200.qwen import QwenStreamPool
    host = host_for(rt, tower, merger)
    pool = QwenStreamPool(host)
    alone = {pool.open(seed=s): Alone(host, s) for s in range(3)}
    run(pool, alone, [{s: clip(s, 2) for s in alone} for _ in range(3)], "before")
    before = {s: pool.checkpoint(s) for s in alone}
    for bad in ({0: clip(5, 1), 1: clip(6, 1, 16, 8)},                         # another grid than the stream's
                {0: clip(5, 1), 2: (clip(6, 1)[0][:10], torch.tensor([[1, 8, 8]]))},   # pixels short of the grid
                {0: clip(5, 1), 2: clip(6, 1, 8, 10)}):                            # w / 2 odd: temporal_pool refuses
        with pytest.raises((ValueError, NotImplementedError)):
            pool.step(bad)
        for s in alone:
            check(pool, s, alone[s], "refused")
            assert pool.checkpoint(s).counters == before[s].counters
    run(pool, alone, [{s: clip(50 + s, 1) for s in alone}], "after")


def test_checkpoints(rt, tower, merger):
    from flash_vstream_b200.qwen import QwenStreamPool
    host = host_for(rt, tower, merger)
    pool = QwenStreamPool(host)
    alone = {pool.open(seed=s): Alone(host, s) for s in range(3)}
    run(pool, alone, [{s: clip(10 * k + s, 2) for s in alone} for k in range(4)], "pre")
    # pool -> pool, on another device when there is one
    dev = "cuda:1" if torch.cuda.device_count() > 1 else "cuda:0"
    with torch.cuda.device(dev):
        host2 = host_for(rt, tower.to(dev), rt.PatchMerger.from_weights(
            {k: v.to(dev) for k, v in RI.merger_weights(D, DM, "bf16", 7).items()}))
        host2.visual._device = torch.device(dev)
        pool2 = QwenStreamPool(host2)
        moved = pool2.open(checkpoint=pool.checkpoint(1))
    twin = pool.open(checkpoint=pool.checkpoint(1))
    for k in range(3):
        c = clip(200 + k, (1, 8, 2)[k])
        with torch.cuda.device(dev):
            pool2.step({moved: clip(200 + k, (1, 8, 2)[k], device=dev)})
        pool.step({twin: c, 1: c})
        alone[1].step(c)
        check(pool, 1, alone[1], ("twin", k))
        check(pool, twin, alone[1], ("twin", k))
        assert same(pool2.state(moved).video_embeds, alone[1].st.video_embeds), k
        assert same_rng(pool2.state(moved).rng, alone[1].st.rng)
    # pool -> single-stream host (draws from the global generators from then on) and back with seed=
    from flash_vstream_b200.draws import DrawSource
    from flash_vstream_b200.qwen.stream_state import QwenStreamState
    single = host_for(rt, tower, merger)
    single.load_video_stream(pool.checkpoint(2))
    ref = Alone(host, 5)
    ref.st = QwenStreamState.restore(pool.checkpoint(2), host.visual.flash_memory, merger, "cuda:0")
    ref.st.rng = DrawSource(5, "cuda:0")
    torch.manual_seed(5)
    random.seed(5)
    c = clip(300, 2)
    single.embed_new_video_clip(c[0], c[1], pool.state(2).n_frames)
    ref.step(c)
    for i, (u, v) in enumerate(zip(single.video_embedding_memory, ref.st.as_list())):
        assert same(u, v), ("single", i)
    back = pool.open(checkpoint=single.save_video_stream(), seed=9)
    ref.st.rng = DrawSource(9, "cuda:0")
    for k in range(3):
        c = clip(400 + k, 2)
        pool.step({back: c})
        ref.step(c)
        check(pool, back, ref, ("back", k))
    with pytest.raises(ValueError, match="seed="):
        pool.open(checkpoint=single.save_video_stream())


def test_device_frames_capped_equals_uncapped(rt, tower, merger):
    from flash_vstream_b200.qwen import QwenStreamPool
    host = host_for(rt, tower, merger)
    pools = {cap: QwenStreamPool(host, device_frames=cap) for cap in (None, 0, 5)}
    sids = {cap: [p.open(seed=s) for s in range(4)] for cap, p in pools.items()}
    alone = {s: Alone(host, s, device_frames=5) for s in range(4)}
    for k in range(8):
        rnd = {s: clip(10 * k + s, (1, 2, 8)[(k + s) % 3]) for s in range(4) if (k + s) % 4}
        for cap, p in pools.items():
            p.step({sids[cap][s]: c for s, c in rnd.items()})
        for s, c in rnd.items():
            alone[s].step(c)
        for s in range(4):
            check(pools[5], sids[5][s], alone[s], ("cap", k))
            a = pools[None].as_list(sids[None][s]) if pools[None].state(sids[None][s]).n_frames else None
            for cap in (0, 5):
                st = pools[cap].state(sids[cap][s])
                assert st.device_frames == cap and st.bank_x.n <= cap
                if a is not None:
                    for i, (u, v) in enumerate(zip(a, pools[cap].as_list(sids[cap][s]))):
                        assert i == 7 or same(u, v), (cap, k, s, i)
    assert pools[0].state(sids[0][1]).n_host > 0


def test_reader_on_a_pool_stream(rt, tower, merger):
    from flash_vstream_b200.qwen import QwenStreamPool
    from flash_vstream_b200.qwen.serve import QwenMemoryReader, export_qwen_memory
    host = host_for(rt, tower, merger)
    pool = QwenStreamPool(host)
    a, b = pool.open(seed=1), pool.open(seed=2)
    reader = QwenMemoryReader(*export_qwen_memory(pool.stream(b), grid=(8, 8)))
    assert reader.read()[1]["clips"] == 0
    for k in range(6):
        pool.step({a: clip(k, 2), b: clip(50 + k, (1, 8)[k % 2])} if k != 3 else {a: clip(k, 2)})
        ve, meta = reader.read()
        st = pool.state(b)
        assert meta["clips"] == st.steps and meta["n_frames"] == st.n_frames and meta["epoch"] == 1
        assert same(ve, st.video_embeds) and same(meta["spa_positions"], st.spa_positions)
        assert same(meta["tem_timestamp"], st.tem_timestamp.float())


def test_real_tower_336(rt, merger):
    """the 32-layer tower at 336 px and the default Flash Memory config, single-patch clips"""
    from flash_vstream_b200.qwen import QwenStreamPool
    from flash_vstream_b200.qwen.vision_tower import QwenVisionBlocksB200
    t32 = QwenVisionBlocksB200(VI.state_dict(dict(depth=32, embed=D, heads=16, seed=5), "bf16"), depth=32, heads=16,
                               dtype=torch.bfloat16)
    host = rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(rt.FlashMemory(), merger, encode_patches=t32))
    pool = QwenStreamPool(host)
    alone = {pool.open(seed=s): Alone(host, s) for s in range(3)}
    g = torch.Generator().manual_seed(0)
    scenes = [torch.randn(576, 1176, generator=g) for _ in range(6)]

    def frame(k, s):
        return ((scenes[(k + 2 * s) // 5 % 6] + 0.3 * torch.randn(576, 1176, generator=g)).bfloat16().cuda(),
                torch.tensor([[1, 24, 24]]))
    for k in range(66):                                              # past the 60 CSM frames
        rnd = {s: frame(k, s) for s in alone}
        pool.step(rnd)
        for s, c in rnd.items():
            alone[s].step(c)
        if k % 8 == 0 or k >= 60:
            for s in alone:
                check(pool, s, alone[s], ("336", k))
    assert all(pool.state(s).fast_steps >= 5 for s in alone)
    t32.close()
