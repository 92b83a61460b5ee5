"""GPU tests of the batched streaming step (fvs_stream_step_multi / ops.stream_step_many / multistream.StreamPool): every
stream of a batch ends bit-identical to the same stream stepped alone through the single-stream path, whatever the mix of
stream positions and clip lengths, the input kind, or the number of consolidation launches; refused batches move nothing;
each stream draws from its own generators."""
import ctypes as C
import random

import numpy as np
import pytest
import torch

from oracle import fvs_oracle as O
from tests import golden_inputs as GI
from tests.test_gpu_parity import bits, cu, fvs, make_model  # noqa: F401  (fvs is a fixture)
from tests.test_oracle_golden import ulp_diff_f16
from tests.test_stream_step_gpu import small_tower

pytestmark = pytest.mark.gpu


def draws_for(bank, t, seed):
    """explicit draws for a step of t frames on `bank` (None when the step runs no k-means)"""
    if not bank.needs_draws(t):
        return None
    return tuple(cu(d) for d in GI.kmeans_draws(bank.working_rows(t), bank.cfg.long_len, seed))


def host_state(bank):
    b = bank.bank
    return (b.n_frames, b.n_long, b.n_tur, b.n_cur, b.step)


def assert_same_stream(pool_bank, model, tag):
    """bank of a pool stream == the single-stream model's bank: state, buffer length, prefix and step diagnostics"""
    ref = model._fvs_bank
    for x, y, name in zip(pool_bank.state()[:3], model.video_embedding_memory[:3], ("cur", "long", "tur")):
        assert x.shape == y.shape and np.array_equal(bits(x), bits(y)), (tag, name)
    assert pool_bank.bank.n_frames == model.video_embedding_memory[3].shape[0], tag
    assert host_state(pool_bank) == host_state(ref), tag
    assert np.array_equal(bits(pool_bank.prefix()), bits(model.memory_prefix())), (tag, "prefix")
    assert torch.equal(pool_bank.header, ref.header), (tag, "header")
    la, ia, ka, _ = pool_bank.info()
    lb, ib, kb, _ = ref.info()
    assert torch.equal(ia[:4], ib[:4]), (tag, "info", ia[:4].tolist(), ib[:4].tolist())
    if int(ia[3]):
        assert torch.equal(la, lb), (tag, "labels")
    kl = pool_bank.bank.n_cur - min(pool_bank.cfg.cur_len, pool_bank.bank.n_frames)   # key frames of the last step
    assert torch.equal(ka[:max(kl, 0)], kb[:max(kl, 0)]), (tag, "key_idx")


def schedule_mixed(rounds=40):
    """sid -> {round: frames}: single frames, long clips, a late joiner, a first clip across the 25-slot warm-up, gaps"""
    long_clips = [3] + [7] * (rounds - 1)
    return {
        "ones": {r: 1 for r in range(rounds)},
        "long": {r: long_clips[r] for r in range(rounds)},
        "late": {r: 1 for r in range(10, rounds)},
        "cross": {r: (26 if r == 0 else 1) for r in range(rounds)},
        "gaps": {r: (5, 32, 1, 2)[r % 4] for r in range(0, rounds, 3)},
    }


def test_batch_equals_sequential_features(fvs):
    pkg, ops = fvs
    D, seed, rounds = 256, 91, 40
    sched = schedule_mixed(rounds)
    feats = {name: GI.scene_features(sum(s.values()), 576, D, seed + i, scene_len=(3, 9)) for i, (name, s) in enumerate(sched.items())}
    pool = pkg.StreamPool(make_model(D, seed, pkg), chunk_cap=32)
    sid, ref, pos = {}, {}, {name: 0 for name in sched}
    for r in range(rounds):
        clips, draws = {}, {}
        for name, s in sched.items():
            if r not in s:
                continue
            if name not in sid:
                sid[name], ref[name] = pool.open(), make_model(D, seed, pkg)
            t = s[r]
            clips[sid[name]] = feats[name][pos[name]:pos[name] + t].cuda()
            pos[name] += t
            d = draws_for(pool.bank(sid[name]), t, seed * 100 + r)
            if d is not None:
                draws[sid[name]] = d
        pool.step(clips, draws=draws)
        for name, s in sched.items():          # the single-stream path, one stream after the other, same draws
            if r in s:
                ref[name].consolidate_streaming(clips[sid[name]], draws=draws.get(sid[name]))
                assert_same_stream(pool.bank(sid[name]), ref[name], (name, r))
    assert pool.bank(sid["long"]).frames.shape[0] > 256          # the frame buffer grew on the way


def test_batch_equals_sequential_pixels(fvs):
    """pixels through the shared tower: the ViT's batch-composition invariance makes every stream equal to
    embed_video_streaming run alone; micro-batches split clips across streams"""
    pkg, ops = fvs
    cfg, tower = small_tower(pkg)
    D, seed = cfg.hidden, 33
    star = dict(compress_size=4, compress_long_memory_size=2)
    patterns = [[1, 4, 8, 8, 3, 8, 8], [8] * 7, [1] * 7, [2, 5, 7, 1, 8, 8, 8]]
    pix = [(GI.vit_pixels(cfg, sum(p), 5 + i) * 0.5).half().cuda() for i, p in enumerate(patterns)]
    pool = pkg.StreamPool(make_model(D, seed, pkg, tower=tower, **star), chunk_cap=8)
    refs = [make_model(D, seed, pkg, tower=tower, **star) for _ in patterns]
    sids = [pool.open() for _ in patterns]
    pos = [0] * len(patterns)
    lib = ops.L.load()
    for r in range(len(patterns[0])):
        clips, draws = {}, {}
        for i, p in enumerate(patterns):
            clips[sids[i]] = pix[i][pos[i]:pos[i] + p[r]].unsqueeze(0)
            d = draws_for(pool.bank(sids[i]), p[r], seed * 10 + r)
            if d is not None:
                draws[sids[i]] = d
        F = sum(p[r] for p in patterns)
        n0 = lib.fvs_launch_count()
        pool.step(clips, draws=draws)
        launches = lib.fvs_launch_count() - n0
        mb = F
        while mb > tower.engine.max_batch:
            mb = (mb + 1) // 2
        n_mb = -(-F // mb)
        assert launches == n_mb * (1 + 2 + 7 * 2 + 1) + 1, (r, launches, n_mb)   # per micro-batch: im2col, stack, tail; 1 wave
        for i, p in enumerate(patterns):
            refs[i].embed_video_streaming(clips[sids[i]], draws=draws.get(sids[i]))
            pos[i] += p[r]
            assert_same_stream(pool.bank(sids[i]), refs[i], (i, r))


def plan(ops, banks, frames, budget):
    """fvs_stream_plan for these banks stepping `frames` each: (blocks [n, 2], wave [n], waves)"""
    lib = ops.L.load()
    n = len(banks)
    jobs = (ops.L.StreamJob * n)()
    dummy = torch.zeros(1, dtype=torch.int32, device="cuda")
    for i, b in enumerate(banks):
        jobs[i].bank = C.pointer(b.bank)
        jobs[i].ntm = C.pointer(b.ntm)
        jobs[i].frames = frames
        jobs[i].init_idx = jobs[i].refill_idx = dummy.data_ptr()
        jobs[i].workspace, jobs[i].workspace_bytes = b.ws.data_ptr(), b.ws.numel()
    blocks, wave = (C.c_int32 * (2 * n))(), (C.c_int32 * n)()
    waves = lib.fvs_stream_plan(C.byref(banks[0].cfg), jobs, n, budget, blocks, wave)
    assert waves > 0, lib.fvs_last_error()
    return np.array(blocks[:]).reshape(n, 2), np.array(wave[:]), waves


def test_waves_do_not_change_bits(fvs):
    pkg, ops = fvs
    D, seed, rounds, n = 256, 61, 32, 6
    feats = [GI.scene_features(rounds, 576, D, seed + i) for i in range(n)]
    lib = ops.L.load()
    results = {}
    for max_blocks in (0, 4, 2):
        pool = pkg.StreamPool(make_model(D, seed, pkg))
        sids = [pool.open() for _ in range(n)]
        for r in range(rounds):
            banks = [pool.bank(s) for s in sids]
            draws = {s: draws_for(pool.bank(s), 1, seed * 100 + r + 7 * i) for i, s in enumerate(sids)}
            budget = max_blocks or torch.cuda.get_device_properties(0).multi_processor_count
            _, _, waves = plan(ops, banks, 1, budget)
            n0 = lib.fvs_launch_count()
            pool.step({s: feats[i][r:r + 1].cuda() for i, s in enumerate(sids)}, draws=draws, max_blocks=max_blocks)
            assert lib.fvs_launch_count() - n0 == 1 + waves, (max_blocks, r)    # one pool3 launch + one launch per wave
            if r == rounds - 1 and max_blocks:
                assert waves == {4: 3, 2: 6}[max_blocks]          # steady state: every job needs a Lloyd + an abstract block
        results[max_blocks] = [(bits(pool.prefix(s)), pool.bank(s).header.cpu(), host_state(pool.bank(s))) for s in sids]
    for mb in (4, 2):
        for a, b in zip(results[0], results[mb]):
            assert np.array_equal(a[0], b[0]) and torch.equal(a[1], b[1]) and a[2] == b[2], mb


def test_full_size_streams_vs_oracle(fvs):
    pkg, ops = fvs
    D, seed, n, rounds = 1024, 50, 8, 40
    feats = [GI.scene_features(rounds, 576, D, seed + i, scene_len=(3, 9)) for i in range(n)]
    w = GI.ntm_weights(D, 32, seed)
    ntm = tuple(w[k].numpy() for k in ("q_w", "q_b", "k_w", "k_b"))
    pool = pkg.StreamPool(make_model(D, seed, pkg))
    sids = [pool.open() for _ in range(n)]
    states = [O.StreamState() for _ in range(n)]
    for r in range(rounds):
        dn = {s: (GI.kmeans_draws(26, 25, seed * 1000 + 10 * r + i) if r >= 25 else (None, None)) for i, s in enumerate(sids)}
        pool.step({s: feats[i][r:r + 1].cuda() for i, s in enumerate(sids)},
                  draws={s: tuple(cu(d) for d in dn[s]) for s in sids if r >= 25})
        for i, s in enumerate(sids):
            states[i], _ = O.stream_step(states[i], O.spatial_pool(feats[i][r:r + 1].numpy(), 8), O.StarConfig(), ntm,
                                         init_idx=dn[s][0], refill_idx=dn[s][1])
            if r in (0, 24, 25, rounds - 1):
                cur, lng, tur, buf = pool.state(s)
                st = states[i]
                assert np.array_equal(bits(cur), st.cur.view(np.int16)), (i, r)
                assert np.array_equal(bits(lng), st.long.view(np.int16)), (i, r)
                assert ulp_diff_f16(tur.cpu().numpy(), st.tur).max() <= 4, (i, r)
                assert buf.shape[0] == r + 1
    for s in sids:
        bank = pool.bank(s)
        prefix = pool.prefix(s)
        assert prefix.shape == (681, D) and prefix.data_ptr() == bank.prefix_buf.data_ptr()
        out, status = ops.bank_snapshot(bank.prefix_buf, bank.header, 8, 4)
        st = status.cpu().tolist()
        assert st[0] == st[1] == 2 * rounds and st[2:7] == [25, 25, 4, rounds, rounds], st
        assert torch.equal(out[:681], prefix)


def test_rng_contract_each_stream_owns_its_generators(fvs):
    pkg, ops = fvs
    from flash_vstream_b200 import compress_functions as CF
    D, rounds = 256, 32
    seeds = [11, 12, 13]
    feats = [GI.scene_features(rounds, 576, D, 70 + i) for i in range(2)]
    feats.append(GI.scene_features(rounds, 576, D, 72, scene_len=(1000, 1000), noise=0.0))   # identical frames: empty clusters
    pool = pkg.StreamPool(make_model(D, 5, pkg))       # (the module's own init draws from the global generator)
    torch.manual_seed(1234)
    random.seed(1234)
    g0 = (torch.get_rng_state(), torch.cuda.get_rng_state(), random.getstate())
    sids = [pool.open(seed=s) for s in seeds]
    for r in range(rounds):
        pool.step({s: feats[i][r:r + 1].cuda() for i, s in enumerate(sids)})
    torch.cuda.synchronize()
    assert torch.equal(torch.get_rng_state(), g0[0]) and torch.equal(torch.cuda.get_rng_state(), g0[1])
    assert random.getstate() == g0[2], "the pool must not touch the global generators"
    refills = []
    for i, s in enumerate(sids):                       # each stream alone on the single-stream path, seeded like open(seed)
        CF.sync_rng()
        torch.manual_seed(seeds[i])
        random.seed(seeds[i])
        model = make_model(D, 5, pkg)
        for r in range(rounds):
            model.consolidate_streaming(feats[i][r:r + 1].cuda())
            if i == 2:
                refills.append(int(model._fvs_bank.info()[1][1]))
        assert_same_stream(pool.bank(s), model, ("seed", seeds[i]))
    CF.sync_rng()
    assert max(refills) > 0, "the identical-frames stream must consume refill draws"


def test_rejected_batch_moves_nothing(fvs):
    pkg, ops = fvs
    D, seed = 256, 21
    feats = GI.scene_features(40, 576, D, seed)
    pool = pkg.StreamPool(make_model(D, seed, pkg), chunk_cap=2)
    sids = [pool.open(seed=i) for i in range(3)]
    for r in range(27):
        pool.step({s: feats[r:r + 1].cuda() for s in sids})
    banks = [pool.bank(s) for s in sids]

    def snap():
        torch.cuda.synchronize()
        return [(host_state(b), b.header.clone(), b.prefix().clone(), b.ws.clone()) for b in banks]

    def same(a, b):
        return all(x[0] == y[0] and torch.equal(x[1], y[1]) and torch.equal(x[2], y[2]) and torch.equal(x[3], y[3])
                   for x, y in zip(a, b))

    def rng_state():
        return [(st.cpu.clone(), st.cuda.clone(), st.py.getstate()) for st in (pool._streams[s].rng for s in sids)]

    before = snap()
    rng_before = rng_state()
    x1 = feats[27:28].cuda()
    d = draws_for(banks[0], 1, 5)
    lib = ops.L.load()
    n0 = lib.fvs_launch_count()
    with pytest.raises(ValueError):
        ops.stream_step_many([banks[0], banks[0]], [x1, x1], draws=[d, d])
    with pytest.raises(ValueError):
        pool.step({sids[0]: x1, sids[1]: feats[27:30].cuda()})           # 3 frames > chunk_cap 2
    with pytest.raises(ValueError):
        ops.stream_step_many(banks, [x1, x1, x1], draws=[d, d, None])
    # the library's own checks, behind the Python ones: a duplicate bank, then missing draws
    jobs = (ops.L.StreamJob * 3)()
    for i, b in enumerate([banks[0], banks[1], banks[0]]):
        jobs[i].bank, jobs[i].ntm, jobs[i].frames = C.pointer(b.bank), C.pointer(b.ntm), 1
        jobs[i].init_idx, jobs[i].refill_idx = d[0].data_ptr(), d[1].data_ptr()
        jobs[i].workspace, jobs[i].workspace_bytes = b.ws.data_ptr(), b.ws.numel()
    xs = torch.cat([x1] * 3)
    rc = lib.fvs_stream_step_multi(C.byref(banks[0].cfg), jobs, 3, None, xs.data_ptr(), ops.L.INPUT_FEATURES, None, 0, 0,
                                   ops.L.cur_stream())
    assert rc == ops.L.FVS_EINVAL and b"same bank" in lib.fvs_last_error()
    jobs[2].bank, jobs[2].workspace = C.pointer(banks[2].bank), banks[2].ws.data_ptr()
    jobs[1].init_idx = None
    rc = lib.fvs_stream_step_multi(C.byref(banks[0].cfg), jobs, 3, None, xs.data_ptr(), ops.L.INPUT_FEATURES, None, 0, 0,
                                   ops.L.cur_stream())
    assert rc == ops.L.FVS_EINVAL and b"draws" in lib.fvs_last_error()
    assert lib.fvs_launch_count() == n0, "a refused batch launches nothing"
    assert same(before, snap())
    assert all(torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and a[2] == b[2] for a, b in zip(rng_state(), rng_before))
    pool.step({s: x1 for s in sids})                                    # and the pool still steps afterwards
    assert all(b.steps == 28 for b in banks)


def test_memory_reader_on_pool_bank(fvs):
    pkg, ops = fvs
    from flash_vstream_b200 import serve
    D, seed = 256, 8
    feats = GI.scene_features(30, 576, D, seed)
    pool = pkg.StreamPool(make_model(D, seed, pkg))
    a, b = pool.open(seed=1), pool.open(seed=2)
    for r in range(30):
        pool.step({a: feats[r:r + 1].cuda(), b: feats[29 - r:30 - r].cuda()})
    for s in (a, b):
        got, meta = serve.MemoryReader(*serve.export_bank(pool.bank(s))).read()
        assert torch.equal(got, pool.prefix(s)) and meta["step"] == 30
    pool.close(a)
    c = pool.open(seed=3)
    assert pool.bank(c) is not None and pool.bank(c).steps == 0 and len(pool) == 2   # a closed bank is reused, reset


def test_unsupported_config_raises(fvs):
    pkg, ops = fvs
    with pytest.raises(NotImplementedError, match="video_sample_type"):
        pkg.StreamPool(make_model(256, 1, pkg, video_sample_type="kmeans"))
