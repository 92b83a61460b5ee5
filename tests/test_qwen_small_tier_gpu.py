"""GPU tests of the half-resolution host tier of the Qwen2-VL streaming state (DESIGN.md §3.13): the tiered klarge
retrieval against the all-HBM one, streams with a capped half-resolution bank equal to the uncapped stream bit for bit,
the reference goldens with both banks spilled, checkpoints across caps, the pool, the HBM bound and the publication.
Small host chunks make a few frames span several of them."""
import os
import random

import numpy as np
import pytest
import torch

from tests import qwen_rt_inputs as RI
from tests.test_qwen_bank_tier_gpu import D, S_GRID, T_GRID, _clip_sizes, _features, _merger, _run_step, same

pytestmark = pytest.mark.gpu

SMALL_BYTES = S_GRID[0] * S_GRID[1] * D * 2          # one half-resolution frame of the stream tests


@pytest.fixture(scope="module")
def rt():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    from flash_vstream_b200 import _lib
    _lib.load(build_if_missing=False)
    torch.set_grad_enabled(False)
    import flash_vstream_b200.qwen.vstream_qwen2vl_realtime as m
    return m


# ------------------------------------------------------------------------------------------------ 1. the kernel
def _tiered(bank, n_dev, F):
    """bank [t, PD] (device) as a TieredBank: rows [0, n_dev) in HBM, the rest in pinned chunks of F rows"""
    from flash_vstream_b200.qwen import ops as Q
    t = bank.shape[0]
    chunks = []
    for c0 in range(n_dev, t, F):
        buf = torch.full((F, bank.shape[1]), 3, dtype=bank.dtype, pin_memory=True)   # unused rows hold junk
        buf[: min(F, t - c0)].copy_(bank[c0: c0 + F])
        chunks.append(buf)
    tb = Q.TieredBank(bank[:n_dev] if n_dev else None, n_dev, tuple(Q.host_device_ptr(c) for c in chunks), F, t,
                      bank.dtype, bank.device)
    return tb, chunks


@pytest.mark.parametrize("PD", [2048, 144 * 1280])
@pytest.mark.parametrize("metric", ["euclidean", "cosine"])
@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_tiered_retrieval_equals_hbm(rt, dtype, metric, PD):
    from flash_vstream_b200.qwen import ops as Q
    g = torch.Generator().manual_seed(9)
    t, F, st = 11, 4, 70
    bank = torch.randn(t, PD, generator=g).to(dtype)
    bank[6] = bank[2]                                  # a tie (first index wins) across tiers
    if metric == "cosine":
        bank[9] = 0                                    # a zero row: NaN similarity, which wins
    bank = bank.cuda()
    tem_x = torch.randn(st, PD, generator=g).to(dtype).cuda()
    tem_x[3] = bank[7]
    for k in (1, 30, 64, 65):
        kidx = torch.randint(0, st, (k,), generator=g)
        kidx[0] = 3
        kidx = kidx.cuda()
        want_idx, want = Q.klarge_retrieve(tem_x, kidx, bank, want_dist=True, metric=metric)
        for n_dev in (0, 1, 5, t):
            tb, chunks = _tiered(bank, n_dev, F)
            idx, got = Q.klarge_retrieve(tem_x, kidx, tb, want_dist=True, metric=metric)
            assert torch.equal(idx, want_idx), (k, n_dev)
            assert torch.equal(got.view(torch.int32), want.view(torch.int32)), (k, n_dev)
            assert torch.equal(Q.klarge_retrieve(tem_x, kidx, tb, metric=metric), want_idx), (k, n_dev)
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ 2. stream equivalence
def _state(rt, SS, method, cap, small_cap, merger):
    flash = rt.FlashMemory(flash_memory_temporal_length=8, flash_memory_spatial_length=6, flash_memory_spatial_method=method)
    st = SS.QwenStreamState(flash, merger, device_frames=cap, small_device_frames=small_cap)
    st.CHUNK_BYTES = 5 * SMALL_BYTES                 # 5 half-resolution frames per chunk (1 full-resolution frame)
    return st


def _same_state(a, b, tag):
    """everything a step or a reader reads, bit for bit; stand-ins (items 7 / 9 of a spilled bank) are zero-row"""
    for k in ("tem_x", "tem_weights", "tem_timestamp", "spa_positions", "spa_x", "video_embeds"):
        assert same(getattr(a, k), getattr(b, k)), (tag, k)
    la, lb = a.as_list(), b.as_list()
    for i, (u, v) in enumerate(zip(la, lb)):
        spilled = {7: a.n_host or b.n_host, 9: a.n_small_host or b.n_small_host}.get(i, 0)
        if spilled:
            for st, item in ((a, u), (b, v)):
                if (st.n_host if i == 7 else st.n_small_host):
                    assert item.shape == (0, D) and item.is_cuda, (tag, i)
            continue
        assert same(u, v), (tag, i)


@pytest.mark.parametrize("device_frames", [None, 0])
@pytest.mark.parametrize("method", ["klarge_retrieve", "klarge_retrieve_cos", "nearest"])
def test_capped_small_bank_equals_uncapped(rt, method, device_frames):
    from flash_vstream_b200.qwen import stream_state as SS
    sizes = _clip_sizes(40, seed=5)
    clips = _features(sizes, seed=4)
    cum = np.cumsum([0] + sizes)
    merger = _merger(rt)
    ref = _state(rt, SS, method, None, None, merger)
    capped = {c: _state(rt, SS, method, device_frames, c, merger) for c in (0, 3)}
    for k, clip in enumerate(clips):
        _run_step(ref, clip, k, int(cum[k]))
        n = int(cum[k + 1])
        for c, st in capped.items():
            _run_step(st, clip, k, int(cum[k]))
            _same_state(ref, st, (method, device_frames, c, k))
            assert st.bank_small.n == min(n, c) and st.n_small_host == max(0, n - c)
            assert len(st.small_chunks) == -(-max(0, n - c) // 5)
    assert len(clips) >= 12 and len(capped[0].small_chunks) >= 4
    assert ref.redone_steps >= 1 and all(st.redone_steps == ref.redone_steps for st in capped.values())
    assert capped[0].as_list()[9].shape == (0, D) and capped[0].as_list()[10].tolist() == [int(cum[-1]), 2, 2]


# ------------------------------------------------------------------------------------------------ 3. reference goldens
@pytest.mark.parametrize("name", list(RI.REALTIME_CASES))
def test_goldens_with_both_banks_spilled(rt, name):
    """test_streaming_steps_parity's stream with fvs_bank_device_frames = fvs_bank_small_device_frames = 0; both banks
    through a checkpoint"""
    from oracle import qwen_oracle as QO
    from tests.test_qwen_rt_oracle_golden import G, REL, rel, weight_order
    c = RI.REALTIME_CASES[name]
    g = np.load(os.path.join(G, "qwen_realtime.npz"))
    dt = RI.DT[c["dtype"]]
    w = RI.merger_weights(c["xdim"], c["out_dim"], c["dtype"], c["seed"])
    clips = RI.realtime_clips(c)
    t, h, wd = c["t_clip"], c["h"], c["w"]
    cur = {"i": 0}

    def encode(patch_rows, total_grid_thw):
        x, small = clips[cur["i"]]
        return torch.cat([x, small]).cuda()

    flash = rt.FlashMemory(flash_memory_temporal_length=c["temporal_length"], flash_memory_spatial_length=c["spatial_length"])
    host = rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(
        flash, rt.PatchMerger.from_weights({k: v.cuda() for k, v in w.items()}), encode_patches=encode, dtype=dt))
    host.fvs_bank_device_frames = 0
    host.fvs_bank_small_device_frames = 0
    orc = QO.RealtimeOracle(QO.FlashMemoryOracle(c["temporal_length"], c["spatial_length"]), w)
    for s in range(c["n_steps"]):
        cur["i"] = s
        p = f"{name}_s{s}"
        n = int(g[p + "_n_sorts"][0])
        draws = dict(init_idx=g[p + "_init"], refill_idx=g[p + "_refill"], ts_order=g[p + "_sort0"] if n == 2 else None,
                     weight_order=weight_order(g, p))
        host.embed_new_video_clip(torch.zeros(t * h * wd, 1176), torch.tensor([[t, h, wd]]), s * t, draws=draws)
        (tem_x, tem_thw, tem_w, tem_ts, spa_x, spa_thw, spa_pos, bank, thw, small_bank, small_thw, embeds,
         shape) = host.video_embedding_memory
        st = host.stream_state
        assert st.n_host == st.n_small_host == (s + 1) * t and st.bank_small.n == 0
        assert bank.shape[0] == 0 and small_bank.shape[0] == 0 and small_bank.is_cuda
        assert tem_thw.tolist() == g[p + "_tem_thw"].tolist() and spa_thw.tolist() == g[p + "_spa_thw"].tolist()
        assert thw.tolist() == g[p + "_thw"].tolist() and small_thw.tolist() == [(s + 1) * t, h // 2, wd // 2]
        assert tuple(shape) == tuple(embeds.shape)
        assert np.array_equal(spa_pos.cpu().numpy(), g[p + "_spa_pos"])
        assert np.array_equal(tem_ts.float().cpu().numpy(), g[p + "_tem_ts"])
        assert rel(embeds.cpu(), RI.from_bits(g[p + "_embeds"], dt)) < REL[c["dtype"]]
        x, small = clips[s]
        om = orc.embed_new_video_clip(x, [t, h, wd], small, [t, h // 2, wd // 2], s * t, init_idx=g[p + "_init"],
                                      refill_idx=g[p + "_refill"], order=weight_order(g, p))
        assert torch.equal(tem_x.cpu().view(torch.int16), om[0].view(torch.int16))
        assert torch.equal(spa_x.reshape(-1, c["xdim"]).cpu().view(torch.int16), om[4].reshape(-1, c["xdim"]).view(torch.int16))
        ck = host.save_video_stream()
        assert torch.equal(ck.tensor("bank_x").reshape(-1, c["xdim"]).view(torch.int16), om[7].view(torch.int16))
        assert torch.equal(ck.tensor("bank_small").reshape(-1, c["xdim"]).view(torch.int16), om[9].view(torch.int16))
        assert rel(embeds.cpu(), om[11]) < REL[c["dtype"]]
    pos, vis = RI.realtime_positions(c, int(g[name + "_n_vis"][0]))
    ve, new_pos = host.prepare_realtime_inference(pos.cuda(), vis.cuda())
    assert np.array_equal(new_pos.cpu().numpy(), g[name + "_final_pos"])


# ------------------------------------------------------------------------------------------------ 4. checkpoints
def test_checkpoints_across_small_caps(rt, monkeypatch):
    from flash_vstream_b200.qwen import stream_state as SS
    # restored states place their rows with it too: a state's chunk size must not change once frames have spilled
    monkeypatch.setattr(SS.QwenStreamState, "CHUNK_BYTES", 5 * SMALL_BYTES)
    sizes = _clip_sizes(80, seed=4)
    clips = _features(sizes, seed=8)
    cum = np.cumsum([0] + sizes)
    merger = _merger(rt)
    stop = 20
    runs = {c: _state(rt, SS, "klarge_retrieve", None, c, merger) for c in (None, 7)}
    for k in range(stop):
        for st in runs.values():
            _run_step(st, clips[k], k, int(cum[k]))
    assert runs[7].n_small_host > 10
    cks = {c: st.checkpoint() for c, st in runs.items()}
    a, b = cks[None], cks[7]
    assert a.counters == b.counters and a.config == b.config and set(a.tensors) == set(b.tensors)
    for name in a.tensors:                                 # the same stream's checkpoint, capped or not
        assert same(a.tensor(name), b.tensor(name)), name
    ref = runs[None]
    for src, cap in ((None, None), (None, 7), (7, None), (7, 7), (7, 0)):
        st = SS.QwenStreamState.restore(cks[src], ref.flash, merger, "cuda", small_device_frames=cap)
        n = int(cum[stop])
        assert st.small_device_frames == cap and st.bank_small.n == (n if cap is None else cap)
        assert st.n_small_host == (0 if cap is None else n - cap) and len(st.small_chunks) == -(-st.n_small_host // 5)
        twin = SS.QwenStreamState.restore(cks[None], ref.flash, merger, "cuda")
        _same_state(twin, st, ("restored", src, cap))
        for k in range(stop, stop + 15):
            _run_step(st, clips[k], k, int(cum[k]))
            _run_step(twin, clips[k], k, int(cum[k]))
            _same_state(twin, st, ("continued", src, cap, k))
        if src == 7 and cap is None:                       # and the uninterrupted run
            for k in range(stop, stop + 15):
                _run_step(ref, clips[k], k, int(cum[k]))
            _same_state(ref, st, ("uninterrupted", k))


# ------------------------------------------------------------------------------------------------ 5. the pool
def test_pool_with_both_caps_equals_uncapped_streams(rt):
    from flash_vstream_b200.qwen import QwenStreamPool
    from flash_vstream_b200.qwen.vision_tower import QwenVisionBlocksB200
    from tests import qwen_vit_inputs as VI
    from tests.test_qwen_multistream_gpu import Alone, clip, host_for, same_rng
    Dm = 1280
    tower = QwenVisionBlocksB200(VI.state_dict(dict(depth=2, embed=Dm, heads=16, seed=5), "bf16"), depth=2, heads=16,
                                 dtype=torch.bfloat16)
    merger = rt.PatchMerger.from_weights({k: v.cuda() for k, v in RI.merger_weights(Dm, 512, "bf16", 7).items()})
    try:
        host = host_for(rt, tower, merger)
        pool = QwenStreamPool(host, device_frames=0, small_device_frames=0)
        sids = [pool.open(seed=s) for s in range(3)]
        alone = {s: Alone(host, s) for s in range(3)}
        for k in range(10):
            rnd = {s: clip(10 * k + s, (1, 2, 8)[(k + s) % 3]) for s in range(3) if (k + s) % 4}
            pool.step({sids[s]: c for s, c in rnd.items()})
            for s, c in rnd.items():
                alone[s].step(c)
            for s in range(3):
                a, b = pool.state(sids[s]), alone[s].st
                assert a.small_device_frames == 0 and a.bank_small.n == 0 and a.n_small_host == a.n_frames
                assert a.n_frames == b.n_frames and same_rng(a.rng, b.rng), (k, s)
                if a.n_frames == 0:
                    continue
                for i, (u, v) in enumerate(zip(pool.as_list(sids[s]), b.as_list())):
                    assert i in (7, 9) or same(u, v), (k, s, i)
                assert same(a.video_embeds, b.video_embeds) and same(a.spa_positions, b.spa_positions), (k, s)
        back = pool.open(checkpoint=pool.checkpoint(sids[1]))          # a pool checkpoint of a spilled stream
        assert pool.state(back).n_small_host == pool.state(sids[1]).n_frames
    finally:
        tower.close()


# ------------------------------------------------------------------------------------------------ 6. HBM bound
def test_hbm_no_longer_grows_with_both_caps(rt):
    from flash_vstream_b200.qwen import stream_state as SS
    merger = _merger(rt)
    cap = 6
    st = _state(rt, SS, "klarge_retrieve", cap, cap, merger)
    g = torch.Generator(device="cuda").manual_seed(2)

    def caps():
        return tuple(rb.buf.shape[0] for rb in (st.bank_x, st.bank_small, st.bank_merged))

    marks = {}
    for k in range(cap + 200):
        x = torch.randn(16, D, device="cuda", generator=g).bfloat16()
        small = torch.randn(4, D, device="cuda", generator=g).bfloat16()
        torch.manual_seed(k)
        random.seed(k)
        st.step(x, small, 1, T_GRID, S_GRID, k)
        if st.n_frames in (cap + 1, cap + 200):
            torch.cuda.synchronize()
            marks[st.n_frames] = (caps(), torch.cuda.memory_allocated())
    (c1, m1), (c2, m2) = marks[cap + 1], marks[cap + 200]
    assert c1 == c2 and max(c1) <= 2 * cap, marks
    assert st.n_host == st.n_small_host == 200
    assert m2 - m1 < 64 * SMALL_BYTES, marks               # no bank grows in HBM (200 half-resolution frames: 400 KB)


# ------------------------------------------------------------------------------------------------ 7. publication
def test_publication_is_the_same_with_both_caps(rt):
    from flash_vstream_b200.qwen.serve import QwenMemoryReader, export_qwen_memory
    from tests.test_qwen_serve_gpu import H, W, check_against, grab, host_for, record, scripted_clips, step
    n_clips = 20
    clips = scripted_clips(n_clips, seed=21)
    ref, rc = host_for(rt, clips)
    torch.manual_seed(3)
    random.seed(3)
    records = {}
    for s in range(n_clips):
        step(ref, rc, s)
        records[s + 1] = record(ref)
    host, cursor = host_for(rt, clips)
    host.fvs_bank_device_frames = 5
    host.fvs_bank_small_device_frames = 3
    reader = QwenMemoryReader(*export_qwen_memory(host, grid=(H, W)))
    torch.manual_seed(3)
    random.seed(3)
    for s in range(n_clips):
        step(host, cursor, s)
        check_against(records, grab(reader))
    assert host.stream_state.n_small_host == host.stream_state.n_frames - 3 > 0
    assert grab(reader)[0] == n_clips
    host.fvs_bank_small_device_frames = 4                 # mid-stream: refused before anything runs
    with pytest.raises(ValueError, match="fvs_bank_small_device_frames changed from 3 to 4"):
        step(host, cursor, n_clips)
    assert host.stream_state.steps == n_clips
