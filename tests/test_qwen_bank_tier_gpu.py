"""GPU tests of the two-tier feature bank of the Qwen2-VL streaming state (DESIGN.md §3.13): fvs_qwen_dam_gather_multi
against a torch gather, streams capped at every kind of frame count equal to the uncapped stream bit for bit, the
reference goldens with every frame spilled, the real tower, checkpoints across caps, the HBM bound, reuse of the
previous DAM, and the publication."""
import os
import random
import threading
import time

import numpy as np
import pytest
import torch

from tests import qwen_rt_inputs as RI

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def rt():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    from flash_vstream_b200 import _lib
    _lib.load(build_if_missing=False)
    torch.set_grad_enabled(False)
    import flash_vstream_b200.qwen.vstream_qwen2vl_realtime as m
    return m


def bits(t):
    t = t.cpu()
    return t.view(torch.int16) if t.dtype in (torch.bfloat16, torch.float16) else t


def same(a, b):
    if a is None or b is None:
        return a is None and b is None
    if not torch.is_tensor(a):
        return a == b
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(bits(a), bits(b))


# ------------------------------------------------------------------------------------------------ 1. the kernel
def _host_tier(x, m, n_dev, F):
    """pinned chunks of frames [n_dev, n) laid out as the state lays them out, and the device table of their pointers"""
    from flash_vstream_b200.qwen import ops as Q
    n, fx, fm = x.shape[0], x[0].numel(), m[0].numel()
    chunks, ptrs = [], []
    for c0 in range(n_dev, n, F):
        cnt = min(F, n - c0)
        buf = torch.zeros(F * (fx + fm), dtype=x.dtype, pin_memory=True)
        buf[: cnt * fx].copy_(x[c0: c0 + cnt].reshape(-1))
        buf[F * fx: F * fx + cnt * fm].copy_(m[c0: c0 + cnt].reshape(-1))
        chunks.append(buf)
        ptrs.append(Q.host_device_ptr(buf))
    table = torch.tensor(ptrs or [0], dtype=torch.int64).cuda()
    return chunks, table


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
@pytest.mark.parametrize("grid, D, Dm", [((4, 4), 256, 512), ((24, 24), 1280, 3584)])
def test_dam_gather_table_matches_torch(rt, dtype, grid, D, Dm):
    from flash_vstream_b200.qwen import ops as Q
    g = torch.Generator().manual_seed(5)
    n, F = 11, 4
    hw, pm = grid[0] * grid[1], grid[0] * grid[1] // 4
    x = torch.randn(n, hw, D, generator=g).to(dtype)
    m = torch.randn(n, pm, Dm, generator=g).to(dtype)
    xd, md = x.cuda(), m.cuda()
    pick_sets = {
        "dups_and_current_clip": [10, 3, 3, 0, 9, 10, 5, 1, 8, 8],
        "all_prev": [2, 7, 4],
        "none_prev": [0, 1, 5, 6, 9, 10],
        "mixed": [4, 10, 2, 2, 6],
    }
    prev_picks = [7, 2, 4, 4]
    for n_dev in (0, 1, F - 1, F, n):
        chunks, table = _host_tier(x, m, n_dev, F)
        for name, picks in pick_sets.items():
            for use_prev in (False, True):
                p = torch.tensor(picks, dtype=torch.int64).cuda()
                pp = torch.tensor(prev_picks, dtype=torch.int64).cuda()
                prev = (pp, xd[pp], md[pp].reshape(-1, Dm)) if use_prev else None
                cnt = torch.zeros(1, dtype=torch.int64, device="cuda")
                ox = torch.full((len(picks), hw, D), 7, dtype=dtype, device="cuda")
                om = torch.full((len(picks), pm, Dm), 7, dtype=dtype, device="cuda")
                bank = dict(picks=p, n_frames=n, dev_x=xd[:n_dev] if n_dev else None, n_dev=n_dev,
                            chunks=table if n_dev < n else None, chunk_frames=F, x_frame_elems=hw * D,
                            merged_frame_elems=pm * Dm)
                Q.dam_gather_multi([dict(bank, dev_merged=md[:n_dev] if n_dev else None, prev=prev, spa_x_out=ox,
                                         merged_out=om, host_fetches=cnt)])
                assert same(ox, xd[p]) and same(om, md[p]), (n_dev, name, use_prev)
                want = sum(1 for v in picks if v >= n_dev and not (use_prev and v in prev_picks))
                assert int(cnt.item()) == want, (n_dev, name, use_prev)
                ox2 = torch.empty_like(ox)              # one output alone (the restore rebuilds spa_x only)
                Q.dam_gather_multi([dict(bank, dev_merged=None, spa_x_out=ox2)])
                assert same(ox2, xd[p])
    torch.cuda.synchronize()


# ------------------------------------------------------------------------------------------------ 2. stream equivalence
T_GRID, S_GRID, D, DM = (4, 4), (2, 2), 256, 512


def _features(sizes, seed=3, repeat_at=7):
    """seeded (x, small) per clip; clip `repeat_at` repeats its first frame (the duplicate-rows redo path)"""
    g = torch.Generator().manual_seed(seed)
    scenes = torch.randn(6, S_GRID[0] * S_GRID[1], D, generator=g)
    out, f = [], 0
    for k, t in enumerate(sizes):
        small = torch.stack([scenes[(f + i) // 7 % 6] + 0.5 * torch.randn(4, D, generator=g) for i in range(t)])
        x = small.repeat_interleave(4, dim=1) + 0.1 * torch.randn(t, 16, D, generator=g)
        if k == repeat_at and t > 1:
            small[1], x[1] = small[0], x[0]
        out.append((x.reshape(-1, D).bfloat16().cuda(), small.reshape(-1, D).bfloat16().cuda()))
        f += t
    return out


def _clip_sizes(n_patches, seed=11):
    r = random.Random(seed)
    sizes = []
    while sum(sizes) < n_patches:
        sizes.append(r.choice([1, 2, 3]))
    sizes[7] = 3                                          # the repeated-frame clip
    return sizes


def _merger(rt, seed=7):
    return rt.PatchMerger.from_weights({k: v.cuda() for k, v in RI.merger_weights(D, DM, "bf16", seed).items()})


def _state(rt, SS, method, cap, merger, chunk_frames=5):
    flash = rt.FlashMemory(flash_memory_temporal_length=8, flash_memory_spatial_length=6, flash_memory_spatial_method=method)
    st = SS.QwenStreamState(flash, merger, device_frames=cap)
    st.CHUNK_BYTES = chunk_frames * (16 * D + 4 * DM) * 2          # 5 frames per host chunk
    return st


def _run_step(st, clip, k, start):
    torch.manual_seed(100 + k)
    random.seed(100 + k)
    x, small = clip
    t = x.shape[0] // 16
    st.step(x, small, t, T_GRID, S_GRID, start)


def _same_lists(a, b, tag):
    la, lb = a.as_list(), b.as_list()
    for i, (u, v) in enumerate(zip(la, lb)):
        if i == 7:
            continue
        assert same(u, v), (tag, i)
    assert same(a.video_embeds, b.video_embeds), tag


@pytest.mark.parametrize("method", ["klarge_retrieve", "klarge_retrieve_cos", "nearest", "sample"])
def test_capped_stream_equals_uncapped(rt, method):
    from flash_vstream_b200.qwen import stream_state as SS
    sizes = _clip_sizes(150)
    clips = _features(sizes)
    cum = np.cumsum([0] + sizes)
    inside = int(next(c + 1 for c, t in zip(cum, sizes) if c > 20 and t > 1))          # a cap inside a clip
    merger = _merger(rt)
    ref = _state(rt, SS, method, None, merger)
    capped = {cap: _state(rt, SS, method, cap, merger) for cap in (0, inside, 10)}    # 10: a chunk edge of 5
    for k, clip in enumerate(clips):
        _run_step(ref, clip, k, int(cum[k]))
        for cap, st in capped.items():
            _run_step(st, clip, k, int(cum[k]))
            _same_lists(ref, st, (method, cap, k))
            assert st.n_host == max(0, int(cum[k + 1]) - cap) and st.bank_x.n == min(int(cum[k + 1]), cap)
    assert ref.redone_steps >= 1 and ref.fast_steps > 0
    assert all(st.redone_steps == ref.redone_steps for st in capped.values())
    assert capped[0].as_list()[7].shape == (0, D) and capped[0].as_list()[8].tolist() == [int(cum[-1]), 4, 4]
    assert ref.host_fetch_count() == 0 and capped[0].host_fetch_count() > 0


# ------------------------------------------------------------------------------------------------ 3. reference goldens
@pytest.mark.parametrize("name", list(RI.REALTIME_CASES))
def test_goldens_with_every_frame_spilled(rt, name):
    """test_streaming_steps_parity's stream with fvs_bank_device_frames=0; the full-resolution bank through a checkpoint"""
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
        assert host.stream_state.n_host == (s + 1) * t and bank.shape[0] == 0 and bank.is_cuda
        assert tem_thw.tolist() == g[p + "_tem_thw"].tolist() and spa_thw.tolist() == g[p + "_spa_thw"].tolist()
        assert thw.tolist() == g[p + "_thw"].tolist() and tuple(shape) == tuple(embeds.shape)
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
        assert rel(embeds.cpu(), om[11]) < REL[c["dtype"]]
    pos, vis = RI.realtime_positions(c, int(g[name + "_n_vis"][0]))
    ve, new_pos = host.prepare_realtime_inference(pos.cuda(), vis.cuda())
    assert np.array_equal(new_pos.cpu().numpy(), g[name + "_final_pos"])


# ------------------------------------------------------------------------------------------------ 4. the real tower
def test_real_tower_336(rt):
    from flash_vstream_b200.qwen.vision_tower import QwenVisionBlocksB200
    from tests import qwen_vit_inputs as VI
    sd = VI.state_dict(dict(depth=4, embed=1280, heads=16, seed=5), "bf16")
    tower = QwenVisionBlocksB200(sd, depth=4, heads=16, dtype=torch.bfloat16)
    merger = rt.PatchMerger.from_weights({k: v.cuda() for k, v in RI.merger_weights(1280, 3584, "bf16", 7).items()})
    g = torch.Generator().manual_seed(1)
    clips = [torch.randn(2 * 576, 1176, generator=g).bfloat16() for _ in range(6)]
    thw = torch.tensor([[2, 24, 24]])
    hosts = {}
    for cap in (None, 3):
        host = rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(
            rt.FlashMemory(flash_memory_temporal_length=6, flash_memory_spatial_length=4), merger, encode_patches=tower))
        host.fvs_bank_device_frames = cap
        hosts[cap] = host
    for s, clip in enumerate(clips):
        for cap, host in hosts.items():
            torch.manual_seed(s)
            random.seed(s)
            host.embed_new_video_clip(clip, thw, 2 * s)
        a, b = hosts[None].video_embedding_memory, hosts[3].video_embedding_memory
        for i in range(13):
            if i != 7:
                assert same(a[i], b[i]), (s, i)
    assert hosts[3].stream_state.n_host == 2 * len(clips) - 3
    n_vis = hosts[None].video_embedding_memory[11].shape[0]
    c = dict(prefix=2, suffix=3)
    out = []
    for host in hosts.values():
        pos, vis = RI.realtime_positions(c, n_vis)
        out.append(host.prepare_realtime_inference(pos.cuda(), vis.cuda()))
    assert same(out[0][0], out[1][0]) and torch.equal(out[0][1], out[1][1])
    tower.close()


# ------------------------------------------------------------------------------------------------ 5. checkpoints
def test_checkpoints_across_caps(rt):
    from flash_vstream_b200.qwen import stream_state as SS
    sizes = _clip_sizes(120, seed=4)
    clips = _features(sizes, seed=8)
    cum = np.cumsum([0] + sizes)
    merger = _merger(rt)
    stop = 30
    runs = {cap: _state(rt, SS, "klarge_retrieve", cap, merger) for cap in (None, 13)}
    for k in range(stop):
        for st in runs.values():
            _run_step(st, clips[k], k, int(cum[k]))
    cks = {cap: st.checkpoint() for cap, st in runs.items()}
    a, b = cks[None], cks[13]
    assert a.counters == b.counters and a.config == b.config and set(a.tensors) == set(b.tensors)
    for name in a.tensors:                                 # the same stream's checkpoint, capped or not
        assert same(a.tensor(name), b.tensor(name)), name
    ref = runs[None]
    flash = ref.flash
    for src, cap in ((13, None), (None, 13), (13, 5), (13, 0)):
        st = SS.QwenStreamState.restore(cks[src], flash, merger, "cuda", device_frames=cap)
        assert st.device_frames == cap and st.bank_x.n == (int(cum[stop]) if cap is None else cap)
        twin = SS.QwenStreamState.restore(cks[None], flash, merger, "cuda")
        _same_lists(twin, st, ("restored", src, cap))
        for k in range(stop, stop + 20):
            _run_step(st, clips[k], k, int(cum[k]))
            _run_step(twin, clips[k], k, int(cum[k]))
            _same_lists(twin, st, ("continued", src, cap, k))
        if src == 13 and cap is None:                     # and the uninterrupted run
            for k in range(stop, stop + 20):
                _run_step(ref, clips[k], k, int(cum[k]))
            _same_lists(ref, st, ("uninterrupted", k))


# ------------------------------------------------------------------------------------------------ 6. HBM bound
def test_hbm_growth_is_bounded_by_the_small_bank(rt):
    """24x24 frames, 1280 / 3584 wide: capped at 0, HBM grows by the half-resolution bank alone; uncapped, by at least
    the 2.88 MB per temporal patch of the full-resolution and merged rows"""
    from flash_vstream_b200.qwen import stream_state as SS
    merger = rt.PatchMerger.from_weights({k: v.cuda() for k, v in RI.merger_weights(1280, 3584, "bf16", 7).items()})
    g = torch.Generator(device="cuda").manual_seed(2)
    n_clips, t = 20, 2
    x = [torch.randn(t * 576, 1280, device="cuda", generator=g).bfloat16() for _ in range(n_clips)]
    sm = [torch.randn(t * 144, 1280, device="cuda", generator=g).bfloat16() for _ in range(n_clips)]
    growth = {}
    for cap in (0, None):
        flash = rt.FlashMemory(flash_memory_temporal_length=8, flash_memory_spatial_length=6)
        st = SS.QwenStreamState(flash, merger, device_frames=cap)
        warm = 3
        for k in range(n_clips):
            if k == warm:
                torch.cuda.synchronize()
                m0, small0 = torch.cuda.memory_allocated(), st.bank_small.buf.numel() * 2
            torch.manual_seed(k)
            random.seed(k)
            st.step(x[k], sm[k], t, (24, 24), (12, 12), k * t)
        torch.cuda.synchronize()
        growth[cap] = (torch.cuda.memory_allocated() - m0, st.bank_small.buf.numel() * 2 - small0)
        del st
    patches = (n_clips - warm) * t
    g0, small_growth = growth[0]
    assert g0 <= small_growth + (1 << 20), growth
    assert growth[None][0] >= patches * 2_880_000 * 0.99, growth


# ------------------------------------------------------------------------------------------------ 7. reuse
def test_static_scenes_reuse_the_previous_dam(rt):
    """a stream of a few static scenes: the retrieved frames barely change from step to step, so almost every pick is
    served from the previous DAM and the host chunks are rarely read"""
    from flash_vstream_b200.qwen import stream_state as SS
    g = torch.Generator().manual_seed(6)
    scenes = torch.randn(3, 4, D, generator=g)
    merger = _merger(rt)
    flash = rt.FlashMemory(flash_memory_temporal_length=60, flash_memory_spatial_length=60)   # 30 CSM / 30 DAM frames
    st = SS.QwenStreamState(flash, merger, device_frames=0)
    steps, t = 60, 2
    for k in range(steps):
        small = torch.stack([scenes[(2 * k + i) // 25 % 3] + 0.01 * torch.randn(4, D, generator=g) for i in range(t)])
        x = small.repeat_interleave(4, dim=1) + 0.01 * torch.randn(t, 16, D, generator=g)
        torch.manual_seed(k)
        random.seed(k)
        st.step(x.reshape(-1, D).bfloat16().cuda(), small.reshape(-1, D).bfloat16().cuda(), t, T_GRID, S_GRID, k * t)
    fetched = st.host_fetch_count()
    assert 0 < fetched < 0.25 * 30 * steps, fetched


# ------------------------------------------------------------------------------------------------ 8. publication
def test_publication_is_the_same_capped_and_uncapped(rt):
    from flash_vstream_b200.qwen.serve import QwenMemoryReader, export_qwen_memory
    from tests.test_qwen_serve_gpu import H, W, check_against, grab, host_for, record, scripted_clips, step
    n_clips = 30
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
    reader = QwenMemoryReader(*export_qwen_memory(host, grid=(H, W)))
    torch.manual_seed(3)
    random.seed(3)
    stop, seen, errs = threading.Event(), [], []

    def read_loop():
        s = torch.cuda.Stream()
        try:
            with torch.cuda.stream(s):
                while not stop.is_set():
                    seen.append(grab(reader))
        except Exception as e:
            errs.append(e)

    th = threading.Thread(target=read_loop)
    th.start()
    for s in range(n_clips):
        step(host, cursor, s)
    torch.cuda.synchronize()
    time.sleep(0.05)
    stop.set()
    th.join(timeout=120)
    assert not errs, errs
    assert host.stream_state.n_host == 2 * n_clips - 5
    assert len(seen) > 5
    for got in seen + [grab(reader)]:
        check_against(records, got)
    assert grab(reader)[0] == n_clips
