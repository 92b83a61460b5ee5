"""GPU tests of the Qwen2-VL memory publication (qwen/serve.py, fvs_qwen_publish / fvs_qwen_snapshot): readers in a thread,
in another process (CUDA IPC) and on another GPU see only consistent snapshots while the writer streams; the reader's
prepare_realtime_inference equals the writer's; the reference CLI's Manager-list topology with the model pickled into a
spawned memory-manager process; publication is opt-in; refusals; pickling of the vision tower."""
import pickle
import random
import threading
import time

import pytest
import torch

from tests import qwen_rt_inputs as RI
from tests.test_qwen_rt_gpu_parity import _scripted_host, cuda_w

pytestmark = pytest.mark.gpu
T_CLIP, H, W, D = 2, 4, 4, 256
N_CLIPS = 40


@pytest.fixture(scope="module")
def rt():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    from flash_vstream_b200 import _lib
    _lib.load(build_if_missing=False)
    import flash_vstream_b200.qwen.vstream_qwen2vl_realtime as m
    return m


def scripted_clips(n, seed=9, t=T_CLIP, h=H, w=W, d=D):
    """distinct rows in every clip (so every k-means step takes the one-pass path)"""
    g = torch.Generator().manual_seed(seed)
    clips = []
    for _ in range(n):
        small = torch.randn(t, h * w // 4, d, generator=g)
        x = small.repeat_interleave(4, dim=1) + 0.1 * torch.randn(t, h * w, d, generator=g)
        clips.append((x.reshape(-1, d).bfloat16(), small.reshape(-1, d).bfloat16()))
    return clips


def host_for(rt, clips, **kw):
    # temporal_length 8 / spatial_length 4 in the reference's config units: 4 CSM and 2 DAM frames
    return _scripted_host(rt, clips, temporal_length=8, spatial_length=4, **kw)


def step(host, cursor, s, t=T_CLIP, h=H, w=W):
    cursor["i"] = s
    host.embed_new_video_clip(torch.zeros(t * h * w, 1176), torch.tensor([[t, h, w]]), s * t)


def record(host):
    st = host.stream_state
    return st.video_embeds.cpu(), st.tem_timestamp.float().cpu(), st.spa_positions.cpu()


def bits(t):
    return t.view(torch.int16) if t.dtype in (torch.bfloat16, torch.float16) else t


def same(a, b):
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(bits(a.cpu()), bits(b.cpu()))


def check_against(records, got):
    """got: (clips, embeds, ts, pos) of an accepted snapshot; records[k] = the writer's state after its k-th clip"""
    clips, ve, ts, pos = got
    if clips == 0:
        assert ve.shape[0] == 0 and ts.numel() == 0 and pos.numel() == 0
        return
    want = records[clips]
    assert same(ve, want[0]) and same(ts, want[1]) and same(pos, want[2]), clips


def grab(reader):
    ve, m = reader.read()
    return m["clips"], ve.cpu(), m["tem_timestamp"].cpu(), m["spa_positions"].cpu()


# ------------------------------------------------------------------------------------------------ 1. thread reader
def test_thread_reader_sees_consistent_snapshots(rt):
    from flash_vstream_b200.qwen.serve import QwenMemoryReader, export_qwen_memory
    clips = scripted_clips(N_CLIPS)
    host, cursor = host_for(rt, clips)
    reader = QwenMemoryReader(*export_qwen_memory(host, grid=(H, W)))
    assert reader.read()[1]["clips"] == 0                                  # exported before the first clip: empty memory
    torch.manual_seed(3)
    random.seed(3)
    stop, seen, errs = threading.Event(), [], []

    def read_loop():
        s = torch.cuda.Stream()
        try:
            with torch.cuda.stream(s):
                while not stop.is_set():
                    seen.append(grab(reader))
        except Exception as e:        # surfaced in the main thread below
            errs.append(e)

    records = {}
    th = threading.Thread(target=read_loop)
    th.start()
    for s in range(N_CLIPS):
        step(host, cursor, s)
        records[s + 1] = record(host)
    torch.cuda.synchronize()
    time.sleep(0.05)
    stop.set()
    th.join(timeout=120)
    assert not errs, errs
    counters = [g[0] for g in seen]
    assert len(seen) > 5 and counters == sorted(counters), counters[:50]
    for g in seen:
        check_against(records, g)
    final = grab(reader)
    assert final[0] == N_CLIPS
    check_against(records, final)
    assert same(final[1], host.video_embedding_memory[11])


# ------------------------------------------------------------------------------------------------ 2. IPC reader
def _ipc_writer(q, done):
    """child process: owns the host, exports once, then streams; sends its records at the end"""
    import flash_vstream_b200.qwen.vstream_qwen2vl_realtime as rt
    from flash_vstream_b200.qwen.serve import export_qwen_memory
    torch.cuda.set_device(0)
    torch.set_grad_enabled(False)
    clips = scripted_clips(N_CLIPS, seed=13)
    host, cursor = host_for(rt, clips)
    q.put(export_qwen_memory(host, grid=(H, W)))          # one CUDA tensor -> one IPC handle
    torch.manual_seed(4)
    random.seed(4)
    records = {}
    for s in range(N_CLIPS):
        step(host, cursor, s)
        records[s + 1] = record(host)
        if s % 8 == 0:
            time.sleep(0.002)
    torch.cuda.synchronize()
    q.put(records)
    done.wait(timeout=120)                                # keep the publication alive until the reader has finished


def test_cuda_ipc_reader_in_another_process(rt):
    import torch.multiprocessing as mp
    from flash_vstream_b200.qwen.serve import QwenMemoryReader
    ctx = mp.get_context("spawn")
    q, done = ctx.Queue(), ctx.Event()
    p = ctx.Process(target=_ipc_writer, args=(q, done))
    p.start()
    try:
        reader = QwenMemoryReader(*q.get(timeout=300))
        seen = []
        t_end = time.time() + 180
        while time.time() < t_end:
            seen.append(grab(reader))
            if seen[-1][0] >= N_CLIPS:
                break
        records = q.get(timeout=120)
        final = grab(reader)
        counters = [g[0] for g in seen]
        assert final[0] == N_CLIPS and counters == sorted(counters) and len(set(counters)) >= 2, counters[:50]
        for g in seen + [final]:
            check_against(records, g)
    finally:
        done.set()
        p.join(timeout=60)
    assert p.exitcode == 0


# ------------------------------------------------------------------------------------------------ 3. cross-GPU reader
@pytest.mark.skipif(torch.cuda.device_count() < 2, reason="needs 2 GPUs")
def test_cross_gpu_reader(rt):
    """writer on cuda:1, reader on cuda:0 (the reference's topology), over peer access"""
    from flash_vstream_b200.qwen.serve import QwenMemoryReader, export_qwen_memory
    if not torch.cuda.can_device_access_peer(0, 1):
        with torch.cuda.device(1):
            host, _ = host_for(rt, scripted_clips(1))
        with pytest.raises(ValueError, match="peer"):
            QwenMemoryReader(*export_qwen_memory(host, grid=(H, W)), device=0).read()
        return
    clips = scripted_clips(12, seed=17)
    torch.manual_seed(5)
    random.seed(5)
    with torch.cuda.device(1):
        host, cursor = host_for(rt, clips)
        export = export_qwen_memory(host, grid=(H, W))
    reader = QwenMemoryReader(*export, device=0)
    records, seen = {}, []
    for s in range(12):
        with torch.cuda.device(1):
            step(host, cursor, s)
            records[s + 1] = record(host)
        seen.append(grab(reader))
    for g in seen:
        check_against(records, g)
    assert seen[-1][0] == 12 and reader.embeds.device == torch.device("cuda", 0)


# ------------------------------------------------------------------------------------------------ 4. prepare_realtime_inference
@pytest.mark.parametrize("name", list(RI.REALTIME_CASES))
def test_prepare_realtime_inference_through_the_reader(rt, name):
    from flash_vstream_b200.qwen.serve import QwenMemoryReader, export_qwen_memory
    c = RI.REALTIME_CASES[name]
    dt = RI.DT[c["dtype"]]
    clips = RI.realtime_clips(c)
    cursor = {"i": 0}

    def encode(patch_rows, total_grid_thw):
        x, small = clips[cursor["i"]]
        return torch.cat([x, small]).cuda()
    w = RI.merger_weights(c["xdim"], c["out_dim"], c["dtype"], c["seed"])
    flash = rt.FlashMemory(flash_memory_temporal_length=c["temporal_length"], flash_memory_spatial_length=c["spatial_length"])
    host = rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(flash, rt.PatchMerger.from_weights(cuda_w(w)), encode_patches=encode,
                                                            dtype=dt))
    reader = QwenMemoryReader(*export_qwen_memory(host, grid=(c["h"], c["w"])))
    torch.manual_seed(6)
    random.seed(6)
    t, h, wd = c["t_clip"], c["h"], c["w"]
    for s in range(c["n_steps"]):
        cursor["i"] = s
        host.embed_new_video_clip(torch.zeros(t * h * wd, 1176), torch.tensor([[t, h, wd]]), s * t)
    pos, vis = RI.realtime_positions(c, host.video_embedding_memory[11].shape[0])
    ve_w, pos_w = host.prepare_realtime_inference(pos.clone().cuda(), vis.cuda())
    ve_r, pos_r = reader.prepare_realtime_inference(pos.clone().cuda(), vis.cuda())
    assert same(ve_r, ve_w) and ve_r.dtype == dt
    assert torch.equal(pos_r.cpu(), pos_w.cpu())


# ------------------------------------------------------------------------------------------------ 5. Manager topology
def _tower_host(rt, tower, w):
    flash = rt.FlashMemory(flash_memory_temporal_length=6, flash_memory_spatial_length=4)
    return rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(flash, rt.PatchMerger.from_weights(cuda_w(w)), encode_patches=tower))


def _manager_child(model, frame_queue, device, seed):
    """the reference's memory-manager process (cli_server_2gpu.py:197-239): the model arrives PICKLED (spawn)"""
    from flash_vstream_b200.qwen.serve import frame_memory_manager
    torch.manual_seed(seed)
    random.seed(seed)
    frame_memory_manager(model, frame_queue, device=device)


def test_reference_cli_topology_manager_list(rt):
    import torch.multiprocessing as mp
    from flash_vstream_b200.qwen.vision_tower import QwenVisionBlocksB200
    from tests import qwen_vit_inputs as VI
    sd = VI.state_dict(dict(depth=1, embed=1280, heads=16, seed=97), "bf16")
    w = RI.merger_weights(1280, 256, "bf16", 98)
    g = torch.Generator().manual_seed(3)
    clips = [{"pixel_values_videos": (torch.randn(2 * 64, 1176, generator=g) * 1.2).bfloat16(),
              "video_grid_thw": torch.tensor([[2, 8, 8]])} for _ in range(5)]
    dev, seed = torch.cuda.device_count() - 1, 11
    # in-process run: same weights, same draws
    with torch.cuda.device(dev):
        ref = _tower_host(rt, QwenVisionBlocksB200(sd, depth=1, heads=16, dtype=torch.bfloat16), w)
        torch.manual_seed(seed)
        random.seed(seed)
        for s, clip in enumerate(clips):
            ref.embed_new_video_clip(**clip, start_idx=2 * s)
        want = ref.get_video_embedding_memory_cuda_list()
    ctx = mp.get_context("spawn")
    with ctx.Manager() as manager:
        model = _tower_host(rt, QwenVisionBlocksB200(sd, depth=1, heads=16, dtype=torch.bfloat16), w)
        model.video_embedding_mem_lock = ctx.Lock()    # the CLI sets the spawn start method before it builds the model
        model.video_embedding_memory = manager.list()
        frame_queue = ctx.Queue(maxsize=10)
        p3 = ctx.Process(target=_manager_child, args=(model, frame_queue, dev, seed))
        p3.start()
        for clip in clips:
            frame_queue.put(clip)
        frame_queue.put(None)
        p3.join(timeout=300)
        assert p3.exitcode == 0
        got = model.get_video_embedding_memory_cuda_list()
        pos, vis = RI.realtime_positions(dict(prefix=3, suffix=2), got[11].shape[0])
        ve_got, pos_got = model.prepare_realtime_inference(pos.clone().cuda(), vis.cuda())
    with torch.cuda.device(dev):
        ve_want, pos_want = ref.prepare_realtime_inference(pos.clone().cuda(), vis.cuda())
    assert len(got) == 13
    for i in (0, 1, 2, 3, 4, 5, 6, 8, 10, 11):
        assert same(got[i], want[i]), i
    assert got[7].shape[0] == 0 and got[9].shape[0] == 0                   # the banks travel as empty stand-ins
    assert tuple(got[12]) == tuple(want[12])
    assert same(ve_got, ve_want) and torch.equal(pos_got.cpu(), pos_want.cpu())


# ------------------------------------------------------------------------------------------------ 6. opt-in
def test_publication_is_opt_in(rt):
    from flash_vstream_b200 import _lib as L
    from flash_vstream_b200.qwen.serve import QwenMemoryReader, export_qwen_memory
    lib = L.load()
    clips = scripted_clips(8, seed=21)
    plain, c1 = host_for(rt, clips)
    pubd, c2 = host_for(rt, clips)
    reader = QwenMemoryReader(*export_qwen_memory(pubd, grid=(H, W)))
    for s in range(6):
        counts = []
        for host, cur in ((plain, c1), (pubd, c2)):
            torch.manual_seed(100 + s)
            random.seed(100 + s)
            n0 = lib.fvs_launch_count()
            step(host, cur, s)
            counts.append(lib.fvs_launch_count() - n0)
        assert counts[1] == counts[0] + 1, counts
        for a, b in zip(plain.video_embedding_memory, pubd.video_embedding_memory):
            assert same(a, b) if torch.is_tensor(a) else tuple(a) == tuple(b)
    _, m = reader.read()
    assert m["epoch"] == 1 and m["clips"] == 6 and m["seq"] == 12
    # a clip that raises (here: a grid that differs from the stream's) publishes nothing and leaves seq even
    with pytest.raises(AssertionError):
        pubd.embed_new_video_clip(torch.zeros(T_CLIP * 8 * 8, 1176), torch.tensor([[T_CLIP, 8, 8]]), 12)
    _, m2 = reader.read()
    assert m2["seq"] == 12 and m2["clips"] == 6
    # a new stream bumps the epoch; seq keeps growing
    pubd.init_streaming()
    step(pubd, c2, 6)
    _, m3 = reader.read()
    assert m3["epoch"] == 2 and m3["clips"] == 1 and m3["seq"] == 14 and m3["n_frames"] == T_CLIP


# ------------------------------------------------------------------------------------------------ 7. full size
def test_full_size_snapshot(rt):
    """60 CSM + 30 DAM frames at 24x24 / 12x12, features 1280, merger 1280 -> 3584 bf16: a 6480 x 3584 snapshot"""
    from flash_vstream_b200.qwen.serve import QwenMemoryReader, export_qwen_memory
    t, h, w, d = 4, 24, 24, 1280
    g = torch.Generator(device="cuda").manual_seed(7)
    cursor = {"i": 0}

    def encode(patch_rows, total_grid_thw):
        return (torch.randn(t * h * w + t * h * w // 4, d, generator=g, device="cuda") * 0.5).bfloat16()
    wts = RI.merger_weights(d, 3584, "bf16", 77)
    host = rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(rt.FlashMemory(), rt.PatchMerger.from_weights(cuda_w(wts)),
                                                            encode_patches=encode))
    reader = QwenMemoryReader(*export_qwen_memory(host, grid=(h, w)))
    torch.manual_seed(8)
    random.seed(8)
    for s in range(16):                                   # 64 frames: CSM and DAM full
        cursor["i"] = s
        host.embed_new_video_clip(torch.zeros(t * h * w, 1176), torch.tensor([[t, h, w]]), s * t)
    ve, m = reader.read()
    assert ve.shape == (6480, 3584) and m["tem_thw"].tolist() == [60, 12, 12] and m["spa_thw"].tolist() == [30, 24, 24]
    assert same(ve, host.video_embedding_memory[11])
    assert torch.equal(m["spa_positions"].cpu(), host.video_embedding_memory[6].cpu())
    assert torch.equal(m["tem_timestamp"].cpu(), host.video_embedding_memory[3].float().cpu())


# ------------------------------------------------------------------------------------------------ 8. refusals
def test_refusals_launch_nothing(rt):
    from flash_vstream_b200 import _lib as L
    from flash_vstream_b200.qwen.serve import export_qwen_memory
    lib = L.load()
    n0 = lib.fvs_launch_count()
    bare = rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(rt.FlashMemory(), None, encode_patches=lambda r, g: r))
    with pytest.raises(NotImplementedError):
        export_qwen_memory(bare, grid=(4, 4))
    host, _ = host_for(rt, scripted_clips(1))
    buf, tl, sl, rows, dim, dt = export_qwen_memory(host, grid=(H, W))
    small = torch.empty(rows - 1, dim, dtype=dt, device="cuda")
    ts, pos, st = (torch.empty(tl, device="cuda"), torch.empty(sl, dtype=torch.int64, device="cuda"),
                   torch.empty(9, dtype=torch.int64, device="cuda"))
    assert lib.fvs_qwen_snapshot(buf.data_ptr(), buf.numel(), tl, sl, rows, dim, small.data_ptr(), rows - 1, ts.data_ptr(),
                                 tl, pos.data_ptr(), sl, st.data_ptr(), None) == L.FVS_EINVAL    # one row short
    assert "below the publication's capacity" in lib.fvs_last_error().decode()
    assert lib.fvs_qwen_snapshot(buf.data_ptr(), buf.numel(), tl, sl, rows, dim, None, rows, ts.data_ptr(), tl,
                                 pos.data_ptr(), sl, st.data_ptr(), None) == L.FVS_EINVAL
    assert lib.fvs_qwen_publish(None, buf.numel(), tl, sl, rows, dim, small.data_ptr(), 0, None, 0, None, 0, H, W, H // 2,
                                W // 2, 0, 0, 0, None) == L.FVS_EINVAL
    assert lib.fvs_qwen_publish(buf.data_ptr(), 63, tl, sl, rows, dim, small.data_ptr(), 0, None, 0, None, 0, H, W, H // 2,
                                W // 2, 0, 0, 0, None) == L.FVS_EINVAL
    assert lib.fvs_launch_count() == n0
    assert int(buf[:8].view(torch.int64).item()) == 0                    # the publication was never touched


# ------------------------------------------------------------------------------------------------ 9. pickling
def test_vision_blocks_pickle_round_trip(rt):
    from flash_vstream_b200.qwen.vision_tower import QwenVisionBlocksB200
    from tests import qwen_vit_inputs as VI
    sd = VI.state_dict(dict(depth=1, embed=1280, heads=16, seed=97), "bf16")
    tower = QwenVisionBlocksB200(sd, depth=1, heads=16, dtype=torch.bfloat16)
    g = torch.Generator().manual_seed(5)
    px = (torch.randn(2 * 64 + 2 * 16, 1176, generator=g) * 1.2).bfloat16().cuda()
    grids = torch.tensor([[2, 8, 8], [2, 4, 4]])
    out = tower(px, grids)
    clone = pickle.loads(pickle.dumps(tower))
    assert clone.device == tower.device and clone._h.value != tower._h.value
    assert same(clone(px, grids), out)
    assert tower.to(tower.device) is tower
    clone.close()
    tower.close()
