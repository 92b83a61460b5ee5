"""GPU tests of stream checkpoints (DESIGN.md §3.12): a stream checkpointed, written to disk, loaded and restored — into a
fresh bank with another chunk_cap, under a new StreamPool sid, into another model, on another GPU — continues bit for bit
like an uninterrupted run of the same stream: every bank array, the prefix, the header words, the step diagnostics and
the draw source's generators.  Readers that have a bank mapped see the restored state under a larger even sequence
number; refused restores change nothing."""
import random

import pytest
import torch

from flash_vstream_b200 import checkpoint as CK
from tests import golden_inputs as GI
from tests.test_gpu_parity import cu, fvs, make_model  # noqa: F401  (fvs is a fixture)

pytestmark = pytest.mark.gpu

D = 256
CFG = dict(D=D, grid=24, cur_size=8, long_size=4, long_len=25, tur_len=25, cur_len=1, key_len=3, ntm_dim=32, ratio=0.2)


def ntm(seed, device="cuda"):
    w = GI.ntm_weights(D, 32, seed)
    return tuple(w[k].to(device) for k in ("q_w", "q_b", "k_w", "k_b"))


def draws_for(bank, t, seed):
    if not bank.needs_draws(t):
        return None
    return tuple(d.to(bank.device) for d in (torch.from_numpy(x) for x in GI.kmeans_draws(bank.working_rows(t), 25, seed)))


def bank_arrays(bank):
    """everything a bank holds between steps, on the host"""
    b = bank.bank
    torch.cuda.synchronize(bank.device)
    return {"counters": (b.n_tur, b.n_long, b.n_cur, b.n_frames, b.step), "header": bank.header.cpu(),
            "prefix": bank.prefix().cpu(), "long": bank.long_work[:b.n_long].cpu(), "tur": bank.tur_work[:b.n_tur].cpu(),
            "frames": bank.frames[:b.n_frames].cpu()}


def assert_same_bank(a, b, tag):
    x, y = bank_arrays(a), bank_arrays(b)
    assert x["counters"] == y["counters"], (tag, x["counters"], y["counters"])
    for k in ("prefix", "long", "tur", "frames"):
        assert torch.equal(x[k].view(torch.int16), y[k].view(torch.int16)), (tag, k)
    assert torch.equal(x["header"][1:8], y["header"][1:8]), (tag, "header")
    assert int(y["header"][0]) % 2 == 0, (tag, "seq")


def assert_same_info(a, b, tag):
    la, ia, ka, wa = a.info()
    lb, ib, kb, wb = b.info()
    assert torch.equal(ia[:4].cpu(), ib[:4].cpu()), (tag, "info")
    if int(ia[3]):
        assert torch.equal(la.cpu(), lb.cpu()) and torch.equal(wa.cpu(), wb.cpu()), (tag, "labels / wsum")
    kl = a.bank.n_cur - min(a.cfg.cur_len, a.bank.n_frames)
    assert torch.equal(ka[:max(kl, 0)].cpu(), kb[:max(kl, 0)].cpu()), (tag, "key_idx")


def continuation(ops, clips, stop, *, chunk_a, chunk_b, tmp_path, device_b="cuda", seed=3):
    """run `clips` (list of [t, 576, D] features) on bank A; checkpoint A after `stop` clips, save, load, restore into a
    fresh bank B (chunk_b, device_b); step both with the same draws and compare after every later step"""
    w = ntm(seed)
    a = ops.StreamBank(CFG, w, chunk_cap=chunk_a)
    for i, x in enumerate(clips[:stop]):
        a.step(x.cuda(), draws=draws_for(a, x.shape[0], 100 + i))
    ck = a.checkpoint()
    p = tmp_path / f"bank_{stop}.safetensors"
    ck.save(p)
    ck = CK.StreamCheckpoint.load(p)
    assert all(t.is_pinned() for t in ck.tensors.values() if t.numel())
    b = ops.StreamBank(CFG, ntm(seed, device_b), chunk_cap=chunk_b, frames_cap=8, device=device_b)
    with torch.cuda.device(b.device):
        b.restore(ck)
    assert_same_bank(a, b, ("restored", stop))
    refills = 0
    for i, x in enumerate(clips[stop:], start=stop):
        a.step(x.cuda(), draws=draws_for(a, x.shape[0], 100 + i))
        with torch.cuda.device(b.device):
            b.step(x.to(b.device), draws=draws_for(b, x.shape[0], 100 + i))
        assert_same_bank(a, b, ("step", i))
        assert_same_info(a, b, ("step", i))
        refills += int(a.info()[1][1])
    return refills


@pytest.mark.parametrize("stop", [0, 10, 30])
def test_bank_single_frames(fvs, tmp_path, stop):
    pkg, ops = fvs
    f = GI.scene_features(36, 576, D, 40, scene_len=(3, 9))
    continuation(ops, [f[i:i + 1] for i in range(36)], stop, chunk_a=1, chunk_b=4, tmp_path=tmp_path)


def test_bank_warmup_crossing(fvs, tmp_path):
    """3 + 7 + 7 + 7 = 24 frames: the checkpoint lies inside the 25-slot warm-up, the next clip crosses it"""
    pkg, ops = fvs
    sizes = [3] + [7] * 8
    f = GI.scene_features(sum(sizes), 576, D, 41, scene_len=(3, 9))
    cuts = [0]
    for s in sizes:
        cuts.append(cuts[-1] + s)
    clips = [f[cuts[i]:cuts[i + 1]] for i in range(len(sizes))]
    continuation(ops, clips, 4, chunk_a=7, chunk_b=16, tmp_path=tmp_path)


def test_bank_32_frame_clips(fvs, tmp_path):
    """a first clip longer than both memories (32 long / Turing rows before the k-means starts), into a smaller bank"""
    pkg, ops = fvs
    f = GI.scene_features(32 * 5, 576, D, 42, scene_len=(3, 9))
    clips = [f[32 * i:32 * (i + 1)] for i in range(5)]
    continuation(ops, clips, 1, chunk_a=32, chunk_b=32, tmp_path=tmp_path)
    continuation(ops, clips, 3, chunk_a=32, chunk_b=40, tmp_path=tmp_path)


def test_bank_identical_frames_consume_refills(fvs, tmp_path):
    pkg, ops = fvs
    f = GI.scene_features(40, 576, D, 43, scene_len=(1000, 1000), noise=0.0)
    refills = continuation(ops, [f[i:i + 1] for i in range(40)], 28, chunk_a=1, chunk_b=2, tmp_path=tmp_path)
    assert refills > 0, "the identical-frames stream must consume refill draws"


def test_pool_suspend_resume(fvs, tmp_path):
    """stream 2 of four is suspended for 5 rounds (checkpoint, close, the others step), then resumed under a new sid: it
    equals the same stream left idle in another pool — bank and generators — and the other streams are unaffected"""
    pkg, ops = fvs
    rounds, pause = 40, (26, 31)
    feats = [GI.scene_features(rounds, 576, D, 60 + i) for i in range(3)]
    feats.append(GI.scene_features(rounds, 576, D, 63, scene_len=(1000, 1000), noise=0.0))   # identical: refills
    feats[2], feats[3] = feats[3], feats[2]
    ref = pkg.StreamPool(make_model(D, 5, pkg))
    pool = pkg.StreamPool(make_model(D, 5, pkg))
    rs = [ref.open(seed=70 + i) for i in range(4)]
    ps = [pool.open(seed=70 + i) for i in range(4)]
    pos = [0] * 4
    ckpath = tmp_path / "s2.safetensors"
    refills = 0
    for r in range(rounds):
        active = [i for i in range(4) if not (i == 2 and pause[0] <= r < pause[1])]
        if r == pause[0]:
            pool.checkpoint(ps[2]).save(ckpath)
            pool.close(ps[2])
        if r == pause[1]:
            ps[2] = pool.open(checkpoint=CK.StreamCheckpoint.load(ckpath))
            assert ps[2] == 4
        ref.step({rs[i]: feats[i][pos[i]:pos[i] + 1].cuda() for i in active})
        pool.step({ps[i]: feats[i][pos[i]:pos[i] + 1].cuda() for i in active})
        for i in active:
            pos[i] += 1
        for i in active:
            assert_same_bank(ref.bank(rs[i]), pool.bank(ps[i]), (r, i))
            assert_same_info(ref.bank(rs[i]), pool.bank(ps[i]), (r, i))
        if 2 in active:
            refills += int(ref.bank(rs[2]).info()[1][1])
    for i in range(4):
        a, b = ref._streams[rs[i]].rng, pool._streams[ps[i]].rng
        a.settle()
        b.settle()
        assert torch.equal(a.cpu, b.cpu) and torch.equal(a.cuda, b.cuda) and a.py.getstate() == b.py.getstate(), i
    assert refills > 0, "the suspended stream's identical frames must consume refill draws"
    with pytest.raises(ValueError, match="seed="):
        pool.open(checkpoint=_model_checkpoint(pkg))


def _model_checkpoint(pkg):
    m = make_model(D, 5, pkg)
    f = GI.scene_features(3, 576, D, 1)
    for i in range(3):
        m.consolidate_streaming(f[i:i + 1].cuda())
    return m.save_video_stream()


def test_model_save_load(fvs, tmp_path):
    """single-stream model: save_video_stream at step 27, load into another model, continue with the same draws; a
    Manager-style reader sees the republished memory; a model checkpoint opens in a StreamPool with seed="""
    pkg, ops = fvs
    f = GI.scene_features(34, 576, D, 44, scene_len=(3, 9))
    a, b = make_model(D, 9, pkg), make_model(D, 9, pkg)
    for i in range(27):
        a.consolidate_streaming(f[i:i + 1].cuda(), draws=draws_for(a._fvs_bank, 1, 200 + i) if i else None)
    ck = a.save_video_stream()
    ck.save(tmp_path / "m.safetensors")
    b.load_video_stream(CK.StreamCheckpoint.load(tmp_path / "m.safetensors"))
    assert torch.equal(b.memory_prefix(), a.memory_prefix())
    assert all(torch.equal(x, y) for x, y in zip(a.video_embedding_memory, b.video_embedding_memory))
    pool = pkg.StreamPool(make_model(D, 9, pkg))
    sid = pool.open(seed=1, checkpoint=ck)
    for i in range(27, 34):
        d = draws_for(a._fvs_bank, 1, 200 + i)
        a.consolidate_streaming(f[i:i + 1].cuda(), draws=d)
        b.consolidate_streaming(f[i:i + 1].cuda(), draws=d)
        pool.step({sid: f[i:i + 1].cuda()}, draws={sid: d})
        assert_same_bank(a._fvs_bank, b._fvs_bank, i)
        assert_same_bank(a._fvs_bank, pool.bank(sid), i)
        assert all(torch.equal(x, y) for x, y in zip(a.video_embedding_memory, b.video_embedding_memory))
    op = make_model(D, 9, pkg)
    op.fvs_fused_stream = False
    op.consolidate_streaming(f[0:1].cuda())
    with pytest.raises(NotImplementedError, match="fvs_fused_stream"):
        op.save_video_stream()
    with pytest.raises(NotImplementedError, match="fvs_fused_stream"):
        op.load_video_stream(ck)


def test_reader_sees_restored_state(fvs):
    """a MemoryReader attached to a bank with a stream of its own reads the restored prefix and counters afterwards,
    under an even and larger sequence number"""
    pkg, ops = fvs
    from flash_vstream_b200 import serve
    f = GI.scene_features(30, 576, D, 45)
    x, y = ops.StreamBank(CFG, ntm(3)), ops.StreamBank(CFG, ntm(3))
    for i in range(30):
        x.step(f[i:i + 1].cuda(), draws=draws_for(x, 1, 300 + i))
    for i in range(20):
        y.step(f[29 - i:30 - i].cuda(), draws=draws_for(y, 1, 400 + i))
    reader = serve.MemoryReader(*serve.export_bank(x))
    _, before = reader.read()
    x.restore(y.checkpoint())
    got, meta = reader.read()
    assert torch.equal(got, y.prefix())
    assert (meta["step"], meta["n_frames"], meta["n_tur"], meta["n_long"], meta["n_cur"]) == (20, 20, 20, 20, 4)
    assert meta["seq"] % 2 == 0 and meta["seq"] > before["seq"], (before["seq"], meta["seq"])


def test_refusals_change_nothing(fvs):
    pkg, ops = fvs
    lib = ops.L.load()
    f = GI.scene_features(64, 576, D, 46)
    src = ops.StreamBank(CFG, ntm(3), chunk_cap=32)
    src.step(f[:32].cuda())
    ck = src.checkpoint()                                   # 32 long / Turing rows after a first 32-frame clip
    tgt = ops.StreamBank(CFG, ntm(3), chunk_cap=1)
    for i in range(5):
        tgt.step(f[i:i + 1].cuda())
    before = bank_arrays(tgt)
    n0 = lib.fvs_launch_count()
    with pytest.raises(ValueError, match="n_long 32"):
        tgt.restore(ck)
    other = ops.StreamBank({**CFG, "long_len": 24}, ntm(3), chunk_cap=32)
    with pytest.raises(ValueError, match="config.long_len"):
        other.restore(ck)
    with pytest.raises(ValueError, match="pinned"):
        tgt.restore(CK.StreamCheckpoint(ck.family, ck.config, ck.counters, {k: v.clone() for k, v in ck.tensors.items()}))
    assert lib.fvs_launch_count() == n0
    after = bank_arrays(tgt)
    assert after["counters"] == before["counters"] and torch.equal(after["header"], before["header"])


def test_another_gpu(fvs, tmp_path):
    if torch.cuda.device_count() < 2:
        pytest.skip("one CUDA device: restoring on cuda:1 needs two")
    pkg, ops = fvs
    f = GI.scene_features(34, 576, D, 47, scene_len=(3, 9))
    continuation(ops, [f[i:i + 1] for i in range(34)], 28, chunk_a=1, chunk_b=1, tmp_path=tmp_path, device_b="cuda:1")


# ------------------------------------------------------------------------------------------------ Qwen2-VL
def _qwen_host(rt, clips, w, c):
    step = {"i": 0}

    def encode(patch_rows, total_grid_thw):      # stub ViT: the seeded per-clip features
        x, small = clips[step["i"]]
        return torch.cat([x, small]).cuda()

    flash = rt.FlashMemory(flash_memory_temporal_length=c["temporal_length"], flash_memory_spatial_length=c["spatial_length"])
    merger = rt.PatchMerger.from_weights({k: v.cuda() for k, v in w.items()})
    host = rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(flash, merger, encode_patches=encode, dtype=torch.bfloat16))
    return host, step


def _qwen_clips(c, n_steps, redo_at):
    g = torch.Generator().manual_seed(c["seed"])
    t, h, w, xdim = c["t_clip"], c["h"], c["w"], c["xdim"]
    scenes = torch.randn(3, h * w // 4, xdim, generator=g)
    clips = []
    for s in range(n_steps):
        which = torch.sort(torch.randint(0, 3, (t,), generator=g)).values
        small = scenes[which] + 0.3 * torch.randn(t, h * w // 4, xdim, generator=g)
        if s == redo_at:
            small[1] = small[0]                      # duplicate rows: the single-pass k-means is redone
        x = small.repeat_interleave(4, dim=1) + 0.1 * torch.randn(t, h * w, xdim, generator=g)
        if s == redo_at:
            x[1] = x[0]
        clips.append((x.reshape(-1, xdim).bfloat16(), small.reshape(-1, xdim).bfloat16()))
    return clips


def _qwen_step(host, step, s, c):
    t, h, w = c["t_clip"], c["h"], c["w"]
    step["i"] = s
    torch.manual_seed(1000 + s)                      # the same global draws for both runs
    random.seed(1000 + s)
    host.embed_new_video_clip(torch.zeros(t * h * w, 1176), torch.tensor([[t, h, w]]), s * t)


def _same_list(a, b, tag):
    for i, (x, y) in enumerate(zip(a, b)):
        if torch.is_tensor(x):
            assert x.dtype == y.dtype and x.shape == y.shape, (tag, i)
            assert torch.equal(x.cpu().view(torch.int16) if x.element_size() == 2 else x.cpu(),
                               y.cpu().view(torch.int16) if y.element_size() == 2 else y.cpu()), (tag, i)
        else:
            assert x == y, (tag, i)


def _same_state(a, b, tag):
    for k in ("n_frames", "steps", "n_tem", "grid", "small_grid", "fast_steps", "redone_steps"):
        assert getattr(a, k) == getattr(b, k), (tag, k)
    for k in ("bank_x", "bank_small", "bank_merged"):
        ra, rb = getattr(a, k), getattr(b, k)
        assert ra.n == rb.n and (ra.n == 0 or torch.equal(ra.rows(), rb.rows())), (tag, k)
    for k in ("tem_x", "tem_weights", "tem_timestamp", "spa_x", "spa_positions", "video_embeds"):
        assert torch.equal(getattr(a, k), getattr(b, k)), (tag, k)


@pytest.mark.parametrize("stop", [1, 2, 4])
def test_qwen_continuation(tmp_path, stop):
    """checkpoints in the warm-up (1 clip), on the fast path (2) and after the redone clip (4): the resumed host's state,
    its 13-item list and its publication equal the uninterrupted host's after every later clip"""
    import flash_vstream_b200.qwen.vstream_qwen2vl_realtime as rt
    from flash_vstream_b200.qwen import serve as QS
    from tests import qwen_rt_inputs as RI
    c = dict(t_clip=4, h=4, w=4, xdim=256, temporal_length=12, spatial_length=8, seed=51)
    n_steps, redo_at = 7, 3
    w = RI.merger_weights(256, 512, "bf16", 51)
    clips = _qwen_clips(c, n_steps, redo_at)
    a, sa = _qwen_host(rt, clips, w, c)
    b, sb = _qwen_host(rt, clips, w, c)
    for s in range(stop):
        _qwen_step(a, sa, s, c)
    ck = a.save_video_stream()
    ck.save(tmp_path / "q.safetensors")
    buf = QS.export_qwen_memory(b, grid=(c["h"], c["w"]))
    reader = QS.QwenMemoryReader(*buf)
    b.load_video_stream(CK.StreamCheckpoint.load(tmp_path / "q.safetensors"))
    _same_state(a.stream_state, b.stream_state, ("restored", stop))
    _same_list(a.video_embedding_memory, b.video_embedding_memory, ("restored", stop))
    emb, meta = reader.read()
    assert torch.equal(emb, a.stream_state.video_embeds) and meta["epoch"] == 1 and meta["clips"] == stop
    assert torch.equal(meta["spa_positions"], a.stream_state.spa_positions)
    for s in range(stop, n_steps):
        _qwen_step(a, sa, s, c)
        _qwen_step(b, sb, s, c)
        _same_state(a.stream_state, b.stream_state, ("step", s))
        _same_list(a.video_embedding_memory, b.video_embedding_memory, ("step", s))
        emb, meta = reader.read()
        assert torch.equal(emb, a.stream_state.video_embeds) and meta["epoch"] == 1 and meta["clips"] == s + 1
    assert a.stream_state.redone_steps == 1 and a.stream_state.fast_steps >= 3
    other = rt.FlashMemory(flash_memory_temporal_length=10, flash_memory_spatial_length=8)
    with pytest.raises(ValueError, match="flash_memory_temporal_length"):
        rt.QwenStreamState.restore(ck, other, b.visual.merger, "cuda")
