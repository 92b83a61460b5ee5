"""GPU tests of the LLaVA bank's device window (DESIGN.md §3.14): a bank with device_frames = N keeps frames [0, N) and one
clip's slot in HBM and the later frames in pinned host chunks, and is bit-identical, at every step, to the uncapped bank
on the same frames and draws — prefix, header words, step diagnostics and the whole frame buffer; through StreamPool,
checkpoints across caps, a MemoryReader and the single-stream model; with a fixed device footprint."""
import pytest
import torch

from flash_vstream_b200 import checkpoint as CK
from flash_vstream_b200 import serve
from tests import golden_inputs as GI
from tests.test_checkpoint_gpu import CFG, D, assert_same_info, draws_for, ntm
from tests.test_gpu_parity import fvs, make_model  # noqa: F401  (fvs is a fixture)

pytestmark = pytest.mark.gpu


@pytest.fixture(autouse=True)
def small_host_chunks(monkeypatch):
    """1 MiB host chunks (64 frames at D = 256) instead of 32 MiB: streams cross chunk edges, tests pin little memory"""
    from flash_vstream_b200 import ops
    monkeypatch.setattr(ops.StreamBank, "CHUNK_BYTES", 1 << 20)


def arrays(bank):
    b = bank.bank
    torch.cuda.synchronize(bank.device)
    fb = bank.frame_buffer()
    return {"counters": (b.n_tur, b.n_long, b.n_cur, b.n_frames, b.step), "header": bank.header.cpu(),
            "prefix": bank.prefix().cpu(), "long": bank.long_work[:b.n_long].cpu(), "tur": bank.tur_work[:b.n_tur].cpu(),
            "frames": fb.cpu()}


def assert_same(ref, cap, tag, info=True):
    """cap (any device_frames) equals ref (uncapped) bit for bit; cap's state()[3] is the zero-row stand-in once spilled.
    info: compare the last step's diagnostics too (a restored bank has run no step yet)"""
    x, y = arrays(ref), arrays(cap)
    assert x["counters"] == y["counters"], (tag, x["counters"], y["counters"])
    assert torch.equal(x["frames"].view(torch.int16), ref.state()[3].cpu().view(torch.int16)), tag
    for k in ("prefix", "long", "tur", "frames"):
        assert torch.equal(x[k].view(torch.int16), y[k].view(torch.int16)), (tag, k)
    assert torch.equal(x["header"][1:8], y["header"][1:8]), (tag, "header")
    assert int(y["header"][0]) % 2 == 0, (tag, "seq")
    n, N = cap.bank.n_frames, cap.device_frames
    assert cap.state()[3].shape[0] == (0 if N is not None and n > N else n), tag
    if info:
        assert_same_info(ref, cap, tag)


def run_side_by_side(ops, clips, caps, chunk_cap, seed=3, chunk_bytes=None):
    w = ntm(seed)
    ref = ops.StreamBank(CFG, w, chunk_cap=chunk_cap)
    banks = [ops.StreamBank(CFG, w, chunk_cap=chunk_cap, device_frames=N) for N in caps]
    for b in banks:
        if chunk_bytes:
            b.CHUNK_BYTES = chunk_bytes      # small host chunks: clips cross chunk edges
        assert b.frames.shape[0] == b.device_frames + chunk_cap
    for i, x in enumerate(clips):
        x = x.cuda()
        d = draws_for(ref, x.shape[0], 100 + i)
        ref.step(x, draws=d)
        for b in banks:
            b.step(x, draws=d)
            assert_same(ref, b, (b.device_frames, i))
    return ref, banks


def test_single_frames_300_steps(fvs):
    pkg, ops = fvs
    N = ops.min_device_frames(CFG, 1)
    assert N == 26
    f = GI.scene_features(300, 576, D, 50, scene_len=(3, 9))
    ref, banks = run_side_by_side(ops, [f[i:i + 1] for i in range(300)], [N, N + 5], 1, chunk_bytes=7 * 64 * D * 2)
    assert len(banks[0].host_chunks) == -(-(300 - N) // 7)


def test_32_frame_clips_varying_t(fvs):
    """t varies from 1 to 32; the first clip (32 frames) is longer than long_len and than the bank's long memory"""
    pkg, ops = fvs
    N = ops.min_device_frames(CFG, 32)
    assert N == 64
    lens = [32, 7, 19, 1, 32, 25, 3, 32, 32, 11, 30, 32, 5, 32, 17, 32, 32, 2]
    f = GI.scene_features(sum(lens), 576, D, 51, scene_len=(3, 9))
    clips, s = [], 0
    for t in lens:
        clips.append(f[s:s + t])
        s += t
    run_side_by_side(ops, clips, [N, N + 5], 32, chunk_bytes=13 * 64 * D * 2)


def test_first_clip_longer_than_the_bank(fvs):
    """a first clip of 40 frames (> long_len and > min window's long part) in a bank sized for 40-frame clips"""
    pkg, ops = fvs
    N = ops.min_device_frames(CFG, 40)
    f = GI.scene_features(40 * 4, 576, D, 52, scene_len=(3, 9))
    run_side_by_side(ops, [f[40 * i:40 * (i + 1)] for i in range(4)], [N], 40)


def test_pool_capped_equals_uncapped_one_by_one(fvs):
    pkg, ops = fvs
    rounds, S = 40, 8
    feats = [GI.scene_features(rounds, 576, D, 80 + i) for i in range(S)]
    ref = pkg.StreamPool(make_model(D, 5, pkg))
    pool = pkg.StreamPool(make_model(D, 5, pkg), device_frames=26)
    rs = [ref.open(seed=90 + i) for i in range(S)]
    ps = [pool.open(seed=90 + i) for i in range(S)]
    for r in range(rounds):
        for i in range(S):
            ref.step({rs[i]: feats[i][r:r + 1].cuda()})
        pool.step({ps[i]: feats[i][r:r + 1].cuda() for i in range(S)})
        for i in range(S):
            assert_same(ref.bank(rs[i]), pool.bank(ps[i]), (r, i))
    with pytest.raises(ValueError, match="25 < 26"):
        pkg.StreamPool(make_model(D, 5, pkg), device_frames=25)
    pool.close(ps[0])                     # a reused bank keeps the pool's cap
    sid = pool.open(seed=1)
    assert pool.bank(sid).device_frames == 26 and pool.bank(sid).frames.shape[0] == 27


@pytest.mark.parametrize("cap_a, cap_b", [(30, None), (None, 26), (26, 41), (41, 26)])
def test_checkpoints_across_caps(fvs, tmp_path, cap_a, cap_b):
    """checkpoint at 45 frames, restore in memory and from a .safetensors file into a bank with another cap; 20 more steps
    equal an uninterrupted uncapped stream"""
    pkg, ops = fvs
    f = GI.scene_features(65, 576, D, 53, scene_len=(3, 9))
    w = ntm(3)
    ref = ops.StreamBank(CFG, w, chunk_cap=1)
    a = ops.StreamBank(CFG, w, chunk_cap=1, device_frames=cap_a)
    for i in range(45):
        d = draws_for(ref, 1, 100 + i)
        ref.step(f[i:i + 1].cuda(), draws=d)
        a.step(f[i:i + 1].cuda(), draws=d)
    ck = a.checkpoint()
    assert torch.equal(ck.tensor("frames").view(torch.int16), ref.state()[3].cpu().view(torch.int16))
    ck.save(tmp_path / "a.safetensors")
    targets = [ops.StreamBank(CFG, w, chunk_cap=1, device_frames=cap_b) for _ in range(2)]
    targets[0].restore(ck)
    targets[1].restore(CK.StreamCheckpoint.load(tmp_path / "a.safetensors"))
    for b in targets:
        assert_same(ref, b, "restored", info=False)
    for i in range(45, 65):
        d = draws_for(ref, 1, 100 + i)
        ref.step(f[i:i + 1].cuda(), draws=d)
        for b in targets:
            b.step(f[i:i + 1].cuda(), draws=d)
            assert_same(ref, b, i)


def test_memory_reader_of_a_capped_bank(fvs):
    pkg, ops = fvs
    f = GI.scene_features(40, 576, D, 54, scene_len=(3, 9))
    bank = ops.StreamBank(CFG, ntm(3), chunk_cap=1, device_frames=26)
    reader = serve.MemoryReader(*serve.export_bank(bank))
    for i in range(40):
        bank.step(f[i:i + 1].cuda(), draws=draws_for(bank, 1, 100 + i))
        out, meta = reader.read()
        assert torch.equal(out.cpu().view(torch.int16), bank.prefix().cpu().view(torch.int16)), i
        assert meta["n_frames"] == i + 1 and meta["step"] == i + 1


def test_model_path(fvs):
    """the single-stream model with fvs_bank_device_frames: items 0-2 of video_embedding_memory equal the uncapped
    model's, item 3 is the zero-row stand-in once frames have spilled; a config kept op by op is refused"""
    pkg, ops = fvs
    f = GI.scene_features(80, 576, D, 55, scene_len=(3, 9))
    a, b = make_model(D, 9, pkg), make_model(D, 9, pkg)
    b.fvs_bank_device_frames = 70            # fvs_chunk_cap 32: at least max(25, 32) + 32 = 64
    for i in range(80):
        d = draws_for(a._fvs_bank, 1, 200 + i) if i else None
        a.consolidate_streaming(f[i:i + 1].cuda(), draws=d)
        b.consolidate_streaming(f[i:i + 1].cuda(), draws=d)
        ma, mb = a.video_embedding_memory, b.video_embedding_memory
        for k in range(3):
            assert torch.equal(ma[k], mb[k]), (i, k)
        assert mb[3].shape[0] == (0 if i + 1 > 70 else i + 1)
        assert torch.equal(a.memory_prefix(), b.memory_prefix())
    assert b._fvs_bank.device_frames == 70
    assert torch.equal(b._fvs_bank.frame_buffer().cpu(), a.video_embedding_memory[3].cpu())
    b.fvs_bank_device_frames = 75
    with pytest.raises(ValueError, match="in the middle of a stream"):
        b.consolidate_streaming(f[0:1].cuda())
    op = make_model(D, 9, pkg)
    op.fvs_fused_stream = False
    op.fvs_bank_device_frames = 26
    with pytest.raises(NotImplementedError, match="fvs_bank_device_frames.*fvs_fused_stream"):
        op.consolidate_streaming(f[0:1].cuda())
    small = make_model(D, 9, pkg)
    small.fvs_bank_device_frames = 32
    with pytest.raises(ValueError, match="fvs_bank_device_frames 32 < 64"):
        small.consolidate_streaming(f[0:1].cuda())       # fvs_chunk_cap 32: the minimum is 64


def test_device_bytes_bounded_and_uncapped_unchanged(fvs):
    """a capped bank's HBM does not move over 1000 further frames; per step it makes the same library launches as the
    uncapped bank, whose frame buffer starts as before (max(frames_cap, 2 chunk_cap) rows)"""
    pkg, ops = fvs
    lib = ops.L.load()
    w = ntm(3)
    ref = ops.StreamBank(CFG, w, chunk_cap=1)
    assert tuple(ref.frames.shape) == (256, 64, D) and ref.bank.frames_window == 0
    cap = ops.StreamBank(CFG, w, chunk_cap=1, device_frames=26)
    g = torch.Generator(device="cuda").manual_seed(7)

    def step(bank, i):
        x = torch.randn(1, 576, D, generator=g, device="cuda").half()
        c0 = lib.fvs_launch_count()
        bank.step(x, draws=draws_for(bank, 1, i))
        return lib.fvs_launch_count() - c0

    for i in range(100):
        assert step(ref, i) == step(cap, i), i
    torch.cuda.synchronize()
    before = (cap.frames.data_ptr(), cap.frames.numel(), torch.cuda.memory_allocated())
    for i in range(100, 1100):
        step(cap, i)
    torch.cuda.synchronize()
    after = (cap.frames.data_ptr(), cap.frames.numel(), torch.cuda.memory_allocated())
    assert after == before
    assert cap.frames.numel() * 2 == 27 * 64 * D * 2 and cap.n_host() == 1100 - 26
