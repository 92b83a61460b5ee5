"""GPU tests of the lazy full-resolution bank (DESIGN.md §3.18): a lazy_full_res stream, which runs the full-resolution
tower on a frame only the first time the DAM picks it, publishes after every step the bits of an eager twin fed the same
clips and draws — every item of the 13-item list but item 7 (the full-resolution bank, a zero-row stand-in when lazy),
video_embeds, spa_x and the positions — and encodes exactly the frames the NumPy pick plan (test_qwen_lazy_host) finds
in its picks.  Single streams over every spatial method, 1- and 8-patch clips, banks capped at 0 device frames, pools of
several grids and a preprocessor pool against single streams, the host knob, and checkpoints between eager and lazy
streams, pools and the single-stream host."""
import random

import numpy as np
import pytest
import torch

from tests import preprocess_inputs as PI
from tests import qwen_rt_inputs as RI
from tests import qwen_vit_inputs as VI
from tests.test_qwen_lazy_host import np_plan

pytestmark = pytest.mark.gpu
D, DM = 1280, 512
METHODS = ["klarge_retrieve", "klarge_retrieve_cos", "sample", "nearest"]


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


def clip(seed, t, h=8, w=8):
    g = torch.Generator().manual_seed(seed)
    return torch.randn(t * h * w, 1176, generator=g).bfloat16().cuda(), torch.tensor([[t, h, w]])


class Twin:
    """one stream stepped alone through QwenStreamState, eager (the host's two-resolution tower pass) or lazy (the
    half-resolution pass, and the pixel rows with the tower for the picked frames)"""

    def __init__(self, host, seed, lazy, **caps):
        from flash_vstream_b200.draws import DrawSource
        from flash_vstream_b200.qwen.stream_state import QwenStreamState
        self.visual, self.lazy = host.visual, lazy
        self.st = QwenStreamState(self.visual.flash_memory, self.visual.merger, lazy_full_res=lazy, **caps)
        self.st.rng = DrawSource(seed, "cuda")
        self.enc = np.zeros(0, bool)             # the NumPy plan's mask
        self.planned = 0

    def step(self, c):
        pix, thw = c
        t, h, w = (int(v) for v in thw[0])
        v, st = self.visual, self.st
        if self.lazy:
            small, sg = v.flash_memory.temporal_pool(pix, thw[0])
            st.step(pix, v.encode_patches(small, sg.view(1, 3)), t, (h, w), (h // 2, w // 2), st.n_frames,
                    tower=v.encode_patches)
        else:
            feats, _, _ = v.forward_simple_not_merge(pix, thw)
            n = t * h * w
            st.step(feats[:n], feats[n: n + n // 4], t, (h, w), (h // 2, w // 2), st.n_frames)
        follow_plan(self, st)


def follow_plan(tw, st):
    """apply the NumPy plan to the step's picks; a lazy state must have encoded exactly what it plans"""
    tw.enc = np.concatenate([tw.enc, np.zeros(st.n_frames - len(tw.enc), bool)])
    picks = st.spa_positions.cpu().numpy()
    tw.planned += len(np_plan(None if len(picks) == st.n_frames else picks, tw.enc))
    if st.lazy_full_res:
        assert st.n_encoded == tw.planned
        assert np.array_equal(st.encoded.rows().cpu().numpy().astype(bool), tw.enc)


def bits(t):
    t = t.cpu()
    return t.view(torch.int16) if t.dtype in (torch.bfloat16, torch.float16) else t


def same(a, b):
    if a is None or b is None:
        return a is None and b is None
    if not torch.is_tensor(a):
        return a == b
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(bits(a), bits(b))


def check(lazy_list, eager_list, tag):
    assert len(lazy_list) == len(eager_list) == 13, tag
    for i, (u, v) in enumerate(zip(lazy_list, eager_list)):
        if i == 7:
            assert u.shape[0] == 0, tag                          # the zero-row stand-in x[:0]
            continue
        assert same(u, v), (tag, i)


def check_states(a, b, tag):
    for k in ("n_frames", "steps", "fast_steps", "redone_steps", "n_tem"):
        assert getattr(a, k) == getattr(b, k), (tag, k)
    check(a.as_list(), b.as_list(), tag)
    assert same(a.spa_x, b.spa_x) and same(a.video_embeds, b.video_embeds) and same(a.spa_positions, b.spa_positions)


def positions(flash, lst, n_tokens):
    """the AM-RoPE positions prepare_realtime_inference computes from a list"""
    pid = torch.zeros(3, 1, n_tokens + 4, dtype=torch.int64, device="cuda")
    vis = torch.full((n_tokens + 4,), -1, dtype=torch.int64, device="cuda")
    vis[2: 2 + n_tokens] = 0
    tem_pos = torch.round(lst[3].float()).to(torch.int64)
    return flash.calc_am_rope(pid[:, 0], vis, lst[1], tem_pos, lst[5], lst[6])


def test_pick_plan_kernel_matches_numpy(rt):
    from flash_vstream_b200.qwen import ops as Q
    r = np.random.default_rng(3)
    jobs, refs, keep = [], [], []
    for j in range(21):                                          # more jobs than one launch takes
        n_frames = int(r.integers(1, 200))
        enc = r.random(n_frames) < 0.3
        whole = j % 5 == 0
        n = n_frames if whole else int(r.integers(1, 70))
        picks = None if whole else r.integers(-2, n_frames + 2, n)
        if not whole:
            picks[r.random(n) < 0.3] = picks[0]                   # repeated picks
        mask = torch.tensor(enc, dtype=torch.uint8, device="cuda")
        plan = torch.full((n,), -7, dtype=torch.int64, device="cuda")
        count = torch.zeros(1, dtype=torch.int32, device="cuda")
        pk = None if whole else torch.tensor(picks, device="cuda")
        keep.append((mask, plan, count, pk))
        jobs.append((pk, n, mask, n_frames, plan, count.data_ptr()))
        want_enc = enc.copy()
        refs.append((np_plan(picks, want_enc), want_enc))
    Q.pick_plan_multi(jobs)
    for (mask, plan, count, _), (want, want_enc) in zip(keep, refs):
        k = int(count.item())
        assert k == len(want) and plan[:k].cpu().numpy().tolist() == want.tolist()
        assert np.array_equal(mask.cpu().numpy().astype(bool), want_enc)


@pytest.mark.parametrize("method", METHODS)
@pytest.mark.parametrize("t", [1, 8])
def test_lazy_stream_equals_eager(rt, tower, merger, method, t):
    host = host_for(rt, tower, merger, method=method)
    lazy, eager = Twin(host, 11, True), Twin(host, 11, False)
    steps = (3 + 200 if method == "klarge_retrieve" else 40) if t == 1 else 25      # 3 fill steps: S0 = 3 frames
    fl = host.visual.flash_memory
    for k in range(steps):
        c = clip(1000 * t + k, t)
        lazy.step(c)
        eager.step(c)
        check_states(lazy.st, eager.st, (method, t, k))
        n_tok = lazy.st.video_embeds.shape[0]
        assert same(positions(fl, lazy.st.as_list(), n_tok), positions(fl, eager.st.as_list(), n_tok)), (method, t, k)
    assert lazy.st.fast_steps > 0
    if method.startswith("klarge"):           # 'sample' picks the newest frame every step: it encodes every frame
        assert lazy.st.n_encoded < lazy.st.n_frames


def test_spatial_length_zero_never_encodes(rt, tower, merger):
    """no DAM: nothing is retrieved, so no frame is encoded, no pick plan runs and no count is read back"""
    from flash_vstream_b200.qwen import QwenStreamPool
    host = host_for(rt, tower, merger, S=0)
    lazy, eager = Twin(host, 6, True), Twin(host, 6, False)
    pool, ref = QwenStreamPool(host, lazy_full_res=True), QwenStreamPool(host)
    a, b = [pool.open(seed=s) for s in range(4)], [ref.open(seed=s) for s in range(4)]
    for k in range(12):                                      # T0 = 4 frames: past the CSM length from step 3 on
        c = clip(600 + k, 2)
        lazy.step(c)
        eager.step(c)
        check_states(lazy.st, eager.st, ("single", k))
        pool.step({s: clip(700 + 10 * k + s, 2) for s in a})
        ref.step({s: clip(700 + 10 * k + s, 2) for s in b})
        for x, y in zip(a, b):
            check_states(pool.state(x), ref.state(y), ("pool", k, x))
    for st in [lazy.st] + [pool.state(x) for x in a]:
        assert st.n_encoded == 0 and int(st.encoded.rows().sum()) == 0 and st.n_frames == 24
    assert lazy.st.fast_steps > 0


def test_no_tower_is_refused_before_the_plan(rt, tower, merger):
    from flash_vstream_b200.qwen.stream_state import QwenStreamState
    host = host_for(rt, tower, merger)
    v = host.visual
    st = QwenStreamState(v.flash_memory, v.merger, lazy_full_res=True)
    pix, thw = clip(5, 2)
    small, sg = v.flash_memory.temporal_pool(pix, thw[0])
    with pytest.raises(NotImplementedError, match="no full-resolution tower"):
        st.step(pix, v.encode_patches(small, sg.view(1, 3)), 2, (8, 8), (4, 4), 0)
    assert st.n_encoded == 0 and int(st.encoded.rows().sum()) == 0       # no frame marked encoded


@pytest.mark.parametrize("t", [1, 2])
def test_lazy_stream_with_banks_at_zero_device_frames(rt, tower, merger, t):
    host = host_for(rt, tower, merger)
    lazy = Twin(host, 4, True, device_frames=0, small_device_frames=0)
    eager = Twin(host, 4, False, device_frames=0, small_device_frames=0)
    for k in range(40):
        c = clip(77 + k, t)
        lazy.step(c)
        eager.step(c)
        check_states(lazy.st, eager.st, (t, k))
    assert lazy.st.n_host == lazy.st.n_frames and lazy.st.bank_x.n == 0


def test_lazy_pool_equals_eager_single_streams(rt, tower, merger):
    from flash_vstream_b200.qwen import QwenStreamPool
    host = host_for(rt, tower, merger)
    pool = QwenStreamPool(host, lazy_full_res=True)
    grids = [(8, 8), (12, 8)]
    sids = [pool.open(seed=500 + s) for s in range(6)]
    twins = {sid: Twin(host, 500 + sid, False) for sid in sids}
    r = random.Random(2)
    for k in range(14):
        listed = [s for s in sids if r.random() < 0.85] or sids[:1]
        rnd = {s: clip(100 * k + s, r.choice([1, 2, 8]), *grids[s % 2]) for s in listed}
        pool.step(rnd)
        for s, c in rnd.items():
            twins[s].step(c)
            tw = twins[s]
            assert pool.state(s).n_encoded == tw.planned, (k, s)
        for s in sids:
            if pool.state(s).n_frames:
                check_states(pool.state(s), twins[s].st, (k, s))
    assert all(pool.state(s).n_encoded < pool.state(s).n_frames for s in sids)
    assert any(pool.state(s).fast_steps for s in sids)


def test_lazy_preprocessor_pool(rt, tower, merger):
    from flash_vstream_b200 import preprocess as P
    from flash_vstream_b200.qwen import QwenStreamPool
    host = host_for(rt, tower, merger)
    proc = P.Qwen2VLFramePreprocessor(max_pixels=112 * 168, additional_pool_size=2)
    lazy, eager = QwenStreamPool(host, preprocess=proc, lazy_full_res=True), QwenStreamPool(host, preprocess=proc)
    a = [lazy.open(seed=s) for s in range(4)]
    b = [eager.open(seed=s) for s in range(4)]
    for k in range(10):
        frames = [PI.frames(40 * k + s, (2 if s % 2 else 1, 100, 120)) for s in range(4)]
        lazy.step(dict(zip(a, frames)))
        eager.step(dict(zip(b, frames)))
        for x, y in zip(a, b):
            check_states(lazy.state(x), eager.state(y), (k, x))
    assert all(lazy.state(x).n_encoded < lazy.state(x).n_frames for x in a)


def test_host_knob(rt, tower, merger):
    lazy, eager = host_for(rt, tower, merger), host_for(rt, tower, merger)
    lazy.fvs_lazy_full_res = True
    lists = []
    torch.manual_seed(3)
    random.seed(3)
    for k in range(12):
        c = clip(900 + k, 2)
        eager.embed_new_video_clip(c[0], c[1], 2 * k)
        lists.append([v.clone() if torch.is_tensor(v) else v for v in eager.video_embedding_memory])
    torch.manual_seed(3)
    random.seed(3)
    for k in range(12):
        c = clip(900 + k, 2)
        lazy.embed_new_video_clip(c[0], c[1], 2 * k)
        check(lazy.video_embedding_memory, lists[k], k)
    lazy.fvs_lazy_full_res = False
    with pytest.raises(ValueError, match="fvs_lazy_full_res"):
        lazy.embed_new_video_clip(*clip(1, 2), 24)
    lazy.fvs_lazy_full_res = True
    bad = host_for(rt, tower, merger)
    bad.visual.flash_memory.temporal_poolsize = 1
    bad.fvs_lazy_full_res = True
    with pytest.raises(NotImplementedError, match="fvs_lazy_full_res"):
        bad.embed_new_video_clip(*clip(1, 2), 0)


def test_checkpoints(rt, tower, merger):
    from flash_vstream_b200.draws import DrawSource
    from flash_vstream_b200.qwen import QwenStreamPool
    from flash_vstream_b200.qwen.stream_state import QwenStreamState
    host = host_for(rt, tower, merger)
    lazy = QwenStreamPool(host, lazy_full_res=True, device_frames=3)
    eager = QwenStreamPool(host)
    la, ea = lazy.open(seed=1), eager.open(seed=1)
    for k in range(8):
        c = clip(50 + k, 2)
        lazy.step({la: c})
        eager.step({ea: c})
    check_states(lazy.state(la), eager.state(ea), "pre")
    ck_lazy, ck_eager = lazy.checkpoint(la), eager.checkpoint(ea)
    n_enc = int(ck_lazy.tensor("encoded").sum())
    assert n_enc == lazy.state(la).n_encoded < 16
    assert ck_lazy.counters["pix_frames"] == 16 - n_enc == ck_lazy.tensor("pixels").shape[0]    # unencoded frames only
    assert "encoded" not in ck_eager.tensors and "pix_frames" not in ck_eager.counters      # eager: as before
    # lazy -> eager with frames not yet encoded is refused, naming the knob
    with pytest.raises(NotImplementedError, match="lazy_full_res"):
        eager.open(checkpoint=ck_lazy)
    # lazy -> lazy (pool, uncapped) and eager -> lazy, against the eager stream
    moved = QwenStreamPool(host, lazy_full_res=True)
    m1, m2 = moved.open(checkpoint=ck_lazy), moved.open(checkpoint=ck_eager)
    for k in range(6):
        c = clip(80 + k, (1, 8, 2)[k % 3])
        moved.step({m1: c, m2: c})
        eager.step({ea: c})
        check_states(moved.state(m1), eager.state(ea), ("lazy->lazy", k))
        check_states(moved.state(m2), eager.state(ea), ("eager->lazy", k))
    # lazy pool -> lazy single-stream host: the host draws from the global generators, the reference from a seeded source
    single = host_for(rt, tower, merger)
    single.fvs_lazy_full_res = True
    ck = moved.checkpoint(m1)
    single.load_video_stream(ck)
    ref = Twin(host, 5, False)
    ref.st = QwenStreamState.restore(eager.checkpoint(ea), host.visual.flash_memory, merger, "cuda:0")
    ref.st.rng = DrawSource(5, "cuda:0")
    torch.manual_seed(5)
    random.seed(5)
    for k in range(3):
        c = clip(300 + k, 2)
        single.embed_new_video_clip(c[0], c[1], ref.st.n_frames)
        ref.step(c)
        check(single.video_embedding_memory, ref.st.as_list(), ("single", k))
    # a lazy stream whose every frame is encoded restores eagerly
    fill = QwenStreamPool(host, lazy_full_res=True)
    f = fill.open(seed=2)
    fill.step({f: clip(7, 2)})
    assert fill.state(f).n_encoded == fill.state(f).n_frames
    e2 = eager.open(checkpoint=fill.checkpoint(f))
    assert not eager.state(e2).lazy_full_res and eager.state(e2).n_frames == 2
