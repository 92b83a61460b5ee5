"""GPU tests of a Qwen2-VL stream without a full-resolution bank (DESIGN.md §3.19): a lazy_full_res stream with
full_res_bank=False, which keeps no x or merged row beyond its DAM and re-encodes a pick its previous DAM does not hold,
publishes after every step the bits of an eager twin fed the same clips and draws (every item of the 13-item list but
item 7, video_embeds, spa_x, the DAM positions and the AM-RoPE positions) and encodes exactly what the NumPy plan
(test_qwen_no_bank_host) finds in its picks.  The two new entry points against NumPy and torch; single streams over both
retrieval metrics, 1-, 2- and 8-patch clips, the 336 px grid and a non-square one, the half-resolution bank at zero
device frames, the duplicate-rows redo; pools of 1, 2, 5 and 16 streams; the memory it holds; checkpoints in every
direction; the host knob."""
import random

import numpy as np
import pytest
import torch

from tests import test_qwen_lazy_gpu as LT
from tests.test_qwen_lazy_gpu import check, check_states, clip, host_for, merger, positions, rt, same, tower  # noqa: F401
from tests.test_qwen_no_bank_host import np_plan_prev

pytestmark = pytest.mark.gpu
METRICS = ["klarge_retrieve", "klarge_retrieve_cos"]


class NoBank(LT.Twin):
    """one bank-less stream stepped alone through QwenStreamState, following the NumPy plan"""

    def __init__(self, host, seed, **caps):
        super().__init__(host, seed, True, full_res_bank=False, **caps)
        self.fr = np.zeros(0, np.uint8)
        self.again = 0

    def step(self, c):
        pix, thw = c
        t, h, w = (int(v) for v in thw[0])
        v, st = self.visual, self.st
        prev, redone = prev_picks(st), st.redone_steps
        small, sg = v.flash_memory.temporal_pool(pix, thw[0])
        st.step(pix, v.encode_patches(small, sg.view(1, 3)), t, (h, w), (h // 2, w // 2), st.n_frames,
                tower=v.encode_patches)
        follow(self, st, prev, st.redone_steps != redone)


def prev_picks(st):
    return None if st.spa_positions is None else st.spa_positions.cpu().numpy()


def follow(tw, st, prev, redone=False):
    """apply the NumPy plan to the step's picks; the state must have encoded exactly what it plans (a redone clip plans
    twice on the device, so its counts are taken over as they are)"""
    tw.fr = np.concatenate([tw.fr, np.zeros(st.n_frames - len(tw.fr), np.uint8)])
    if redone:
        tw.fr, tw.planned, tw.again = st.encoded.rows().cpu().numpy(), st.n_encoded, st.re_encode_count()
        return
    if st.spa_positions.numel():
        plan, again = np_plan_prev(st.spa_positions.cpu().numpy(), prev, tw.fr)
        tw.planned += len(plan)
        tw.again += again
    assert st.n_encoded == tw.planned
    assert st.re_encode_count() == tw.again
    assert np.array_equal(st.encoded.rows().cpu().numpy(), tw.fr)


def holds_no_bank(st):
    assert st.bank_x.buf is None and st.bank_merged.buf is None and st.host_chunks == [] and st.n_host == 0


# ---------------------------------------------------------------------------------------------------------- kernels
def test_bankless_plan_matches_numpy_and_single_calls(rt):
    from flash_vstream_b200.qwen import ops as Q
    r = np.random.default_rng(4)
    cases, jobs = [], []
    for j in range(21):                                          # more jobs than one launch takes
        n_frames = int(r.integers(1, 200))
        fr = r.choice(np.array([0, 0, 1, 2], np.uint8), n_frames)
        n = int(r.integers(1, 70))
        picks = r.integers(-2, n_frames + 2, n)
        picks[r.random(n) < 0.3] = picks[0]                      # repeated picks
        prev = r.integers(0, n_frames, int(r.integers(0, 40)))
        if j % 7 == 1:
            prev = np.unique(np.clip(picks, 0, n_frames - 1))    # every pick in the previous DAM
        if j % 7 == 2:
            prev = np.setdiff1d(np.arange(n_frames), picks)[:30]  # none of them
        cases.append((picks, prev, fr))
    outs = []
    for single in (False, True):
        got = []
        for picks, prev, fr in cases:
            t = dict(picks=torch.tensor(picks, device="cuda"), frames=torch.tensor(fr, device="cuda"),
                     prev=torch.tensor(prev, dtype=torch.int64, device="cuda") if len(prev) else None,
                     plan=torch.full((len(picks),), -7, dtype=torch.int64, device="cuda"),
                     count=torch.zeros(1, dtype=torch.int32, device="cuda"),
                     again=torch.zeros(1, dtype=torch.int64, device="cuda"))
            got.append(t)
        js = [(t["picks"], len(p), t["frames"], len(fr), t["plan"], t["count"].data_ptr(), 2, t["prev"], t["again"])
              for t, (p, _, fr) in zip(got, cases)]               # no bank: byte 2 is stored
        if single:
            for jb in js:
                Q.pick_plan_multi([jb])
        else:
            Q.pick_plan_multi(js)
        outs.append(got)
    for k, (picks, prev, fr) in enumerate(cases):
        want_fr = fr.copy()
        want, again = np_plan_prev(picks, prev, want_fr)
        for got in outs:
            t = got[k]
            c = int(t["count"].item())
            assert c == len(want) and t["plan"][:c].cpu().numpy().tolist() == want.tolist(), k
            assert np.array_equal(t["frames"].cpu().numpy(), want_fr) and int(t["again"].item()) == again, k
        if k % 7 == 1:
            assert len(want) == 0


def test_bankless_dam_gather_matches_torch_and_single_calls(rt):
    from flash_vstream_b200.qwen import ops as Q
    g = torch.Generator().manual_seed(9)
    fx, fm, F = 16 * 32, 4 * 64, 5                               # 16 rows of 32 wide, 4 merged rows of 64; 5 per chunk

    def job(n_frames, n_base, n_dev, m, n_fresh, n, seed):
        r = np.random.default_rng(seed)
        base_x = torch.randn(n_base, fx, generator=g).bfloat16()
        base_m = torch.randn(n_base, fm, generator=g).bfloat16()
        chunks = []
        for c0 in range(n_dev, n_base, F):
            buf = torch.zeros(F * (fx + fm), dtype=torch.bfloat16).pin_memory()
            k = min(F, n_base - c0)
            buf[: F * fx].view(F, fx)[:k] = base_x[c0: c0 + k]
            buf[F * fx:].view(F, fm)[:k] = base_m[c0: c0 + k]
            chunks.append(buf)
        table = torch.tensor([Q.host_device_ptr(b) for b in chunks] or [0], dtype=torch.int64, device="cuda")
        prev = r.choice(n_frames, m, replace=False)
        fresh = r.choice(np.setdiff1d(np.arange(n_frames), prev), n_fresh, replace=False)
        picks = r.integers(-1, n_frames + 1, n)
        px, pm = torch.randn(m, fx, generator=g).bfloat16(), torch.randn(m, fm, generator=g).bfloat16()
        qx, qm = torch.randn(n_fresh, fx, generator=g).bfloat16(), torch.randn(n_fresh, fm, generator=g).bfloat16()
        want_x, want_m, fetches = torch.zeros(n, fx, dtype=torch.bfloat16), torch.zeros(n, fm, dtype=torch.bfloat16), 0
        for i, p in enumerate(picks):
            if not 0 <= p < n_frames:
                continue
            if p in prev:
                k = int(np.nonzero(prev == p)[0][0])
                want_x[i], want_m[i] = px[k], pm[k]
            elif p in fresh:
                k = int(np.nonzero(fresh == p)[0][0])
                want_x[i], want_m[i] = qx[k], qm[k]
            elif p < n_base:
                want_x[i], want_m[i] = base_x[p], base_m[p]
                fetches += int(p >= n_dev)
        cu = lambda t: t.cuda()
        a = dict(picks=torch.tensor(picks, device="cuda"), n_frames=n_frames,
                 prev=(torch.tensor(prev, device="cuda"), cu(px), cu(pm)) if m else None,
                 fresh=(torch.tensor(fresh, device="cuda"), n_fresh, cu(qx), cu(qm)) if n_fresh else None,
                 n_base=n_base, dev_x=cu(base_x[:n_dev]) if n_dev else None, dev_merged=cu(base_m[:n_dev]) if n_dev else None,
                 n_dev=n_dev, chunks=table, chunk_frames=F, x_frame_elems=fx, merged_frame_elems=fm)
        return a, chunks, (want_x, want_m, fetches)

    specs = [(40, 20, 7, 6, 9, 50), (30, 0, 0, 10, 12, 40), (25, 25, 25, 0, 0, 20), (33, 12, 0, 8, 5, 64)]
    jobs = [job(*s, seed=i) for i, s in enumerate(specs)]

    def outs():
        return [dict(a, spa_x_out=torch.full((len(a["picks"]), fx), 7, dtype=torch.bfloat16, device="cuda"),
                     merged_out=torch.full((len(a["picks"]), fm), 7, dtype=torch.bfloat16, device="cuda"),
                     host_fetches=torch.zeros(1, dtype=torch.int64, device="cuda")) for a, _, _ in jobs]

    multi, single = outs(), outs()
    Q.dam_gather_multi(multi)
    for a in single:
        Q.dam_gather_multi([a])
    for (_, _, (wx, wm, fetches)), a, b in zip(jobs, multi, single):
        for o in (a, b):
            assert same(o["spa_x_out"], wx) and same(o["merged_out"], wm)
            assert int(o["host_fetches"].item()) == fetches
    torch.cuda.synchronize()


# ---------------------------------------------------------------------------------------------------------- one stream
def run_twins(host, steps, make_clip, **caps):
    nob, eager = NoBank(host, 11, **caps), LT.Twin(host, 11, False, **caps)
    fl = host.visual.flash_memory
    for k in range(steps):
        c = make_clip(k)
        nob.step(c)
        eager.step(c)
        check_states(nob.st, eager.st, k)
        n_tok = nob.st.video_embeds.shape[0]
        assert same(positions(fl, nob.st.as_list(), n_tok), positions(fl, eager.st.as_list(), n_tok)), k
        holds_no_bank(nob.st)
    return nob, eager


@pytest.mark.parametrize("method", METRICS)
@pytest.mark.parametrize("t", [1, 2, 8])
def test_no_bank_stream_equals_eager(rt, tower, merger, method, t):
    host = host_for(rt, tower, merger, method=method)             # S0 = 3 frames, T0 = 4: every phase is passed
    nob, _ = run_twins(host, {1: 40, 2: 25, 8: 10}[t], lambda k: clip(2000 * t + k, t))
    assert nob.st.fast_steps > 0 and nob.st.n_frames > 4


@pytest.mark.parametrize("grid", [(24, 24), (24, 36)])
def test_no_bank_stream_real_grids(rt, tower, merger, grid):
    host = host_for(rt, tower, merger)
    nob, _ = run_twins(host, 7, lambda k: clip(3000 + k, 2, *grid))
    assert nob.st.fast_steps > 0


def test_re_encodes_a_frame_that_left_the_dam(rt, tower, merger):
    """'sample' retrieval picks linspace(0, n - 1, S0) rounded: with S0 = 3, frame 3 is picked at n = 4, not at 5 or 6,
    and again at 7"""
    host = host_for(rt, tower, merger, method="sample")
    nob, _ = run_twins(host, 24, lambda k: clip(4000 + k, 1))
    assert nob.st.re_encode_count() > 0 and nob.again == nob.st.re_encode_count()


def test_small_bank_at_zero_device_frames(rt, tower, merger):
    host = host_for(rt, tower, merger)
    nob, _ = run_twins(host, 30, lambda k: clip(77 + k, 1), small_device_frames=0)
    assert nob.st.n_small_host == nob.st.n_frames


def test_duplicate_rows_redo(rt, tower, merger):
    """a frozen video (every frame of a clip the same) gives the CSM duplicate rows: complete() redoes the clip through
    the synchronous path, which plans against the same previous DAM"""
    host = host_for(rt, tower, merger)

    def frozen(k):
        pix, thw = clip(5000 + k // 3, 1)
        return pix.repeat(2, 1), torch.tensor([[2, 8, 8]])

    nob, _ = run_twins(host, 14, frozen)
    assert nob.st.redone_steps > 0


def test_memory_held(rt, tower, merger):
    """no x or merged storage; pinned bytes = pixel chunks + half-resolution chunks past the cap (DESIGN.md §3.19)"""
    from flash_vstream_b200.host_tier import chunk_frames
    host = host_for(rt, tower, merger)
    nob = NoBank(host, 3, small_device_frames=2)
    nob.st.CHUNK_BYTES = 5 * 64 * 1176 * 2                       # 5 frames of pixel rows per chunk: several chunks
    for k in range(10):
        nob.step(clip(6000 + k, 2))
    st = nob.st
    holds_no_bank(st)
    n, hw, D = st.n_frames, 64, 1280
    fp = chunk_frames(hw * 1176 * 2, st.CHUNK_BYTES)
    fs = chunk_frames(hw // 4 * D * 2, st.CHUNK_BYTES)
    want = -(-n // fp) * fp * hw * 1176 * 2 + -(-(n - 2) // fs) * fs * hw // 4 * D * 2
    assert fp == 5 and st.pinned_bytes() == want
    assert st.spa_x.shape[0] == 3 and st.bank_small.n == 2


# ---------------------------------------------------------------------------------------------------------- pools
@pytest.mark.parametrize("S", [1, 2, 5, 16])
def test_no_bank_pool_equals_eager_pool(rt, tower, merger, S):
    from flash_vstream_b200.qwen import QwenStreamPool
    host = host_for(rt, tower, merger)
    pool, ref = QwenStreamPool(host, lazy_full_res=True, full_res_bank=False), QwenStreamPool(host)
    a = [pool.open(seed=700 + s) for s in range(S)]
    b = [ref.open(seed=700 + s) for s in range(S)]
    tw = {x: NoBank(host, 0) for x in a}                         # the NumPy plan of each stream
    r = random.Random(S)
    for k in range(10):
        listed = [i for i in range(S) if r.random() < 0.85] or [0]
        rnd = {i: clip(100 * k + i, r.choice([1, 2, 8])) for i in listed}
        prev = {i: prev_picks(pool.state(a[i])) for i in listed}
        red = {i: pool.state(a[i]).redone_steps for i in listed}
        pool.step({a[i]: c for i, c in rnd.items()})
        ref.step({b[i]: c for i, c in rnd.items()})
        for i in listed:
            st = pool.state(a[i])
            follow(tw[a[i]], st, prev[i], st.redone_steps != red[i])
        for x, y in zip(a, b):
            if pool.state(x).n_frames:
                check_states(pool.state(x), ref.state(y), (S, k, x))
                holds_no_bank(pool.state(x))
    assert any(pool.state(x).fast_steps for x in a)


def test_pool_refuses_bank_less_without_lazy(rt, tower, merger):
    from flash_vstream_b200.qwen import QwenStreamPool
    with pytest.raises(ValueError, match="full_res_bank=False needs lazy_full_res=True"):
        QwenStreamPool(host_for(rt, tower, merger), full_res_bank=False)


# ---------------------------------------------------------------------------------------------------------- checkpoints
def test_checkpoints(rt, tower, merger):
    from flash_vstream_b200.qwen import QwenStreamPool
    host = host_for(rt, tower, merger)
    nob = QwenStreamPool(host, lazy_full_res=True, full_res_bank=False)
    lazy = QwenStreamPool(host, lazy_full_res=True)
    eager = QwenStreamPool(host)
    na, la, ea = nob.open(seed=1), lazy.open(seed=1), eager.open(seed=1)
    for k in range(8):                                           # 16 frames: past T0 = 4
        c = clip(50 + k, 2)
        nob.step({na: c})
        lazy.step({la: c})
        eager.step({ea: c})
    check_states(nob.state(na), eager.state(ea), "pre")
    ck_n, ck_l, ck_e = nob.checkpoint(na), lazy.checkpoint(la), eager.checkpoint(ea)
    assert ck_n.counters["bank_frames"] == 0 and ck_n.counters["pix_frames"] == 16
    assert ck_n.tensor("bank_x").shape[0] == 0 and ck_n.tensor("pixels").shape[0] == 16
    assert ck_n.tensor("spa_x").shape[0] == 3
    with pytest.raises(NotImplementedError, match="full_res_bank"):                  # bank-less -> eager
        eager.open(checkpoint=ck_n)
    # bank-less, eager and lazy -> bank-less (the base bank split across the two tiers), bank-less -> lazy
    moved = QwenStreamPool(host, lazy_full_res=True, full_res_bank=False, device_frames=5)
    back = QwenStreamPool(host, lazy_full_res=True)
    m = {"n->n": (moved, moved.open(checkpoint=ck_n)), "e->n": (moved, moved.open(checkpoint=ck_e)),
         "l->n": (moved, moved.open(checkpoint=ck_l)), "n->l": (back, back.open(checkpoint=ck_n))}
    assert moved.state(m["e->n"][1]).bank_x.n == 5 and moved.state(m["e->n"][1]).n_host == 11
    for k in range(6):
        c = clip(80 + k, (1, 8, 2)[k % 3])
        eager.step({ea: c})
        for tag, (p, sid) in m.items():
            p.step({sid: c})
            check_states(p.state(sid), eager.state(ea), (tag, k))
    # a bank-less stream with a base bank: its checkpoint keeps the base and the later frames' pixel rows
    ck_b = moved.checkpoint(m["e->n"][1])
    assert ck_b.counters["bank_frames"] == 16 and ck_b.counters["pix_frames"] == ck_b.counters["n_frames"] - 16
    again = QwenStreamPool(host, lazy_full_res=True, full_res_bank=False)
    sid = again.open(checkpoint=ck_b)
    for k in range(3):
        c = clip(90 + k, 2)
        eager.step({ea: c})
        again.step({sid: c})
        check_states(again.state(sid), eager.state(ea), ("base", k))


def test_host_knob(rt, tower, merger):
    nob, eager = host_for(rt, tower, merger), host_for(rt, tower, merger)
    nob.fvs_lazy_full_res, nob.fvs_full_res_bank = True, False
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
        nob.embed_new_video_clip(c[0], c[1], 2 * k)
        check(nob.video_embedding_memory, lists[k], k)
    holds_no_bank(nob.stream_state)
    nob.fvs_full_res_bank = True
    with pytest.raises(ValueError, match="fvs_full_res_bank"):
        nob.embed_new_video_clip(*clip(1, 2), 24)
    bad = host_for(rt, tower, merger)
    bad.fvs_full_res_bank = False
    with pytest.raises(ValueError, match="fvs_full_res_bank=False needs fvs_lazy_full_res=True"):
        bad.embed_new_video_clip(*clip(1, 2), 0)
