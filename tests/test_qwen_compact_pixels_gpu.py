"""GPU tests of 8-bit pixel codes (DESIGN.md §3.20): FVS_PRE_QWEN_CODES then fvs_qwen_pixel_decode against the fp32
pre-processing cast to the tower dtype, fvs_qwen_pixel_gather_multi of codes against a torch decode of the same frames,
and compact_pixels pools (lazy and bank-less) against their non-compact twins fed the same frames and draws: every
13-item list, spa_x, video_embeds and the positions after every round, the pinned bytes, every legal checkpoint
direction, and pool_memory_manager."""
import queue
import random

import numpy as np
import pytest
import torch

from tests import preprocess_inputs as PI
from tests.test_qwen_lazy_gpu import check_states, host_for, merger, positions, rt, same, tower  # noqa: F401

pytestmark = pytest.mark.gpu
METRICS = ["klarge_retrieve", "klarge_retrieve_cos"]


def proc(**kw):
    from flash_vstream_b200 import preprocess as P
    return P.Qwen2VLFramePreprocessor(**kw)


def decode_ref(codes, table, dtype):
    """torch: dtype(table[column // 392][code]), codes [..., whole rows of 1176]"""
    ch = (torch.arange(codes.shape[-1], device=codes.device) % 1176 // 392).expand_as(codes)
    return table[ch, codes.long()].to(dtype)


# ---------------------------------------------------------------------------------------------------------- kernels
@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_codes_then_decode_equals_the_cast_rows(rt, dtype):
    from flash_vstream_b200.qwen import ops as Q
    p = proc(max_pixels=336 * 504)
    table = p.device_table()
    for shape in [(1, 336, 336), (2, 100, 120), (4, 480, 640), (2, 336, 504), (1, 57, 301)]:
        f = torch.from_numpy(PI.frames(sum(shape), shape))
        rows = p(f)["pixel_values_videos"]
        codes = p(f, codes=True)
        assert codes["pixel_values_videos"].dtype == torch.uint8
        assert torch.equal(codes["video_grid_thw"], p(f)["video_grid_thw"])
        c = codes["pixel_values_videos"]
        assert torch.equal(Q.pixel_decode(c, table, dtype).view(torch.int16), rows.type(dtype).view(torch.int16)), shape
        assert torch.equal(decode_ref(c, table, torch.float32), rows), shape
    rng = np.random.default_rng(11)
    for n in (1, 2, 7, 33, 40):                                      # job tables of mixed sizes, one-frame clips included
        clips = [torch.from_numpy(PI.frames(1000 * n + i, (int(rng.choice([1, 2, 4])), int(rng.integers(40, 500)),
                                                           int(rng.integers(40, 500))))) for i in range(n)]
        out, views, grids = p.many(clips)
        cout, cviews, cgrids = p.many(clips, codes=True)
        assert cout.dtype == torch.uint8 and cout.shape == out.shape
        assert all(torch.equal(a, b) for a, b in zip(grids, cgrids))
        dec = Q.pixel_decode(cout, table, dtype)
        assert torch.equal(dec.view(torch.int16), out.type(dtype).view(torch.int16)), n
        for i, (v, cv) in enumerate(zip(views, cviews)):
            assert torch.equal(cv, p(clips[i], codes=True)["pixel_values_videos"]), (n, i)


@pytest.mark.parametrize("dtype", [torch.bfloat16, torch.float16])
def test_pixel_gather_of_codes_equals_torch_decode(rt, dtype):
    from flash_vstream_b200.qwen import ops as Q
    from flash_vstream_b200.qwen.stream_state import PixelStore
    table = proc().device_table()
    g = torch.Generator().manual_seed(3)
    jobs, want = [], []
    for j, (hw, base, n) in enumerate([(16, 0, 9), (64, 3, 14), (4, 5, 9), (36, 1, 20)] * 5):
        fe = hw * 1176
        st = PixelStore(torch.uint8, fe, base, chunk_bytes=3 * fe, values=table, out_dtype=dtype)   # 3 frames a chunk
        codes = torch.randint(0, 256, (n - base, fe), generator=g, dtype=torch.uint8)
        st.append(codes[: (n - base) // 2].cuda(), "cuda")                       # device and host sources
        st.append(codes[(n - base) // 2:], "cuda")
        plan = torch.tensor([n - 1, base, -1, n, base + 2, n + 5] + ([base - 1] if base else []) + list(range(base, n)),
                            dtype=torch.int64)
        out = torch.empty(plan.numel(), fe, dtype=dtype, device="cuda")
        jobs.append((plan.cuda(), plan.numel(), n, base, st.table, st.chunk_frames, out, fe, table))
        w = torch.zeros(plan.numel(), fe, dtype=dtype)
        for i, f in enumerate(plan.tolist()):
            if base <= f < n:
                w[i] = decode_ref(codes[f - base].cuda()[None], table, dtype)[0].cpu()
        want.append((w, st))
    Q.pixel_gather_multi(jobs)
    for (w, _), job in zip(want, jobs):
        assert torch.equal(job[6].cpu().view(torch.int16), w.view(torch.int16))
    for (w, _), job in zip(want, jobs):                              # each job alone: the one-job table
        job[6].zero_()
        Q.pixel_gather_multi([job])
        assert torch.equal(job[6].cpu().view(torch.int16), w.view(torch.int16))


# ---------------------------------------------------------------------------------------------------------- pools
def pools(host, p, bank, **caps):
    from flash_vstream_b200.qwen import QwenStreamPool
    kw = dict(preprocess=p, lazy_full_res=True, full_res_bank=bank, **caps)
    return QwenStreamPool(host, compact_pixels=True, **kw), QwenStreamPool(host, **kw)


def frames_of(seed, t, size):
    return torch.from_numpy(PI.frames(seed, (t,) + size))


def run_rounds(host, comp, twin, S, rounds, sizes, ts, seed):
    """S streams per pool, the same seeded frames each round; every stream equals its twin after every round"""
    a = [comp.open(seed=seed + s) for s in range(S)]
    b = [twin.open(seed=seed + s) for s in range(S)]
    r = random.Random(seed)
    fl = host.visual.flash_memory
    for k in range(rounds):
        listed = [i for i in range(S) if r.random() < 0.85] or [0]
        rnd = {i: frames_of(1000 * k + i + seed, r.choice(ts), sizes[i % len(sizes)]) for i in listed}
        comp.step({a[i]: f for i, f in rnd.items()})
        twin.step({b[i]: f for i, f in rnd.items()})
        for x, y in zip(a, b):
            u, v = comp.state(x), twin.state(y)
            if u.n_frames:
                check_states(u, v, (S, k, x))
                n_tok = u.video_embeds.shape[0]
                assert same(positions(fl, u.as_list(), n_tok), positions(fl, v.as_list(), n_tok)), (S, k, x)
                assert u.n_encoded == v.n_encoded and u.re_encode_count() == v.re_encode_count()
    return a, b


@pytest.mark.parametrize("S, bank, method", [(1, True, METRICS[0]), (2, False, METRICS[1]), (5, True, METRICS[1]),
                                             (16, False, METRICS[0])])
def test_compact_pool_equals_twin(rt, tower, merger, S, bank, method):
    host = host_for(rt, tower, merger, method=method)
    comp, twin = pools(host, proc(), bank)
    # 1-, 2- and 8-patch clips (1, 2 and 16 frames); grids 8 x 8 and 8 x 12
    a, b = run_rounds(host, comp, twin, S, 8, [(112, 112), (112, 168)], [1, 2, 4, 16], 50 * S)
    assert any(comp.state(x).fast_steps for x in a)
    assert all(comp.state(x).pixels.dtype == torch.uint8 for x in a if comp.state(x).n_frames)


@pytest.mark.parametrize("bank", [True, False])
def test_compact_pool_real_grids(rt, tower, merger, bank):
    """the 336 px grid (24, 24) and (24, 36), banks capped at zero device frames"""
    host = host_for(rt, tower, merger)
    comp, twin = pools(host, proc(), bank, small_device_frames=0, device_frames=0 if bank else None)
    a, _ = run_rounds(host, comp, twin, 2, 6, [(336, 336), (336, 504)], [2], 77)
    assert comp.state(a[0]).grid == (24, 24) and comp.state(a[1]).grid == (24, 36)
    assert all(comp.state(x).n_small_host == comp.state(x).n_frames for x in a)


def test_compact_pool_re_encodes(rt, tower, merger):
    """'sample' retrieval re-encodes frames that left the DAM (§3.19): they come back decoded from their codes"""
    host = host_for(rt, tower, merger, method="sample")
    comp, twin = pools(host, proc(), False)
    a, _ = run_rounds(host, comp, twin, 2, 16, [(112, 112)], [1], 9)
    assert all(comp.state(x).re_encode_count() > 0 for x in a)


@pytest.mark.parametrize("bank", [True, False])
def test_pinned_bytes_halve(rt, tower, merger, bank):
    host = host_for(rt, tower, merger)
    comp, twin = pools(host, proc(), bank)
    a, b = run_rounds(host, comp, twin, 2, 6, [(336, 336)], [2, 4], 5)
    for x, y in zip(a, b):
        pc, pt = comp.state(x).pixels, twin.state(y).pixels
        n = pc.n - pc.base
        assert pc.chunk_frames >= 2 * pt.chunk_frames - 1
        bc = sum(c.numel() * c.element_size() for c in pc.chunks)
        bt = sum(c.numel() * c.element_size() for c in pt.chunks)
        assert bc == -(-n // pc.chunk_frames) * pc.chunk_frames * pc.frame_elems               # one byte per code
        assert bt == -(-n // pt.chunk_frames) * pt.chunk_frames * pt.frame_elems * 2
        assert bc <= bt / 2 + pc.chunk_frames * pc.frame_elems                                  # up to chunk rounding
        assert comp.state(x).pinned_bytes() - bc == twin.state(y).pinned_bytes() - bt         # the rest is the same


# ---------------------------------------------------------------------------------------------------------- checkpoints
def test_checkpoints(rt, tower, merger, tmp_path):
    from flash_vstream_b200 import checkpoint as CK
    from flash_vstream_b200.qwen import QwenStreamPool
    host = host_for(rt, tower, merger)
    p = proc()
    eager = QwenStreamPool(host, preprocess=p)
    ea = eager.open(seed=1)
    made = {}
    for bank in (True, False):
        comp, twin = pools(host, p, bank)
        x, y = comp.open(seed=1), twin.open(seed=1)
        made[bank] = (comp, x, twin, y)
    size = (112, 112)
    for k in range(8):
        f = frames_of(50 + k, 2, size)
        eager.step({ea: f})
        for comp, x, twin, y in made.values():
            comp.step({x: f})
            twin.step({y: f})
            check_states(comp.state(x), eager.state(ea), ("pre", k))
    cks = {}
    for bank, (comp, x, twin, y) in made.items():
        ck = comp.checkpoint(x)
        assert ck.config["compact_pixels"] and "pixels" not in ck.tensors
        assert ck.tensor("pix_codes").dtype == torch.uint8 and ck.tensor("pix_codes").shape[0] == ck.counters["pix_frames"]
        assert torch.equal(ck.tensor("pixel_table"), p.device_table().cpu())
        ck_twin = twin.checkpoint(y)
        assert ck.nbytes() < ck_twin.nbytes()
        ck.save(tmp_path / f"{bank}.safetensors")
        cks[bank] = (CK.StreamCheckpoint.load(tmp_path / f"{bank}.safetensors"), ck_twin)
        with pytest.raises(NotImplementedError, match="compact_pixels"):            # tower-dtype rows -> compact
            comp.open(checkpoint=ck_twin)
        other = QwenStreamPool(host, preprocess=proc(image_mean=(0.5, 0.5, 0.5)), lazy_full_res=True,
                               full_res_bank=bank, compact_pixels=True)
        with pytest.raises(ValueError, match="pixel_table"):                         # codes of another table
            other.open(checkpoint=ck)
        with pytest.raises(NotImplementedError, match="lazy_full_res"):              # compact -> eager: today's rule
            eager.open(checkpoint=ck)
    # every legal direction, continued against the eager stream
    moved = {}
    for src in (True, False):
        ck = cks[src][0]
        for dst in (True, False):
            comp, _ = pools(host, p, dst, device_frames=2)
            moved[f"{src}->{dst} compact"] = (comp, comp.open(checkpoint=ck))
            _, plain = pools(host, p, dst)
            moved[f"{src}->{dst} decoded"] = (plain, plain.open(checkpoint=ck))
    e2c, _ = pools(host, p, True)
    moved["eager->compact"] = (e2c, e2c.open(checkpoint=eager.checkpoint(ea)))
    for k in range(6):
        f = frames_of(80 + k, (1, 16, 2)[k % 3], size)
        eager.step({ea: f})
        for tag, (pool, sid) in moved.items():
            pool.step({sid: f})
            check_states(pool.state(sid), eager.state(ea), (tag, k))


def test_pool_memory_manager(rt, tower, merger):
    from flash_vstream_b200.qwen.serve import pool_memory_manager
    host = host_for(rt, tower, merger)
    for bank in (True, False):
        comp, twin = pools(host, proc(), bank)
        r = random.Random(bank)
        clips = [[frames_of(100 * s + k, r.choice([1, 2, 4]), [(112, 112), (112, 168)][s % 2]) for k in range(6)]
                 for s in range(4)]
        sids = {}
        for pool in (comp, twin):
            qs = {}
            for s in range(4):
                sid = pool.open(seed=300 + s)
                qs[sid] = queue.Queue()
                for c in clips[s]:
                    qs[sid].put(c)
                qs[sid].put(None)
            counts = pool_memory_manager(pool, qs)
            assert counts == {sid: sum(c.shape[0] for c in clips[s]) for s, sid in enumerate(qs)}
            sids[id(pool)] = list(qs)
        for x, y in zip(sids[id(comp)], sids[id(twin)]):
            check_states(comp.state(x), twin.state(y), (bank, x))
