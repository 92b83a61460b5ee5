"""CPU tests of a Qwen2-VL stream without a full-resolution bank (DESIGN.md §3.19): the pick plan against the previous
DAM restated in NumPy (what the GPU tests hold fvs_qwen_pick_plan_multi and a bank-less stream's encode counts to),
the count the host knows while the DAM is the whole bank, the knob's refusals, the checkpoint's tensor set, and the
refusals of the plan and gather jobs a bank-less stream sends (returned before any CUDA call, nothing launched)."""
import numpy as np
import pytest
import torch

from flash_vstream_b200 import _lib as L

A = 0x10000          # a 16-byte aligned stand-in address: the refusals happen before anything is dereferenced


def np_plan_prev(picks, prev, frames):
    """picks: the DAM's frame indices in pick order; prev: the previous DAM's (or None); frames: uint8 byte per frame
    (0 never encoded, 1 encoded before, 2 rows stored in the base bank), updated in place -> (the frames encoded now:
    picks in range, not in prev, not stored, unique, in pick order; how many of them were encoded before)"""
    n = len(frames)
    held = set() if prev is None else {int(p) for p in prev}
    out, again = [], 0
    for p in picks:
        p = int(p)
        if 0 <= p < n and frames[p] != 2 and p not in held and p not in out:
            again += int(frames[p] == 1)
            frames[p] = 1
            out.append(p)
    return np.asarray(out, dtype=np.int64), again


def test_plan_skips_the_previous_dam_duplicates_and_the_base():
    fr = np.zeros(12, np.uint8)
    fr[[0, 1]] = 2                                                   # a base bank of two frames
    fr[[5, 6]] = 1                                                   # encoded before, since left the DAM
    plan, again = np_plan_prev([6, 0, 3, 3, 9, 5, 1, 7, 9], [3, 7], fr)
    assert plan.tolist() == [6, 9, 5] and again == 2
    assert fr.tolist() == [2, 2, 0, 0, 0, 1, 1, 0, 0, 1, 0, 0]
    plan, again = np_plan_prev([9, 6, 5], [6, 9, 5], fr)             # all picks in the previous DAM
    assert plan.tolist() == [] and again == 0
    plan, again = np_plan_prev([9, 2], [4], fr)                      # none in it: 9 comes back, 2 is new
    assert plan.tolist() == [9, 2] and again == 1


def test_plan_out_of_range_picks_are_skipped():
    fr = np.zeros(4, np.uint8)
    assert np_plan_prev([-1, 4, 2, 2, 100], None, fr)[0].tolist() == [2]


@pytest.mark.parametrize("base", [0, 3])
def test_whole_bank_count_is_what_the_host_knows(base):
    """while n <= spatial_length the DAM is frames [0, n) and the previous one [0, m): the plan is n - m frames, the
    count encode_picked takes without waiting"""
    fr = np.zeros(base, np.uint8) + 2
    m = base
    for t in (1, 2, 3):
        fr = np.concatenate([fr, np.zeros(t, np.uint8)])
        n = len(fr)
        plan, again = np_plan_prev(np.arange(n), np.arange(m) if m else None, fr)
        assert len(plan) == n - m and plan.tolist() == list(range(m, n)) and again == 0
        m = n


def test_plan_random_against_a_direct_statement():
    r = np.random.default_rng(1)
    for _ in range(200):
        n = int(r.integers(1, 80))
        fr = r.choice(np.array([0, 1, 2], np.uint8), n)
        picks = r.integers(-2, n + 2, int(r.integers(1, 40)))
        prev = r.integers(0, n, int(r.integers(0, 30)))
        before = fr.copy()
        plan, again = np_plan_prev(picks, prev, fr)
        want = []
        for p in picks:
            if 0 <= p < n and before[p] != 2 and p not in prev and p not in want:
                want.append(int(p))
        assert plan.tolist() == want
        assert again == sum(before[p] == 1 for p in want)
        assert all(fr[p] == 1 for p in want) and np.array_equal(np.delete(fr, want), np.delete(before, want))


def _flash(**kw):
    from flash_vstream_b200.qwen.vstream_qwen2vl_realtime import FlashMemory
    return FlashMemory(flash_memory_temporal_length=8, flash_memory_spatial_length=6, **kw)


def test_knob_refusals():
    from flash_vstream_b200.qwen.stream_state import QwenStreamState, check_full_res_bank
    with pytest.raises(ValueError, match="full_res_bank=False needs lazy_full_res=True"):
        QwenStreamState(_flash(), None, full_res_bank=False)
    for bad in (0, None, "no"):
        with pytest.raises(ValueError, match="full_res_bank must be True or False"):
            QwenStreamState(_flash(), None, lazy_full_res=True, full_res_bank=bad)
    st = QwenStreamState(_flash(), None, lazy_full_res=True, full_res_bank=False)
    assert not st.full_res_bank and st.lazy_full_res
    assert QwenStreamState(_flash(), None).full_res_bank                     # the default is untouched
    with pytest.raises(ValueError, match="fvs_full_res_bank=False needs fvs_lazy_full_res=True"):
        check_full_res_bank(False, False, "fvs_full_res_bank", "fvs_lazy_full_res")


def test_pool_and_host_defaults():
    from flash_vstream_b200.qwen.vstream_qwen2vl_realtime import FlashVStreamQwen2VLRealtimeB200
    assert FlashVStreamQwen2VLRealtimeB200.fvs_full_res_bank is True
    import inspect
    from flash_vstream_b200.qwen import QwenStreamPool
    assert inspect.signature(QwenStreamPool).parameters["full_res_bank"].default is True


def _ckpt(encoded, bank_frames, n_spa=2):
    from flash_vstream_b200 import checkpoint as CK
    n, h, w, hs, ws, D = len(encoded), 4, 4, 2, 2, 16
    cfg = {"flash": dict(_flash().config), "grid": [h, w], "small_grid": [hs, ws], "dtype": "bfloat16", "dim": D,
           "merger_dim": None}
    enc = np.asarray(encoded)
    cnt = {"n_frames": n, "steps": n, "n_tem": 2, "n_spa": n_spa, "fast_steps": 0, "redone_steps": 0, "merged": 0,
           "tem_weights_dtype": "float32", "tem_timestamp_dtype": "float32",
           "pix_frames": int(np.sum(enc != 2)), "bank_frames": bank_frames}
    bf = torch.bfloat16
    t = {"bank_x": torch.zeros(bank_frames, h * w, D, dtype=bf), "bank_small": torch.zeros(n, hs * ws, D, dtype=bf),
         "tem_x": torch.zeros(2 * hs * ws, D, dtype=bf), "tem_timestamp": torch.zeros(2), "tem_weights": torch.ones(2),
         "spa_positions": torch.zeros(n_spa, dtype=torch.int64), "encoded": torch.tensor(enc, dtype=torch.uint8),
         "pixels": torch.zeros(cnt["pix_frames"], h * w, 1176, dtype=bf), "spa_x": torch.zeros(n_spa, h * w, D, dtype=bf)}
    return CK.qwen(cfg, cnt, t, pin=False)


def test_checkpoint_tensor_set_and_refusals():
    from flash_vstream_b200 import checkpoint as CK
    from flash_vstream_b200.qwen.stream_state import QwenStreamState
    ck = _ckpt([2, 0, 2, 1, 0, 1], 3)                        # base of 3 frames (one not encoded when it was taken)
    lay = ck.layout()
    assert set(lay) == {"bank_x", "bank_small", "tem_x", "tem_timestamp", "tem_weights", "spa_positions", "encoded",
                        "pixels", "spa_x"}
    assert lay["bank_x"][0] == (3, 16, 16) and lay["pixels"][0] == (4, 16, 1176) and lay["spa_x"][0] == (2, 16, 16)
    assert lay["bank_small"][0] == (6, 4, 16) and lay["encoded"] == ((6,), torch.uint8)
    with pytest.raises(ValueError, match="'spa_x'"):
        CK.StreamCheckpoint(CK.QWEN, ck.config, ck.counters, {k: v for k, v in ck.tensors.items() if k != "spa_x"})
    with pytest.raises(ValueError, match="bank_frames"):
        CK.StreamCheckpoint(CK.QWEN, ck.config, dict(ck.counters, bank_frames=7), ck.tensors)
    flash = _flash()
    with pytest.raises(NotImplementedError, match="full_res_bank"):                  # bank-less -> eager
        QwenStreamState.restore(ck, flash, None, "cpu")
    bad = CK.StreamCheckpoint(CK.QWEN, ck.config, dict(ck.counters, pix_frames=3),
                              dict(ck.tensors, pixels=torch.zeros(3, 16, 1176, dtype=torch.bfloat16)))
    with pytest.raises(ValueError, match="pix_frames"):                                # rows that do not match the mask
        QwenStreamState.restore(bad, flash, None, "cpu", lazy_full_res=True, full_res_bank=False)
    enc = ck.tensors["encoded"].clone()
    enc[4] = 2                                                                         # "stored" past the base
    bad = CK.StreamCheckpoint(CK.QWEN, ck.config, dict(ck.counters, pix_frames=3),
                              dict(ck.tensors, encoded=enc, pixels=torch.zeros(3, 16, 1176, dtype=torch.bfloat16)))
    with pytest.raises(ValueError, match="past counters.bank_frames"):
        QwenStreamState.restore(bad, flash, None, "cpu", lazy_full_res=True)


def test_bankless_symbols_exported():
    lib = L.load()
    for name in ("fvs_qwen_pick_plan_multi", "fvs_qwen_dam_gather_multi"):
        assert hasattr(lib, name) and name in L.SIGNATURES


def _refused(fn, arr, *args, msg):
    lib = L.load()
    before = lib.fvs_launch_count()
    assert getattr(lib, fn)(arr, *args) == L.FVS_EINVAL
    assert msg in lib.fvs_last_error().decode()
    assert lib.fvs_launch_count() == before


@pytest.mark.parametrize("kw, msg", [
    (dict(n=-1), "bad sizes"),
    (dict(m=70000), "bad sizes"),
    (dict(picks=None, n=11), "null picks"),              # null picks stand for frames 0..n-1
    (dict(prev_picks=None), "null picks or previous"),
    (dict(frames=None), "null frame bytes"),
    (dict(count=None), "null frame bytes"),
    (dict(plan=A + 4), "misaligned"),
    (dict(re_encodes=A + 4), "misaligned"),
])
def test_bankless_plan_refusals_launch_nothing(kw, msg):
    a = dict(picks=A, n=4, n_frames=10, frames=A, prev_picks=A, m=2, plan=A, count=A, re_encodes=A, stored=2)
    a.update(kw)
    _refused("fvs_qwen_pick_plan_multi", (L.QwenPickPlanJob * 1)(L.QwenPickPlanJob(**a)), 1, None, msg=msg)


def test_bankless_plan_refuses_shared_outputs():
    a = dict(picks=A, n=4, n_frames=10, frames=A, prev_picks=A, m=2, plan=A, count=A, re_encodes=A, stored=2)
    jobs = (L.QwenPickPlanJob * 2)(L.QwenPickPlanJob(**a), L.QwenPickPlanJob(**dict(a, frames=2 * A)))
    _refused("fvs_qwen_pick_plan_multi", jobs, 2, None, msg="share an output")


def _fresh(**kw):
    a = dict(picks=A, n=4, n_frames=10, prev_picks=A, m=2, prev_x=A, prev_merged=A, fresh_frames=A, n_fresh=2, fresh_x=A,
             fresh_merged=A, n_base=5, dev_x=A, dev_merged=A, n_dev=3, host_chunks=A, chunk_frames=2, x_frame_elems=64,
             merged_frame_elems=32, spa_x_out=A, merged_out=A, host_fetches=A)
    a.update(kw)
    return L.QwenGatherJob(**a)


@pytest.mark.parametrize("kw, msg", [
    (dict(picks=None), "need picks"),
    (dict(n=0), "0 < n"),
    (dict(spa_x_out=None, merged_out=None), "no output"),
    (dict(n_base=11), "n_base <= n_frames"),
    (dict(n_dev=6), "n_dev <= n_base"),
    (dict(x_frame_elems=60), "16 bytes"),
    (dict(merged_frame_elems=0), "merged_out without"),
    (dict(prev_x=None), "previous DAM"),
    (dict(fresh_x=None), "fresh rows"),
    (dict(fresh_merged=None), "fresh rows"),
    (dict(n_fresh=-1), "fresh rows"),
    (dict(dev_x=None), "device tier"),
    (dict(host_chunks=None), "chunk table"),
    (dict(fresh_x=A + 8), "aligned"),
    (dict(fresh_frames=A + 4), "8-byte"),
])
def test_bankless_gather_refusals_launch_nothing(kw, msg):
    _refused("fvs_qwen_dam_gather_multi", (L.QwenGatherJob * 1)(_fresh(**kw)), 1, L.BF16, None, msg=msg)


def test_bankless_gather_refuses_dtype_and_shared_outputs():
    _refused("fvs_qwen_dam_gather_multi", (L.QwenGatherJob * 1)(_fresh()), 1, L.F32, None, msg="dtype")
    jobs = (L.QwenGatherJob * 2)(_fresh(), _fresh(merged_out=1 << 30, host_fetches=1 << 29))
    _refused("fvs_qwen_dam_gather_multi", jobs, 2, L.BF16, None, msg="share an output")
