"""CPU tests of the lazy full-resolution bank of a Qwen2-VL stream (DESIGN.md §3.18): the pick plan restated in NumPy
(what the GPU tests hold fvs_qwen_pick_plan_multi and a lazy stream's encode count to), the knob's refusals and the
checkpoint layout of a lazy stream."""
import numpy as np
import pytest
import torch


def np_plan(picks, encoded):
    """picks: the DAM's frame indices in pick order (None: the whole bank, frames 0..len(encoded)-1); encoded: bool mask
    per frame, updated in place -> the frames encoded now: first-time frames, unique, in pick order"""
    n = len(encoded)
    seq = range(n) if picks is None else picks
    out = []
    for p in seq:
        p = int(p)
        if 0 <= p < n and not encoded[p]:
            encoded[p] = True
            out.append(p)
    return np.asarray(out, dtype=np.int64)


def test_plan_first_time_frames_in_pick_order():
    enc = np.zeros(10, bool)
    enc[[1, 4]] = True
    assert np_plan([7, 1, 3, 7, 4, 9, 3, 0], enc).tolist() == [7, 3, 9, 0]
    assert enc[[0, 1, 3, 4, 7, 9]].all() and not enc[[2, 5, 6, 8]].any()
    assert np_plan([7, 3, 9], enc).tolist() == []                   # picked before: never encoded again


def test_plan_fill_phase_is_the_new_frames():
    enc = np.zeros(0, bool)
    total = 0
    for t in (1, 3, 2):                                              # the DAM is the whole bank while it is filling
        enc = np.concatenate([enc, np.zeros(t, bool)])
        got = np_plan(None, enc)
        assert got.tolist() == list(range(len(enc) - t, len(enc)))
        total += len(got)
    assert total == len(enc) and enc.all()


def test_plan_out_of_range_picks_are_skipped():
    enc = np.zeros(4, bool)
    assert np_plan([-1, 4, 2, 2, 100], enc).tolist() == [2]


def _flash(**kw):
    from flash_vstream_b200.qwen.vstream_qwen2vl_realtime import FlashMemory
    return FlashMemory(flash_memory_temporal_length=8, flash_memory_spatial_length=6, **kw)


def test_refusals():
    from flash_vstream_b200.qwen.stream_state import QwenStreamState, check_lazy_full_res
    with pytest.raises(NotImplementedError, match="lazy_full_res.*temporal_poolsize"):
        QwenStreamState(_flash(flash_memory_temporal_poolsize=1), None, lazy_full_res=True)
    QwenStreamState(_flash(flash_memory_temporal_poolsize=1), None, lazy_full_res=False)     # the default is untouched
    for bad in (1, None, "yes"):
        with pytest.raises(ValueError, match="lazy_full_res"):
            QwenStreamState(_flash(), None, lazy_full_res=bad)
    with pytest.raises(NotImplementedError, match="fvs_lazy_full_res"):
        check_lazy_full_res(True, _flash(flash_memory_temporal_poolsize=1), "fvs_lazy_full_res")
    from flash_vstream_b200.qwen.vstream_qwen2vl_realtime import FlashMemory
    st = QwenStreamState(FlashMemory(flash_memory_spatial_length=0), None, lazy_full_res=True)   # never encodes
    assert st.lazy_full_res and st.n_encoded == 0


def _lazy_ckpt(encoded):
    from flash_vstream_b200 import checkpoint as CK
    n, h, w, hs, ws, D = len(encoded), 4, 4, 2, 2, 16
    flash = _flash()
    cfg = {"flash": dict(flash.config), "grid": [h, w], "small_grid": [hs, ws], "dtype": "bfloat16", "dim": D,
           "merger_dim": None}
    cnt = {"n_frames": n, "steps": n, "n_tem": 2, "n_spa": 2, "fast_steps": 0, "redone_steps": 0, "merged": 0,
           "tem_weights_dtype": "float32", "tem_timestamp_dtype": "float32",
           "pix_frames": int(np.sum(np.asarray(encoded) == 0))}
    bf = torch.bfloat16
    t = {"bank_x": torch.zeros(n, h * w, D, dtype=bf), "bank_small": torch.zeros(n, hs * ws, D, dtype=bf),
         "tem_x": torch.zeros(2 * hs * ws, D, dtype=bf), "tem_timestamp": torch.zeros(2), "tem_weights": torch.ones(2),
         "spa_positions": torch.zeros(2, dtype=torch.int64), "encoded": torch.tensor(encoded, dtype=torch.uint8),
         "pixels": torch.zeros(cnt["pix_frames"], h * w, 1176, dtype=bf)}
    return flash, CK.qwen(cfg, cnt, t, pin=False)


def test_lazy_checkpoint_layout_and_lazy_to_eager_refusal():
    from flash_vstream_b200 import checkpoint as CK
    from flash_vstream_b200.qwen.stream_state import QwenStreamState
    flash, ck = _lazy_ckpt([1, 0, 1])
    assert ck.layout()["encoded"] == ((3,), torch.uint8) and ck.layout()["pixels"][0] == (1, 16, 1176)
    with pytest.raises(ValueError, match="'pixels'"):
        CK.StreamCheckpoint(CK.QWEN, ck.config, ck.counters, {k: v for k, v in ck.tensors.items() if k != "pixels"})
    with pytest.raises(NotImplementedError, match="lazy_full_res"):
        QwenStreamState.restore(ck, flash, None, "cpu")
    bad = CK.StreamCheckpoint(CK.QWEN, ck.config, dict(ck.counters, pix_frames=2),
                              dict(ck.tensors, pixels=torch.zeros(2, 16, 1176, dtype=torch.bfloat16)))
    with pytest.raises(ValueError, match="pix_frames"):                # rows that do not match the mask
        QwenStreamState.restore(bad, flash, None, "cpu", lazy_full_res=True)
