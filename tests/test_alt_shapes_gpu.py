"""GPU parity of the alternate temporal compressors at the shapes and magnitudes a video produces (tests/alt_shapes_inputs.py):
the product mirror (compress_functions.*) bit for bit against oracle/alternates_oracle.py, the refusals that must launch
nothing, and the model-level glue of every alternate `video_sample_type` (offline and streaming) against the extended
oracle (fvs_oracle.compress_temporal_features / stream_step with a compressor)."""
from __future__ import annotations

import random

import numpy as np
import pytest
import torch

from oracle import fvs_oracle as O
from tests import alt_shapes_inputs as AS
from tests import golden_inputs as GI
from tests.test_alt_shapes_host import ALT_NAMES, coin_count, expected_exception, oracle_compressor, run_oracle
from tests.test_oracle_golden import ulp_diff_f16

pytestmark = pytest.mark.gpu

DROPS = ("drop_feature", "k_drop_feature")


@pytest.fixture(scope="module")
def lib():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    from flash_vstream_b200 import _lib
    return _lib.load(build_if_missing=False)


def bits(t):
    return t.detach().cpu().contiguous().view(torch.int16).numpy()


def run_product(name):
    """(feat, sim, steps, (labels, info) | None) of the product on case `name`"""
    from flash_vstream_b200 import compress_functions as mcf
    from flash_vstream_b200 import ops
    c = AS.CASES[name]
    x = AS.features(name).cuda()
    s = AS.sim_in(name)
    s = None if s is None else s.cuda()
    if c["fn"] == "kmeans_feature":
        init, refill = AS.kmeans_draws(name)
        feat, sim, steps = mcf.kmeans_feature(x, c["T0"], init_idx=init, refill_idx=refill)
        _, labels, info = ops.alt_kmeans(x.view(c["T"], -1), torch.from_numpy(init).cuda(), torch.from_numpy(refill).cuda(),
                                         c["T0"], AS.MAX_ITER)
        return feat, sim, steps, (labels.cpu().numpy(), info.cpu().numpy())
    if c["fn"] in DROPS:
        kw = dict(coins=AS.coins(name))
        if c["fn"] == "drop_feature":
            kw["img_similarity"] = s
        return (*getattr(mcf, c["fn"])(x, c["T0"], **kw), None)
    return (*getattr(mcf, c["fn"])(x, c["T0"], s), None)


@pytest.mark.parametrize("name", list(AS.CASES))
def test_alternate_shapes_parity(lib, name):
    c = AS.CASES[name]
    o_feat, o_sim, o_steps, res = run_oracle(name)
    feat, sim, steps, km = run_product(name)
    assert steps == o_steps                                                     # every step's member lists (pos / kept)
    assert np.array_equal(bits(feat), np.asarray(o_feat, np.float16).view(np.int16))
    if o_sim is None:
        assert sim is None
    else:
        assert np.array_equal(bits(sim), np.asarray(o_sim, np.float16).view(np.int16))
    if km is not None:
        labels, info = km
        assert np.array_equal(labels, res["labels"])
        assert (int(info[0]), int(info[1]), int(info[2])) == (res["exit_step"], res["refills"], int(res["converged"]))
        print(f"\n[{name}] |x|^2 = inf on {res['xn_inf'][0]:.0%} of the rows, NaN distances in "
              f"{sum(res['dist_nan'])} of {len(res['dist_nan'])} iterations; exit step {res['exit_step']}, "
              f"{res['refills']} refills, converged {res['converged']}")
    again = run_product(name)                                                   # a second identical call: identical bits
    assert again[2] == steps and torch.equal(again[0].view(torch.int16), feat.view(torch.int16))
    if sim is not None:
        assert torch.equal(again[1].view(torch.int16), sim.view(torch.int16))


# ------------------------------------------------------------------------------------------------ refusals: no launch
@pytest.mark.parametrize("method", ["ALT_DROP", "ALT_MERGE", "ALT_KDROP", "ALT_KMERGE"])
def test_sequential_refusals_launch_nothing(lib, method):
    from flash_vstream_b200 import _lib as L
    from flash_vstream_b200 import ops
    m = getattr(ops, method)
    cases = (("T0 = 1024", 1030, 1024, 1024), ("PD not a multiple of 1024", 30, 25, 1536),
             ("PD = 2^20 + 1024", 4, 2, (1 << 20) + 1024), ("T = T0", 25, 25, 1024))
    for what, T, T0, PD in cases:
        X = torch.randn(T, PD, device="cuda").half()
        coins = torch.zeros(max(T - T0, 1), dtype=torch.int32, device="cuda")
        torch.cuda.synchronize()
        n0 = lib.fvs_launch_count()
        with pytest.raises(ValueError):
            ops.alt_sequential(m, X, T0, coins)
        assert lib.fvs_launch_count() == n0, what
    # a workspace one byte short
    T, T0, PD = 30, 25, 2048
    X = torch.randn(T, PD, device="cuda").half()
    need = lib.fvs_alt_workspace_bytes(m, T, T0, PD)
    ws = torch.empty(need, dtype=torch.uint8, device="cuda")
    kept = torch.empty(T0, dtype=torch.int32, device="cuda")
    feat = torch.empty(T0, PD, dtype=torch.float16, device="cuda")
    sim = torch.empty(T0 * T0, dtype=torch.float16, device="cuda")
    pos = torch.empty(T - T0, dtype=torch.int32, device="cuda")
    coins = torch.zeros(T - T0, dtype=torch.int32, device="cuda")
    torch.cuda.synchronize()
    n0 = lib.fvs_launch_count()
    with pytest.raises(ValueError, match="workspace"):
        L.check(lib.fvs_alt_sequential(m, L.ptr(X), T, T0, PD, None, L.ptr(coins), L.ptr(kept), L.ptr(feat), L.ptr(sim),
                                       L.ptr(pos), L.ptr(ws), need - 1, L.F16, L.cur_stream()), "fvs_alt_sequential")
    assert lib.fvs_launch_count() == n0
    L.check(lib.fvs_alt_sequential(m, L.ptr(X), T, T0, PD, None, L.ptr(coins), L.ptr(kept), L.ptr(feat), L.ptr(sim),
                                   L.ptr(pos), L.ptr(ws), need, L.F16, L.cur_stream()), "fvs_alt_sequential")
    assert lib.fvs_launch_count() == n0 + 1                                   # the exact size is enough


def make_model(name, seed=5, **cfg):
    from flash_vstream_b200.vstream_arch import FlashVStreamB200, NeuralTuringMachine
    ntm = NeuralTuringMachine(1024, 32)
    GI.load_ntm(ntm, seed)
    model = FlashVStreamB200(None, ntm.half().cuda(), video_sample_type=name, **cfg)
    w = GI.ntm_weights(1024, 32, seed)
    return model, tuple(w[k].numpy() for k in ("q_w", "q_b", "k_w", "k_b"))


@pytest.fixture
def no_compressor_launch(monkeypatch):
    """a refused call must not reach the compressor kernels nor key retrieval"""
    from flash_vstream_b200 import ops

    def stub(*a, **k):
        raise AssertionError("a kernel was reached with a weight the reference cannot sort")
    for f in ("alt_sequential", "alt_kmeans", "key_retrieve", "argsort_desc"):
        monkeypatch.setattr(ops, f, stub)


def test_model_kmerge_refused_before_any_launch(lib, no_compressor_launch):
    """long memory of 59 rows, video_long_memory_length 25: k_merge's [25, 25] weight would be sorted flat into indices up
    to 624 and read past the long memory.  Rows already 4 x 4, so nothing but the compressor could launch."""
    feats = torch.randn(60, 16, 1024, device="cuda").half()
    for name in ("kmerge", "uni_kmerge", "both_kmerge", "split_kmerge"):
        model, _ = make_model(name, compress_size=4, compress_Turing_memory_size=4)
        torch.cuda.synchronize()
        n0 = lib.fvs_launch_count()
        if name == "kmerge":
            with pytest.raises(RuntimeError) as e:
                model.compress_temporal_features([feats])
            print(f"\n[offline {name}, T 59 > T0 25] {e.type.__name__}: {e.value}")
        model.consolidate_streaming(feats[:30])
        with pytest.raises(RuntimeError) as e:
            model.consolidate_streaming(feats[30:])
        print(f"[streaming {name}, T 60 > T0 25] {e.type.__name__}: {e.value}")
        assert lib.fvs_launch_count() == n0


# ------------------------------------------------------------------------------------------------ model level
def video(T, P, seed):
    g = torch.Generator().manual_seed(seed)
    scenes = torch.randn(6, P, 1024, generator=g)
    which = torch.sort(torch.randint(0, 6, (T,), generator=g)).values
    return (scenes[which] + 0.4 * torch.randn(T, P, 1024, generator=g)).half()


@pytest.mark.parametrize("name", ALT_NAMES)
def test_model_offline(lib, name, monkeypatch):
    """compress_temporal_features at the default STAR config (long 25 x 4^2, Turing 25 x 1^2), a 60-frame and a 20-frame
    video, against the extended oracle; the coins come from the global `random` and end where the reference's end"""
    for T in (60, 20):
        feat = video(T, 64, 40 + T)
        model, ntm = make_model(name)
        seed = 900 + T
        if name not in ("drop", "merge", "kmeans", "kdrop", "kmerge"):        # streaming-only aliases
            with pytest.raises(NotImplementedError):
                model.compress_temporal_features([feat.cuda()])
            continue
        want = expected_exception(name, T - 1, 25)
        rng = random.Random(seed)
        coins = [rng.randint(0, 1) for _ in range(coin_count(name, T - 1, 25))]   # drop, kdrop: one per incoming frame
        random.seed(seed)
        if want is not None:
            torch.cuda.synchronize()
            n0 = lib.fvs_launch_count()
            with monkeypatch.context() as mp:
                from flash_vstream_b200 import ops
                for f in ("alt_sequential", "alt_kmeans", "key_retrieve"):
                    mp.setattr(ops, f, lambda *a, **k: pytest.fail("a refused call reached a compressor kernel"))
                with pytest.raises(want) as e:
                    model.compress_temporal_features([feat.cuda()])
            assert lib.fvs_launch_count() == n0                                  # not even the pooling
            with pytest.raises(want):
                O.compress_temporal_features(feat.numpy(), O.StarConfig(), ntm, compressor=oracle_compressor(name, 25, coins))
            print(f"\n[offline {name}, long {T - 1} rows, T0 25] {e.type.__name__}: {e.value}")
            assert random.random() == rng.random()                               # the reference's draws, no more
            continue
        mem = model.compress_temporal_features([feat.cuda()])[0]
        omem, _ = O.compress_temporal_features(feat.numpy(), O.StarConfig(), ntm, compressor=oracle_compressor(name, 25, coins))
        assert random.random() == rng.random()                                  # the coins the reference draws, no more
        mem = mem.cpu().numpy()
        assert mem.shape == omem.shape == (25 + 25 * 16 + 4 * 64, 1024)
        assert np.array_equal(mem[25:].view(np.int16), omem[25:].view(np.int16))     # long + key + cur rows
        assert ulp_diff_f16(mem[:25], omem[:25]).max() <= 4                          # Turing rows: GEMM rule


@pytest.mark.parametrize("name", ALT_NAMES)
@pytest.mark.parametrize("long_len", [4, 25])
def test_model_streaming(lib, name, long_len, monkeypatch):
    """op-by-op consolidate_streaming, chunks of 4 frames: with long 4 every compression sees T = 8 > T0 (drop and merge
    run, the others raise on the second call); with long 25 the second call compresses 8 <= 25 rows and every name raises"""
    from flash_vstream_b200 import ops
    model, ntm = make_model(name, video_long_memory_length=long_len)
    cfg = O.StarConfig(long_len=long_len)
    seed = 77 + long_len
    rng = random.Random(seed)
    random.seed(seed)
    st = O.StreamState()
    frames = video(28, 576, 300 + long_len)
    for s in range(7):
        f576 = frames[4 * s:4 * s + 4]
        want = expected_exception(name, 8, long_len) if s > 0 else None
        coins = [rng.randint(0, 1) for _ in range(coin_count(name, 8, long_len))] if s > 0 else []
        if want is not None:
            before = list(model.video_embedding_memory)
            n_buf = model.__dict__["_fvs_buf"]["n"]
            x = f576.cuda()
            torch.cuda.synchronize()
            n0 = lib.fvs_launch_count()
            with monkeypatch.context() as mp:
                for f in ("alt_sequential", "alt_kmeans", "key_retrieve"):
                    mp.setattr(ops, f, lambda *a, **k: pytest.fail("a refused call reached a compressor kernel"))
                with pytest.raises(want) as e:
                    model.consolidate_streaming(x)
            assert lib.fvs_launch_count() == n0                                  # not even the pooling
            with pytest.raises(want):
                O.stream_step(st, O.spatial_pool(f576.numpy(), 8), cfg, ntm,
                              compressor=oracle_compressor(name, long_len, coins))
            assert all(a is b for a, b in zip(before, model.video_embedding_memory))      # the stream is as it was
            assert model.__dict__["_fvs_buf"]["n"] == n_buf                              # the chunk is not buffered
            print(f"\n[streaming {name}, long {long_len}, call {s}] {e.type.__name__}: {e.value}")
            break
        model.consolidate_streaming(f576.cuda())
        st, _ = O.stream_step(st, O.spatial_pool(f576.numpy(), 8), cfg, ntm,
                              compressor=oracle_compressor(name, long_len, coins))
        cur, lng, tur, buf = model.video_embedding_memory
        assert np.array_equal(bits(cur), st.cur.view(np.int16)), s              # key + current frames
        assert np.array_equal(bits(lng), st.long.view(np.int16)), s             # long memory
        assert ulp_diff_f16(tur.cpu().numpy(), st.tur).max() <= 4, s            # Turing rows: GEMM rule
        assert buf.shape[0] == 4 * (s + 1)
    else:
        assert name in ("drop", "merge") and long_len == 4
    assert random.random() == rng.random()                                      # draws end where the reference's end
