"""GPU parity tests of the Qwen2-VL Flash Memory (pytest -m gpu on the GPU).  Every test calls the product mirror
(flash_vstream_b200.qwen) -> C ABI -> sm_90a kernels and compares with (a) oracle/qwen_oracle.py on the same seeded inputs
(bit-exact: every op and summation order is specified) and (b) the goldens recorded from the reference (exact for indices,
timestamps, position ids and pooled pixels; one output-dtype rounding for k-means centroids, whose fp32 summation order
differs from ATen's)."""
import numpy as np
import pytest
import torch

from oracle import qwen_oracle as QO
from tests import qwen_inputs as QI
from tests.test_qwen_oracle_golden import _load, _members, assert_close_dtype

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def qwen():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    from flash_vstream_b200 import _lib
    _lib.load(build_if_missing=False)  # the prebuilt in-tree .so must be what runs
    import flash_vstream_b200.qwen as pkg
    from flash_vstream_b200.qwen import ops as qops
    return pkg, qops


def same_bits(a: torch.Tensor, b: torch.Tensor):
    a, b = a.detach().cpu().contiguous(), b.detach().cpu().contiguous()
    assert a.dtype == b.dtype and a.shape == b.shape, (a.dtype, b.dtype, a.shape, b.shape)
    assert torch.equal(a.view(torch.uint8), b.view(torch.uint8)), f"{(a != b).float().mean().item():.4f} of elements differ"


# ------------------------------------------------------------------------------------------------ temporal_pool
@pytest.mark.parametrize("case", QI.POOL_CASES, ids=[c[0] for c in QI.POOL_CASES])
def test_temporal_pool_bit_exact(qwen, case):
    pkg, _ = qwen
    name, t, h, w, dt, seed = case
    g = _load("qwen_pool.npz")
    x = QI.pool_input(t, h, w, dt, seed)
    fm = pkg.FlashMemory()
    y, thw = fm.temporal_pool(x.cuda(), torch.tensor([t, h, w]).cuda())
    assert thw.tolist() == g[name + "_thw"].tolist()
    assert np.array_equal(QI.to_bits(y.cpu()), g[name + "_y"])          # the reference's own output
    same_bits(y, QO.temporal_pool(x, [t, h, w])[0])


def test_temporal_pool_full_size_and_errors(qwen):
    pkg, _ = qwen
    fm = pkg.FlashMemory()
    t, h, w = 8, 24, 24                                               # 8 temporal patches of a 336x336 clip
    x = QI.pool_input(t, h, w, "bf16", 77)
    y, thw = fm.temporal_pool(x.cuda(), torch.tensor([t, h, w]).cuda())
    assert thw.tolist() == [t, 12, 12] and y.shape == (t * 144, 1176)
    same_bits(y, QO.temporal_pool(x, [t, h, w])[0])
    # mean preservation: the pooled clip has the same per-(frame, channel-plane) mean as the source (fp32 check)
    src = x.float().reshape(t, -1, 6, 196).mean(dim=(1, 3))
    dst = y.float().cpu().reshape(t, -1, 6, 196).mean(dim=(1, 3))
    assert torch.allclose(src, dst, atol=2e-3)
    with pytest.raises(NotImplementedError):
        fm.temporal_pool(torch.zeros(6 * 4, 1176, dtype=torch.bfloat16).cuda(), torch.tensor([1, 6, 4]).cuda())


# ------------------------------------------------------------------------------------------------ unique rows
def test_unique_rows_matches_torch_unique(qwen):
    _, qops = qwen
    g = torch.Generator().manual_seed(9)
    for dt in (torch.bfloat16, torch.float32):
        base = torch.randn(7, 2048, generator=g).to(dt)
        base[1, :2000] = base[0, :2000]                              # rows that differ only near the end
        X = base[torch.randint(0, 7, (23,), generator=g)]
        idx, n = qops.unique_rows(X.cuda())
        n = int(n.item())
        got = X[idx[:n].cpu().long()]
        assert torch.equal(got, torch.unique(X.float(), dim=0).to(dt))
        assert np.array_equal(idx[:n].cpu().numpy(), QO.unique_rows_order(X.float().numpy()))


# ------------------------------------------------------------------------------------------------ ordered k-means
@pytest.mark.parametrize("name", list(QI.KMEANS_CASES))
def test_kmeans_ordered_parity(qwen, name):
    pkg, _ = qwen
    c = QI.KMEANS_CASES[name]
    g = _load("qwen_kmeans.npz")
    x, w = QI.kmeans_input(c)
    kw = dict(init_idx=g[name + "_init"], refill_idx=g[name + "_refill"])
    feat, weights, ts, idx = pkg.weighted_kmeans_ordered_feature(x.cuda(), c["K"], None if w is None else w.cuda(),
                                                                 order=g[name + "_order"] if c["kind"] != "degenerate" else None,
                                                                 **kw)
    o_feat, o_w, o_ts, o_idx = QO.weighted_kmeans_ordered_feature(x, c["K"], w, **kw)
    # (a) oracle: bit-exact
    assert idx == o_idx
    same_bits(feat, o_feat)
    same_bits(weights.float(), o_w)
    same_bits(ts.float(), o_ts)
    # (b) reference golden
    assert idx == _members(g, name)
    assert np.array_equal(ts.cpu().numpy(), g[name + "_ts"])
    np.testing.assert_allclose(weights.cpu().numpy(), g[name + "_weights"], rtol=1e-5)
    assert_close_dtype(feat.cpu(), QI.from_bits(g[name + "_feat"], feat.dtype), c["dtype"])


def test_kmeans_ordered_pass_through_and_rng(qwen):
    pkg, _ = qwen
    import random
    x = torch.randn(4, 2, 512).bfloat16().cuda()
    out = pkg.weighted_kmeans_ordered_feature(x, 6)
    assert len(out) == 3 and out[0].dtype == torch.float32 and out[2] == [[[0], [1], [2], [3]]]
    # default draws come from torch / random exactly like the reference: same seeds -> same result, and Python's `random`
    # is left advanced by the number of refills actually consumed (0 here)
    c = QI.KMEANS_CASES["ko_scene_bf16"]
    xs, _ = QI.kmeans_input(c)
    res = []
    for _ in range(2):
        torch.manual_seed(3)
        random.seed(3)
        feat, wts, ts, idx = pkg.weighted_kmeans_ordered_feature(xs.cuda(), c["K"])
        after = random.random()
        res.append((feat.cpu(), idx, after))
    assert torch.equal(res[0][0], res[1][0]) and res[0][1] == res[1][1]
    random.seed(3)
    assert res[0][2] == random.random()


def test_kmeans_ordered_draws_after_pending_llava_refills(qwen):
    """Python's `random` is one generator for both model families: the refills a LLaVA k-means consumed, still pending
    (weighted_kmeans_device reads the count back asynchronously), are applied before a Qwen k-means draws its candidates,
    so the Qwen draws are the ones the reference's single `random` would give"""
    pkg, _ = qwen
    import random
    from flash_vstream_b200 import compress_functions as LCF
    name = "ko_zero_weight_f32"                                       # zero weights: clusters get refilled
    c = QI.KMEANS_CASES[name]
    x, w = QI.kmeans_input(c)
    init = _load("qwen_kmeans.npz")[name + "_init"]
    LCF.sync_rng()
    random.seed(17)
    rows = torch.ones(10, 4, 256, dtype=torch.float16, device="cuda")   # identical rows: every cluster but one empties
    *_, info = LCF.weighted_kmeans_device(rows, 4)                     # no sync_rng(): its refill count stays pending
    got = pkg.weighted_kmeans_ordered_feature(x.cuda(), c["K"], w.cuda(), init_idx=init)
    consumed = int(info[1])
    assert consumed > 0

    def with_refills_after(skip):
        random.seed(17)
        for _ in range(skip):
            random.randint(0, rows.shape[0] - 1)
        refill = [random.randint(0, c["T"] - 1) for _ in range(10 * c["K"])]
        return pkg.weighted_kmeans_ordered_feature(x.cuda(), c["K"], w.cuda(), init_idx=init, refill_idx=refill)
    want, unsettled = with_refills_after(consumed), with_refills_after(0)
    assert got[3] != unsettled[3], "the input must be one on which the LLaVA refills change the Qwen result"
    assert got[3] == want[3]
    for a, b in zip(got[:3], want[:3]):
        same_bits(a, b)


def test_kmeans_ordered_full_size_properties(qwen):
    """BASELINE-size CSM update: 61 half-resolution frames of 144 tokens x 1280 -> 60 centroids (PD = 184320)."""
    pkg, _ = qwen
    g = torch.Generator().manual_seed(123)
    T, P, D, K = 61, 144, 1280, 60
    scenes = torch.randn(40, P, D, generator=g)
    which = torch.sort(torch.randint(0, 40, (T,), generator=g)).values
    x = (scenes[which] + 0.3 * torch.randn(T, P, D, generator=g)).bfloat16().cuda()
    torch.manual_seed(1)
    feat, weights, ts, idx = pkg.weighted_kmeans_ordered_feature(x, K)
    assert feat.shape == (K, P, D) and feat.dtype == torch.bfloat16
    assert sorted(j for m in idx for j in m) == list(range(T))        # the member lists partition the frames
    assert all(len(m) > 0 for m in idx)
    assert float(weights.sum()) == float(T)                           # unit weights: exact in fp32
    tsc = ts.cpu().numpy()
    assert (np.diff(tsc) >= 0).all()                                  # ordered by mean member index
    assert np.allclose(tsc, [sum(m) / len(m) for m in idx])
    # every centroid is the mean of its members unless the loop stopped on the tolerance (old centroids kept): singletons
    # must equal their frame exactly in both cases
    xf = x.float()
    for k, m in enumerate(idx):
        if len(m) == 1:
            assert torch.equal(feat[k], x[m[0]])
        else:
            mean = xf[m].mean(dim=0)
            assert (feat[k].float() - mean).norm() / mean.norm() < 0.75   # stays inside its cluster


# ------------------------------------------------------------------------------------------------ retrieval pieces
@pytest.mark.parametrize("dt", ["bf16", "f16"])
def test_klarge_retrieve_bit_exact(qwen, dt):
    """distances (every rounding step) and the argmin against the oracle; includes exact duplicates of bank frames, whose
    16-bit radicand can round to a small negative number -> NaN -> wins the argmin (torch semantics)"""
    _, qops = qwen
    g = torch.Generator().manual_seed(41)
    tdt = QI.DT[dt]
    bank = (torch.randn(37, 4096, generator=g) * 0.5).to(tdt)
    tem = torch.zeros(9, 4096, dtype=tdt)
    tem[:5] = bank[[3, 30, 11, 3, 22]] + (0.05 * torch.randn(5, 4096, generator=g)).to(tdt)
    tem[5:] = bank[[7, 8, 9, 36]]                                      # exact copies
    kidx = torch.tensor([4, 0, 8, 2, 6, 1, 5])
    idx, dist = qops.klarge_retrieve(tem.cuda(), kidx.cuda(), bank.cuda(), want_dist=True)
    want = QO.klarge_distances(tem[kidx], bank)
    got = dist.cpu().numpy()
    assert np.array_equal(np.isnan(got), np.isnan(want))
    assert np.array_equal(got[~np.isnan(got)], want[~np.isnan(want)])
    assert np.array_equal(idx.cpu().numpy(), QO.argmin_first_nan(want, axis=1))
    sel = idx.cpu().tolist()
    assert [sel[i] for i in (0, 1, 3, 5)] == [22, 3, 11, 30]          # perturbed copies find their source frame
    # more than 64 centroids: swept in groups
    many = torch.randint(0, 9, (70,), generator=g)
    idx2 = qops.klarge_retrieve(tem.cuda(), many.cuda(), bank.cuda())
    assert np.array_equal(idx2.cpu().numpy(), QO.argmin_first_nan(QO.klarge_distances(tem[many], bank), axis=1))


@pytest.mark.parametrize("dt", ["bf16", "f16"])
def test_klarge_retrieve_cos_bit_exact(qwen, dt):
    """§8f-4 'klarge_retrieve_cos': similarities (norms, normalised rows, dot products: every rounding step) and the argmin
    of the similarity against the oracle, bit for bit; a zero bank row is 0/0 = NaN and wins (torch semantics)"""
    _, qops = qwen
    g = torch.Generator().manual_seed(43)
    tdt = QI.DT[dt]
    bank = (torch.randn(37, 4096, generator=g) * 0.5).to(tdt)
    bank[20:24] = (-bank[3:7].float() + 0.3 * torch.randn(4, 4096, generator=g)).to(tdt)   # anti-correlated with frames 3..6
    tem = torch.zeros(9, 4096, dtype=tdt)
    tem[:5] = bank[[3, 30, 5, 6, 22]] + (0.05 * torch.randn(5, 4096, generator=g)).to(tdt)
    tem[5:] = bank[[7, 8, 9, 36]]
    kidx = torch.tensor([4, 0, 8, 2, 6, 1, 3])
    idx, sim = qops.klarge_retrieve(tem.cuda(), kidx.cuda(), bank.cuda(), want_dist=True, metric="cosine")
    want = QO.klarge_cosine(tem[kidx], bank)
    assert not np.isnan(want).any()
    assert np.array_equal(sim.cpu().numpy(), want)
    assert np.array_equal(idx.cpu().numpy(), QO.argmin_first_nan(want, axis=1))
    sel = idx.cpu().tolist()
    assert [sel[i] for i in (1, 3, 6)] == [20, 22, 23]                 # the least similar frame = the anti-correlated one
    # NaN rule + more than 64 centroids (swept in groups)
    bank2 = bank.clone()
    bank2[11] = 0
    many = torch.randint(0, 9, (70,), generator=g)
    idx2, sim2 = qops.klarge_retrieve(tem.cuda(), many.cuda(), bank2.cuda(), want_dist=True, metric="cosine")
    want2 = QO.klarge_cosine(tem[many], bank2)
    assert np.isnan(want2[:, 11]).all()
    assert np.array_equal(np.isnan(sim2.cpu().numpy()), np.isnan(want2))
    assert (idx2.cpu().numpy() == 11).all()


@pytest.mark.parametrize("name", list(QI.COS_CASES))
def test_spatial_enhance_cos_matches_reference(qwen, name):
    """the mirror's FlashMemory(flash_memory_spatial_method='klarge_retrieve_cos').spatial_enhance against what the
    reference's returned (tests/golden/make_golden_qwen_cos.py): DAM positions and rows"""
    pkg, _ = qwen
    c = QI.COS_CASES[name]
    g = _load("qwen_klarge_cos.npz")
    x, small, thw, small_thw, pos, vis = QI.memory_input(c)
    dt = QI.DT[c["dtype"]]
    fm = pkg.FlashMemory(flash_memory_temporal_length=c["temporal_length"], flash_memory_spatial_length=c["spatial_length"],
                         flash_memory_spatial_method="klarge_retrieve_cos")
    tem_x = QI.from_bits(g[name + "_tem_x"], dt).cuda()
    tem_thw = torch.as_tensor(g[name + "_tem_thw"]).cuda()
    spa_x, spa_thw, spa_pos = fm.spatial_enhance(x.cuda(), small.cuda(), thw[0].cuda(), tem_x, tem_thw,
                                                 torch.from_numpy(g[name + "_tem_w"]).cuda(), None, None,
                                                 draws=dict(weight_order=g[name + "_sort1"]))
    assert np.array_equal(spa_pos.cpu().numpy(), g[name + "_spa_pos"])
    assert torch.equal(spa_x.reshape(-1, x.shape[-1]).cpu(), QI.from_bits(g[name + "_spa_x"], dt).reshape(-1, x.shape[-1]))


def test_am_rope_matches_oracle(qwen):
    pkg, _ = qwen
    fm = pkg.FlashMemory()
    spa_thw, tem_thw = torch.tensor([3, 4, 6]), torch.tensor([5, 2, 4])
    spa_pos, tem_pos = torch.tensor([7, 2, 11]), torch.tensor([0, 3, 4, 9, 10])
    n = 3 * 2 * 3 + 5 * 1 * 2
    L = 4 + n + 2
    pos = (torch.arange(L) + 13).view(1, L).expand(3, L).clone()
    vis = torch.full((L,), -1, dtype=torch.long)
    vis[4:4 + n] = torch.arange(n)
    want = QO.FlashMemoryOracle.calc_am_rope(pos, vis, tem_thw, tem_pos, spa_thw, spa_pos)
    got = fm.calc_am_rope(pos.clone().cuda(), vis.cuda(), tem_thw.cuda(), tem_pos.cuda(), spa_thw.cuda(), spa_pos.cuda())
    assert torch.equal(got.cpu(), want)


# ------------------------------------------------------------------------------------------------ FlashMemory.forward
@pytest.mark.parametrize("name", list(QI.MEMORY_CASES))
def test_flash_memory_forward_parity(qwen, name):
    pkg, _ = qwen
    c = QI.MEMORY_CASES[name]
    g = _load("qwen_memory.npz")
    x, small, thw, small_thw, pos, vis = QI.memory_input(c)
    fm = pkg.FlashMemory(flash_memory_temporal_length=c["temporal_length"], flash_memory_spatial_length=c["spatial_length"])
    two = int(g[name + "_n_sorts"][0]) >= 2
    draws = [dict(init_idx=g[name + "_init"], refill_idx=g[name + "_refill"], ts_order=g[name + "_sort0"] if two else None,
                  weight_order=g[name + "_sort1"] if two else None)]
    new_x, new_pos = fm(torch.cat([x, small]).cuda(), thw.cuda(), small_thw.cuda(), pos.clone().cuda(), vis.cuda(), draws=draws)
    # (b) the reference's own outputs
    assert np.array_equal(new_pos.cpu().numpy(), g[name + "_new_pos"])
    assert_close_dtype(new_x[0].cpu(), QI.from_bits(g[name + "_new_x"], new_x.dtype), c["dtype"])
    # (a) oracle, bit-exact
    orc = QO.FlashMemoryOracle(c["temporal_length"], c["spatial_length"])
    o_x, o_pos, aux = orc.forward_one(x, thw[0], small, small_thw[0], pos[:, 0], vis[0], init_idx=g[name + "_init"],
                                      refill_idx=g[name + "_refill"], order=g[name + "_sort1"] if two else None)
    same_bits(new_x[0], o_x)
    assert torch.equal(new_pos[:, 0].cpu(), o_pos)
    # DAM positions equal the reference's
    n_spa = len(g[name + "_spa_pos"])
    assert new_pos.shape[-1] == pos.shape[-1] and n_spa == aux["spa_positions"].numel()
    assert np.array_equal(aux["spa_positions"].numpy(), g[name + "_spa_pos"])


def test_flash_memory_full_size_properties(qwen):
    """BASELINE-size query-time consolidation: 120 frames, 24x24 full-resolution tokens (12x12 half-resolution), xdim 1280:
    60 CSM centroids + 30 DAM frames -> 11520 memory tokens."""
    pkg, _ = qwen
    g = torch.Generator().manual_seed(7)
    t, h, w, xdim = 120, 24, 24, 1280
    hs, ws = h // 2, w // 2
    scenes = torch.randn(45, hs * ws, xdim, generator=g)
    which = torch.sort(torch.randint(0, 45, (t,), generator=g)).values
    small = (scenes[which] + 0.3 * torch.randn(t, hs * ws, xdim, generator=g)).bfloat16()
    x = (small.float().repeat_interleave(4, dim=1) + 0.1 * torch.randn(t, h * w, xdim, generator=g)).bfloat16()
    fm = pkg.FlashMemory()
    n_vis = (60 * hs * ws + 30 * h * w) // 4
    Ltot = 10 + n_vis + 5
    pos = torch.arange(Ltot).view(1, 1, Ltot).expand(3, 1, Ltot).clone().cuda()
    vis = torch.full((1, Ltot), -1, dtype=torch.long)
    vis[0, 10:10 + n_vis] = torch.arange(n_vis)
    torch.manual_seed(5)
    xin = torch.cat([x.reshape(-1, xdim), small.reshape(-1, xdim)]).cuda()
    new_x, new_pos = fm(xin, torch.tensor([[t, h, w]]).cuda(), torch.tensor([[t, hs, ws]]).cuda(), pos, vis.cuda())
    assert new_x.shape == (1, 4 * n_vis, xdim) and new_pos.shape == (3, 1, Ltot)
    # DAM rows are verbatim bank frames; recover their indices from the temporal position ids and check the gather
    spa_t = new_pos[0, 0, 10:10 + 30 * h * w // 4].view(30, -1)
    assert (spa_t == spa_t[:, :1]).all()
    spa_idx = (spa_t[:, 0] - 10).cpu()
    assert ((spa_idx >= 0) & (spa_idx < t)).all()
    assert torch.equal(new_x[0, : 30 * h * w].view(30, h * w, xdim).cpu(), x[spa_idx])
    # text positions untouched, visual h / w ids inside the grid
    assert torch.equal(new_pos[:, 0, :10].cpu(), torch.arange(10).expand(3, 10))
    assert torch.equal(new_pos[:, 0, 10 + n_vis:].cpu(), torch.arange(10 + n_vis, Ltot).expand(3, 5))
    assert int(new_pos[1, 0, 10:10 + 30 * h * w // 4].max()) == 10 + hs - 1
    # each retrieved frame is (one of) the nearest bank frames of its centroid in fp32 arithmetic
    tem = new_x[0, 30 * h * w:].view(60, hs * ws * xdim).float()
    bank = small.reshape(t, -1).float().cuda()
    d = torch.cdist(tem, bank)                                        # [60, t]
    best = d.min(dim=1).values
    hit = (d[:, spa_idx.cuda()] <= best[:, None] * 1.02 + 1e-3).any(dim=0)   # every DAM frame is nearest to some centroid
    assert hit.all()


def test_flash_memory_full_size_matches_reference(qwen):
    """BASELINE dimensions (64 temporal patches of 576 + 144 tokens x 1280 -> 60 CSM centroids + 30 DAM frames) against
    the reference's own FlashMemory.forward run (tests/golden/make_golden_qwen_full.py): every index the reference
    produced — cluster member lists, timestamps, retrieved DAM positions, AM-RoPE ids — must match exactly."""
    pkg, _ = qwen
    g = _load("qwen_full.npz")
    c = QI.FULL_CASE
    x, small, thw, small_thw, pos, vis = QI.full_input(c)
    assert (QI.checksum(small) == g["chk"]).all(), "seeded input drifted"
    fm = pkg.FlashMemory()
    draws = [dict(init_idx=g["init"], refill_idx=g["refill"], ts_order=g["sort0"], weight_order=g["sort1"])]
    new_x, new_pos = fm(torch.cat([x, small]).cuda(), thw.cuda(), small_thw.cuda(), pos.clone().cuda(), vis.cuda(), draws=draws)
    assert np.array_equal(new_pos.cpu().numpy(), g["new_pos"])                     # includes the 30 DAM positions
    n_spa = 30 * 576
    spa_pos = (new_pos[0, 0, c["prefix"]: c["prefix"] + n_spa // 4].view(30, -1)[:, 0] - c["prefix"]).cpu().numpy()
    assert np.array_equal(spa_pos, g["spa_pos"])
    assert torch.equal(new_x[0, :n_spa].view(30, 576, 1280).cpu(), x.view(64, 576, 1280)[torch.from_numpy(spa_pos)])
    # the CSM side through the same entry point the reference's temporal_compress uses
    feat, weights, ts, idx = pkg.weighted_kmeans_ordered_feature(small.view(64, 144, 1280).cuda(), 60, init_idx=g["init"],
                                                                 refill_idx=g["refill"], order=g["sort0"])
    cnt, flat = g["members"], g["members_flat"]
    want_idx, p = [], 0
    for n in cnt:
        want_idx.append(flat[p:p + n].tolist())
        p += n
    assert idx == want_idx
    assert np.array_equal(ts.cpu().numpy(), g["tem_ts"])
    np.testing.assert_allclose(weights.cpu().numpy(), g["tem_w"], rtol=1e-6)
    tem = feat.reshape(60, -1).float().cpu()
    assert torch.equal(new_x[0, n_spa:].reshape(60, -1).float().cpu(), tem)
    np.testing.assert_allclose(tem.sum(dim=1).numpy(), g["tem_rowsum"], rtol=0, atol=2.0)   # 184320 bf16 values of O(1) per row
    samp = tem[:, :: tem.shape[1] // 256][:, :256].numpy()
    assert (samp != g["tem_sample"]).mean() < 0.01 and np.abs(samp - g["tem_sample"]).max() <= 0.04   # one bf16 step on a few


def test_fast_kmeans_ordered_is_served_by_the_same_kernels(qwen):
    """'fast_kmeans_ordered' (compress_functions.py:301): identical arithmetic in the reference
    (tests/test_qwen_oracle_golden.py::test_reference_fast_variant_is_the_same_arithmetic), identical results here"""
    pkg, _ = qwen
    from flash_vstream_b200.qwen import compress_functions as CF
    name = "ko_scene_bf16"
    c = QI.KMEANS_CASES[name]
    g = _load("qwen_kmeans.npz")
    x, w = QI.kmeans_input(c)
    kw = dict(init_idx=g[name + "_init"], refill_idx=g[name + "_refill"], order=g[name + "_order"])
    a = pkg.weighted_kmeans_ordered_feature(x.cuda(), c["K"], None if w is None else w.cuda(), **kw)
    b = CF.fast_weighted_kmeans_ordered_feature(x.cuda(), c["K"], None if w is None else w.cuda(), **kw)
    assert torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and torch.equal(a[2], b[2]) and a[3] == b[3]
    assert b[3] == _members(g, name)
