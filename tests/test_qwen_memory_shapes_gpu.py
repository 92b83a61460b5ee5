"""The Qwen2-VL Flash Memory kernels bit for bit against oracle/qwen_oracle.py at the shapes a real stream runs
(pytest -m gpu).  The cases and the branch each one reaches live in test_qwen_memory_shapes_host.py; every comparison
here is an exact one on the bits (NaN pattern included)."""
import random

import numpy as np
import pytest
import torch

from oracle import qwen_oracle as QO
from tests import qwen_rt_inputs as RI
from tests.test_qwen_memory_shapes_host import (KLARGE_CASES, KMEANS_CASES, PD_REAL, kmeans_input, kmeans_oracle,
                                                klarge_input, klarge_oracle)
from tests.test_qwen_rt_oracle_golden import REL, rel
from tests.test_qwen_vit_grids_host import REAL_GRIDS

pytestmark = pytest.mark.gpu


@pytest.fixture(scope="module")
def qwen():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    from flash_vstream_b200 import _lib
    _lib.load(build_if_missing=False)
    import flash_vstream_b200.qwen as pkg
    from flash_vstream_b200.qwen import ops as qops
    return pkg, qops


def same_bits(a, b):
    """bit-identical, NaN pattern included (a NaN's sign and payload differ between the GPU and the host's numpy)"""
    a = torch.as_tensor(a).detach().cpu().contiguous()
    b = torch.as_tensor(b).detach().cpu().contiguous()
    assert a.dtype == b.dtype and a.shape == b.shape, (a.dtype, b.dtype, a.shape, b.shape)
    if a.is_floating_point():
        assert torch.equal(torch.isnan(a), torch.isnan(b)), "NaN patterns differ"
        a, b = torch.nan_to_num(a, nan=0.0, posinf=torch.inf, neginf=-torch.inf), \
            torch.nan_to_num(b, nan=0.0, posinf=torch.inf, neginf=-torch.inf)
    eq = a.view(torch.uint8).reshape(a.numel(), -1) == b.view(torch.uint8).reshape(b.numel(), -1)
    bad = (~eq.all(dim=1)).sum().item()
    assert bad == 0, f"{bad} of {a.numel()} elements differ"


# ------------------------------------------------------------------------------------------------ a. ordered k-means
@pytest.mark.parametrize("name", list(KMEANS_CASES))
def test_kmeans_ordered_bit_exact(qwen, name):
    _, qops = qwen
    c = KMEANS_CASES[name]
    x, w, init, refill = kmeans_input(c)
    C, wsum, labels, info = qops.kmeans_ordered(x.cuda(), w.cuda(), None, init.cuda(), refill.cuda(), c["K"], c["max_iter"],
                                                c["tol"])
    o_C, o_labels, o_wsum, o_info, _ = kmeans_oracle(c)
    same_bits(labels, torch.from_numpy(o_labels))
    same_bits(C, torch.from_numpy(o_C))
    assert info[:3].cpu().tolist() == o_info
    if o_wsum is not None:                                             # max_iter == 0 computes no weight sums
        same_bits(wsum, torch.from_numpy(o_wsum))


# ------------------------------------------------------------------------------------------------ b. end to end
def test_weighted_kmeans_ordered_feature_baseline_bit_exact(qwen):
    """the BASELINE CSM update through the mirror of weighted_kmeans_ordered_feature (unique rows, k-means, bookkeeping,
    cast), with recorded draws: centroids, weights, timestamps and members bit for bit"""
    pkg, _ = qwen
    c = KMEANS_CASES["k60_s180_bf16_baseline"]
    x, _, _, _ = kmeans_input(c)
    x = x.view(c["T"], 144, 1280)
    g = torch.Generator().manual_seed(c["seed"] + 1)
    init = torch.randperm(c["T"], generator=g)[: c["K"]].numpy()                   # indices into the sorted unique rows
    refill = torch.randint(0, c["T"], (10 * c["K"],), generator=g).numpy()
    feat, wts, ts, idx = pkg.weighted_kmeans_ordered_feature(x.cuda(), c["K"], init_idx=init, refill_idx=refill)
    o_feat, o_w, o_ts, o_idx = QO.weighted_kmeans_ordered_feature(x, c["K"], init_idx=init, refill_idx=refill)
    assert list(idx) == o_idx
    same_bits(feat, o_feat)
    same_bits(wts.float(), o_w)
    same_bits(ts.float(), o_ts)


# ------------------------------------------------------------------------------------------------ c. klarge retrieval
@pytest.mark.parametrize("name", list(KLARGE_CASES))
def test_klarge_retrieve_bit_exact(qwen, name):
    _, qops = qwen
    c = KLARGE_CASES[name]
    tem, kidx, bank = klarge_input(c)
    idx, dist = qops.klarge_retrieve(tem.cuda(), kidx.cuda(), bank.cuda(), want_dist=True, metric=c["metric"])
    want, want_idx = klarge_oracle(c)
    same_bits(dist, torch.from_numpy(want))
    assert np.array_equal(idx.cpu().numpy(), want_idx)


# ------------------------------------------------------------------------------------------------ d. unique rows
def unique_input(T, dt, seed):
    """T rows of PD_REAL drawn from duplicate classes whose prototypes differ from a base row only in element 0, 1023,
    1024 or the last one (either direction), in 1023 and 1024 with opposite signs, or by +0.0 against -0.0"""
    g = torch.Generator().manual_seed(seed)
    base = torch.randn(PD_REAL, generator=g)
    base[5] = 0.0
    protos = [base]
    for e in (0, 1023, 1024, PD_REAL - 1):
        for s in (1.0, -1.0):
            p = base.clone()
            p[e] += s * 0.5
            protos.append(p)
    for s in (1.0, -1.0):
        p = base.clone()
        p[1023] += s * 0.5
        p[1024] -= s * 0.5
        protos.append(p)
    neg0 = base.clone()
    neg0[5] = -0.0                                                     # equal to base under torch.unique
    protos.append(neg0)
    protos += [torch.randn(PD_REAL, generator=g) for _ in range(6)]
    P = torch.stack(protos).to(dt)
    rows = torch.cat([torch.arange(len(protos)), torch.randint(0, len(protos), (T - len(protos),), generator=g)])
    rows = rows[torch.randperm(T, generator=g)]
    return P[rows]


def torch_unique_order(X):
    """torch.unique(X, dim=0) as the first row index of each class, in the sorted order of the classes"""
    _, inv = torch.unique(X.float(), dim=0, return_inverse=True)
    first = torch.full((int(inv.max()) + 1,), X.shape[0], dtype=torch.long)
    first.scatter_reduce_(0, inv, torch.arange(X.shape[0]), reduce="amin")
    return first.numpy()


@pytest.mark.parametrize("dt", ["bf16", "f16", "f32"])
def test_unique_rows_at_real_width(qwen, dt):
    _, qops = qwen
    tdt = {"bf16": torch.bfloat16, "f16": torch.float16, "f32": torch.float32}[dt]
    X = unique_input(61, tdt, 901)
    idx, n = qops.unique_rows(X.cuda())
    n = int(n.item())
    want = QO.unique_rows_order(X.float().numpy())
    assert n == len(want) == 17                                          # -0.0 joins +0.0's class
    assert np.array_equal(idx[:n].cpu().numpy(), want)
    assert np.array_equal(want, torch_unique_order(X))
    X = unique_input(300, tdt, 902)
    idx, n = qops.unique_rows(X.cuda())
    n = int(n.item())
    assert np.array_equal(idx[:n].cpu().numpy(), torch_unique_order(X))


def test_unique_rows_at_the_row_limit(qwen):
    _, qops = qwen
    from flash_vstream_b200 import _lib
    g = torch.Generator().manual_seed(903)
    X = torch.randn(1500, 1024, generator=g).bfloat16()
    X = X[torch.randint(0, 1500, (4096,), generator=g)]
    X[7, 1023] = -X[7, 1023]                                             # one more class, by the chunk's last element
    idx, n = qops.unique_rows(X.cuda())
    n = int(n.item())
    assert np.array_equal(idx[:n].cpu().numpy(), torch_unique_order(X))
    lib = _lib.load()
    torch.cuda.synchronize()
    n0 = lib.fvs_launch_count()
    with pytest.raises(Exception, match="bad shape"):
        qops.unique_rows(torch.zeros(4097, 1024, dtype=torch.bfloat16, device="cuda"))
    assert lib.fvs_launch_count() == n0


# ------------------------------------------------------------------------------------------------ e. streaming
class _Counted(list):
    """the refill draws handed to the oracle; records how many it consumed"""
    used = 0

    def __getitem__(self, i):
        self.used = max(self.used, int(i) + 1)
        return super().__getitem__(i)


def test_streaming_at_the_default_memory_lengths(qwen):
    """temporal_length 120 / spatial_length 60 (CSM 60 frames, DAM 30), 4-patch clips of 8x8 / 4x4 x 1280: fill the CSM,
    then six steady-state clips, each one a 64 -> 60 k-means with carried weights.  The product draws from the global
    generators; the oracle replays the same draws, and both generators must end where the reference leaves them."""
    import flash_vstream_b200.qwen.vstream_qwen2vl_realtime as rt
    from flash_vstream_b200.draws import GLOBAL
    t, h, w, xdim, n_steps = 4, 8, 8, 1280, 21
    g = torch.Generator().manual_seed(911)
    scenes = torch.randn(12, 16, xdim, generator=g)
    clips = []
    for s in range(n_steps):
        which = torch.randint(0, 12, (t,), generator=g)
        small = scenes[which] + 0.3 * torch.randn(t, 16, xdim, generator=g)
        x = small.repeat_interleave(4, dim=1) + 0.1 * torch.randn(t, 64, xdim, generator=g)
        clips.append((x.reshape(-1, xdim).bfloat16(), small.reshape(-1, xdim).bfloat16()))
    mw = RI.merger_weights(xdim, 256, "bf16", 912)
    step = {"i": 0}

    def encode(patch_rows, total_grid_thw):
        x, small = clips[step["i"]]
        return torch.cat([x, small]).cuda()
    flash = rt.FlashMemory(flash_memory_temporal_length=120, flash_memory_spatial_length=60)
    host = rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(flash, rt.PatchMerger.from_weights({k: v.cuda() for k, v in mw.items()}),
                                                            encode_patches=encode, dtype=torch.bfloat16))
    orc = QO.RealtimeOracle(QO.FlashMemoryOracle(120, 60), mw)
    torch.manual_seed(913)
    random.seed(913)
    steady = 0
    for s in range(n_steps):
        step["i"] = s
        GLOBAL.settle()
        py0, cu0 = random.getstate(), torch.cuda.get_rng_state()
        host.embed_new_video_clip(torch.zeros(t * h * w, 1176), torch.tensor([[t, h, w]]), s * t)
        GLOBAL.settle()
        py1, cu1 = random.getstate(), torch.cuda.get_rng_state()
        T = min(60, s * t) + t
        init, refill = None, _Counted([0])
        if T > 60:                                                      # the k-means runs: replay its draws
            steady += 1
            torch.cuda.set_rng_state(cu0)
            init = torch.randperm(T, device="cuda")[:60].cpu().numpy()
            assert torch.equal(torch.cuda.get_rng_state(), cu1)
            r = random.Random()
            r.setstate(py0)
            refill = _Counted(r.randint(0, T - 1) for _ in range(10 * 60))
        else:
            assert torch.equal(cu0, cu1)
        x, small = clips[s]
        om = orc.embed_new_video_clip(x, [t, h, w], small, [t, h // 2, w // 2], s * t, init_idx=init, refill_idx=refill)
        r = random.Random()
        r.setstate(py0)
        for _ in range(refill.used if T > 60 else 0):
            r.randint(0, T - 1)
        assert r.getstate() == py1, f"step {s}: random left at the wrong position"
        tem_x, tem_thw, tem_w, tem_ts, spa_x, spa_thw, spa_pos, bank, thw, small_bank, small_thw, embeds, _ = \
            host.video_embedding_memory
        same_bits(tem_x, om[0])
        same_bits(spa_x.reshape(-1, xdim), om[4].reshape(-1, xdim))
        same_bits(tem_w.float(), om[2].float())
        assert torch.equal(spa_pos.cpu(), om[6])
        same_bits(bank, om[7])
        same_bits(small_bank, om[9])
        assert rel(embeds.cpu(), om[11]) < REL["bf16"]
    assert steady == 6 and tem_thw.tolist() == [60, 4, 4] and spa_thw.tolist() == [30, 8, 8]


# ------------------------------------------------------------------------------------------------ f. real grids
GRIDS = sorted({g for *_, g, _ in REAL_GRIDS} | {(t, w, h) for *_, (t, h, w), _ in REAL_GRIDS})


@pytest.mark.parametrize("grid", GRIDS, ids=[f"{t}x{h}x{w}" for t, h, w in GRIDS])
def test_temporal_pool_and_am_rope_at_real_grids(qwen, grid):
    pkg, _ = qwen
    t, h, w = grid
    fm = pkg.FlashMemory()
    for dt, seed in ((torch.bfloat16, 921), (torch.float16, 922)):
        x = (torch.randn(t * h * w, 1176, generator=torch.Generator().manual_seed(seed)) * 1.5).to(dt)
        y, thw = fm.temporal_pool(x.cuda(), torch.tensor([t, h, w]))
        want, want_thw = QO.temporal_pool(x, [t, h, w])
        assert thw.tolist() == want_thw
        same_bits(y, want)
    # AM-RoPE of a full memory on this grid: 30 DAM frames at full resolution, 60 CSM centroids at half resolution
    g = torch.Generator().manual_seed(923)
    spa_thw, tem_thw = torch.tensor([30, h, w]), torch.tensor([60, h // 2, w // 2])
    spa_pos = torch.sort(torch.randperm(500, generator=g)[:30]).values
    tem_pos = torch.sort(torch.randint(0, 500, (60,), generator=g)).values
    n = 30 * h * w // 4 + 60 * (h // 2) * (w // 2) // 4
    L = 7 + n + 3
    pos = (torch.arange(L) + 11).view(1, L).expand(3, L).clone()
    vis = torch.full((L,), -1, dtype=torch.long)
    vis[7:7 + n] = torch.arange(n)
    want = QO.FlashMemoryOracle.calc_am_rope(pos, vis, tem_thw, tem_pos, spa_thw, spa_pos)
    got = fm.calc_am_rope(pos.clone().cuda(), vis.cuda(), tem_thw.cuda(), tem_pos.cuda(), spa_thw.cuda(), spa_pos.cuda())
    assert torch.equal(got.cpu(), want)
