"""GPU: the Qwen2-VL vision tower at the non-square grids real videos produce (REAL_GRIDS: 4:3, portrait, 16:9, extreme
aspect, and the 4784-token grid of the processor's default max_pixels), against the fp64 oracle evaluated on the GPU;
a non-square grid must be no worse per row than the square control.  Also: many grids in one call, graph replay of
non-square signatures, and the product path from uint8 480x640 frames to the Flash Memory state."""
import random

import pytest
import torch

from oracle import qwen_oracle as QO
from tests import qwen_vit_inputs as VI
from tests.test_qwen_vit_gpu_parity import TOL, hf_vision_blocks, rel
from tests.test_qwen_vit_grids_host import TEETH_CASES, clip_rows, vit_forward

pytestmark = pytest.mark.gpu

CONTROL = (2, 24, 24)
GRIDS = {"land_864": (2, 24, 36), "port_864": (2, 36, 24), "wide_960": (2, 24, 40), "wide_864": (2, 12, 72),
         "default_4784": (2, 52, 92)}


@pytest.fixture(scope="module")
def qv():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    from flash_vstream_b200 import _lib
    _lib.load(build_if_missing=False)
    from flash_vstream_b200.qwen import vision_tower, vstream_qwen2vl_realtime
    return vision_tower, vstream_qwen2vl_realtime


def row_rel(y, want):
    """relative error of every row"""
    y, want = y.double(), want.double()
    return (y - want).norm(dim=1) / want.norm(dim=1)


class Towers:
    """one depth-2 full-width tower per dtype, and the per-row error of the square control measured in this run"""

    def __init__(self, vt, rt):
        self.vt, self.rt, self.cache, self.control = vt, rt, {}, {}

    def get(self, wdt):
        if wdt not in self.cache:
            c = dict(depth=2, embed=1280, heads=16, seed=94)
            sd = VI.state_dict(c, wdt)
            tower = self.vt.QwenVisionBlocksB200(sd, depth=2, heads=16, dtype=VI.DT[wdt])
            self.cache[wdt] = (c, sd, tower)
        return self.cache[wdt]

    def run(self, wdt, grid):
        """the tower through VisualB200.forward_simple_not_merge, the fp64 oracle on the same rows, and the two
        mutated-position oracles"""
        c, sd, tower = self.get(wdt)
        t, h, w = grid
        cc = dict(c, t=t, h=h, w=w, seed=c["seed"] + h * 100 + w)
        px = VI.pixels(cc, wdt)
        visual = self.rt.VisualB200(self.rt.FlashMemory(), None, encode_patches=tower, dtype=VI.DT[wdt])
        y, _, g2 = visual.forward_simple_not_merge(px.cuda(), torch.tensor([[t, h, w]]).cuda())
        rows, grids = clip_rows(cc, wdt)
        assert g2.tolist() == [list(grids[1])] and y.shape == (rows.shape[0], 1280)
        want = vit_forward(rows, grids, sd, depth=2, heads=16, device="cuda")
        return y, want, grids, (rows, sd)

    def control_worst(self, wdt):
        if wdt not in self.control:
            y, want, _, _ = self.run(wdt, CONTROL)
            self.control[wdt] = float(row_rel(y, want).max())
        return self.control[wdt]


@pytest.fixture(scope="module")
def towers(qv):
    tw = Towers(*qv)
    yield tw
    for _, _, tower in tw.cache.values():
        tower.close()


@pytest.mark.parametrize("wdt", ["f16", "bf16"])
@pytest.mark.parametrize("name", list(GRIDS))
def test_tower_at_real_grids(towers, name, wdt):
    y, want, grids, (rows, sd) = towers.run(wdt, GRIDS[name])
    # every (temporal patch, resolution) segment within the square-grid tolerance
    r0, worst_seg = 0, 0.0
    for t, h, w in grids:
        for _ in range(t):
            e = rel(y[r0:r0 + h * w], want[r0:r0 + h * w])
            worst_seg = max(worst_seg, e)
            assert e < TOL[wdt], ((t, h, w), r0, e)
            r0 += h * w
    worst, control = float(row_rel(y, want).max()), towers.control_worst(wdt)
    print(f"\n[{name} {wdt}] worst segment {worst_seg:.3e}; worst row {worst:.3e}, square control {control:.3e}, "
          f"ratio {worst / control:.3f}")
    assert worst <= 1.5 * control
    # the grid separates the true positions from a swapped or transposed layout by far more than the tolerance
    for m in ("swap", "transpose"):
        d = rel(vit_forward(rows, grids, sd, depth=2, heads=16, device="cuda", mutation=m), want)
        assert d > 10 * TOL[wdt], (m, d)


def test_depth32_two_sided_on_a_non_square_grid(qv):
    """test_vit_depth32_two_sided_vs_library_bf16_run at (1, 24, 36) + (1, 12, 18): ours is no farther from the fp32
    truth than transformers' own bf16 run of the same weights"""
    vt, _ = qv
    c = dict(depth=32, embed=1280, heads=16, t=1, h=24, w=36, seed=93)
    sd = VI.state_dict(c, "bf16")
    rows, grids = clip_rows(c, "bf16")
    assert grids == [(1, 24, 36), (1, 12, 18)]
    tower = vt.QwenVisionBlocksB200(sd, depth=32, heads=16, dtype=torch.bfloat16)
    ours = tower(rows.cuda(), grids).float().cpu()
    tower.close()
    lib16 = hf_vision_blocks(sd, c, rows, grids, torch.bfloat16, "cuda").float().cpu()
    tf32 = torch.backends.cuda.matmul.allow_tf32
    torch.backends.cuda.matmul.allow_tf32 = False
    try:
        truth = hf_vision_blocks(sd, c, rows, grids, torch.float32, "cuda").float().cpu()
    finally:
        torch.backends.cuda.matmul.allow_tf32 = tf32
    r_ours, r_lib = rel(ours, truth), rel(lib16, truth)
    print(f"\n[qwen vit depth 32, bf16, 24x36] ours vs fp32: {r_ours:.3e}; transformers bf16 vs fp32: {r_lib:.3e}")
    assert torch.isfinite(ours).all()
    assert r_ours <= r_lib


def test_sixteen_grids_in_one_call_equal_sixteen_calls(qv):
    """qwen_pos_kernel's grid search and the row0 offsets: one call over 16 distinct non-square grids is bit-identical to
    16 calls; a 17th grid is refused before anything is launched"""
    vt, _ = qv
    grids = TEETH_CASES["many"]
    assert len(set(grids)) == 16 and all(h != w for _, h, w in grids)
    sd = VI.state_dict(dict(depth=1, embed=1280, heads=16, seed=95), "bf16")
    tower = vt.QwenVisionBlocksB200(sd, depth=1, heads=16, dtype=torch.bfloat16)
    n = [t * h * w for t, h, w in grids]
    x = (torch.randn(sum(n), 1176, generator=torch.Generator().manual_seed(6)) * 1.2).bfloat16().cuda()
    both = tower(x, grids)
    parts = torch.cat([tower(xi, [g]) for xi, g in zip(x.split(n), grids)])
    assert torch.equal(both, parts)
    want = vit_forward(x, grids, sd, depth=1, heads=16, device="cuda")
    assert rel(both, want) < TOL["bf16"]
    lib = tower.lib
    extra = torch.cat([x, x[:8]])
    torch.cuda.synchronize()
    n0 = lib.fvs_launch_count()
    with pytest.raises(ValueError, match="16 grids"):
        tower(extra, grids + [(1, 2, 4)])
    torch.cuda.synchronize()
    assert lib.fvs_launch_count() == n0
    tower.close()


def test_graph_replay_of_non_square_signatures(qv):
    """landscape and portrait signatures with the same row count are different graphs; every replay equals the eager
    launches bit for bit"""
    vt, _ = qv
    sd = VI.state_dict(dict(depth=2, embed=1280, heads=16, seed=96), "bf16")
    eager = vt.QwenVisionBlocksB200(sd, depth=2, heads=16, dtype=torch.bfloat16)
    graph = vt.QwenVisionBlocksB200(sd, depth=2, heads=16, dtype=torch.bfloat16, use_graphs=True, graph_max_rows=4000)
    sigs = [[(1, 24, 36), (1, 12, 18)], [(1, 36, 24), (1, 18, 12)], [(2, 12, 72), (2, 6, 36)]]
    g = torch.Generator().manual_seed(7)
    for rep in range(2):
        for grids in sigs:
            rows = sum(t * h * w for t, h, w in grids)
            x = (torch.randn(rows, 1176, generator=g) * 1.2).bfloat16().cuda()
            assert torch.equal(graph(x, grids), eager(x, grids)), (rep, grids)
    assert len(graph._graphs) == 3
    eager.close()
    graph.close()


def test_480p_frames_through_preprocessor_tower_and_flash_memory(qv):
    """uint8 480x640 frames -> the GPU pre-processor at the reference CLI's settings -> a depth-1 tower -> the Flash Memory
    streaming step, three clips; the consolidation is bit-exact against the oracle fed with the tower's own features"""
    from flash_vstream_b200.preprocess import Qwen2VLFramePreprocessor
    from tests import preprocess_inputs as PI
    from tests import qwen_rt_inputs as RI
    from tests.test_qwen_rt_gpu_parity import cuda_w
    from tests.test_qwen_rt_oracle_golden import REL
    vt, rt = qv
    proc = Qwen2VLFramePreprocessor(max_pixels=4 * 224 * 224, additional_pool_size=2)
    sd = VI.state_dict(dict(depth=1, embed=1280, heads=16, seed=97), "bf16")
    tower = vt.QwenVisionBlocksB200(sd, depth=1, heads=16, dtype=torch.bfloat16)
    w = RI.merger_weights(1280, 256, "bf16", 98)
    flash = rt.FlashMemory(flash_memory_temporal_length=6, flash_memory_spatial_length=4)
    host = rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(flash, rt.PatchMerger.from_weights(cuda_w(w)), encode_patches=tower))
    orc = QO.RealtimeOracle(QO.FlashMemoryOracle(6, 4), w)
    seen = {}
    real_call = tower.__call__

    def spy(rows, grids):
        seen["grids"] = grids.tolist() if torch.is_tensor(grids) else [list(g) for g in grids]
        seen["y"] = real_call(rows, grids)
        return seen["y"]
    host.visual.encode_patches = spy
    torch.manual_seed(11)
    random.seed(11)
    n_full = 2 * 24 * 36
    for s in range(3):
        inputs = proc(torch.from_numpy(PI.frames(40 + s, (4, 480, 640))).cuda())
        assert inputs["video_grid_thw"].tolist() == [[2, 24, 36]]
        perm_state = torch.cuda.get_rng_state()
        host.embed_new_video_clip(**inputs, start_idx=2 * s)
        assert seen["grids"] == [[2, 24, 36], [2, 12, 18]]
        (tem_x, tem_thw, tem_w, tem_ts, spa_x, spa_thw, spa_pos, bank, thw, small_bank, small_thw, embeds,
         shape) = host.video_embedding_memory
        assert thw.tolist() == [2 * (s + 1), 24, 36] and small_thw.tolist() == [2 * (s + 1), 12, 18]
        assert tem_thw.tolist() == [min(2 * (s + 1), 3), 12, 18] and embeds.shape[1] == 256
        y = seen["y"].cpu()
        assert y.shape[0] == n_full + 2 * 12 * 18
        T = min(3 + 2, 2 * (s + 1)) if s else 2                       # replay the same RNG draws for the oracle
        init = None
        if T > 3:
            torch.cuda.set_rng_state(perm_state)
            init = torch.randperm(T, device="cuda")[:3].cpu().numpy()
        om = orc.embed_new_video_clip(y[:n_full], [2, 24, 36], y[n_full:], [2, 12, 18], s * 2, init_idx=init,
                                      refill_idx=[0] * 30)
        assert torch.equal(tem_x.cpu().view(torch.int16), om[0].view(torch.int16))
        assert torch.equal(spa_x.reshape(-1, 1280).cpu().view(torch.int16), om[4].reshape(-1, 1280).view(torch.int16))
        assert torch.equal(bank.cpu().view(torch.int16), om[7].view(torch.int16))
        assert torch.equal(spa_pos.cpu(), om[6]) and torch.equal(tem_w.float().cpu(), om[2].float())
        assert rel(embeds.cpu(), om[11]) < REL["bf16"]
    tower.close()
