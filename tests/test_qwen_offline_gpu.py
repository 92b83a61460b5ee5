"""GPU: the offline Qwen2-VL vision pass, VisualB200.forward (qwen/offline.py), which runs the full-resolution tower only
on the frames the memory keeps and the tower in chunks of whole temporal patches.

1. bit for bit the unpruned composition of tested parts: the tower over every row of both resolutions at once
   (forward_simple_not_merge), FlashMemory.forward and the PatchMerger, drawing from the same global generators, which
   must end in the same state;
2. the reference's own visual.forward (tests/golden/qwen_offline.npz): picks, timestamps and position ids exact, the
   embeddings within the tower tolerance of tests/test_qwen_vit_gpu_parity.py;
3. the full-resolution rows the tower actually encodes, min(t, S) h w a video;
4. the peak memory of a long video, bounded by the half-resolution bank, the DAM rows and one chunk;
5. refusals: nothing launched, no generator moved."""
import os
import random
import types

import numpy as np
import pytest
import torch

from tests import qwen_offline_inputs as OI
from tests.qwen_inputs import DT
from tests.test_qwen_vit_grids_host import REAL_GRIDS

pytestmark = pytest.mark.gpu
G = os.path.join(os.path.dirname(os.path.abspath(__file__)), "golden", "qwen_offline.npz")
TOL = {"f16": 1.5e-3, "bf16": 1.0e-2}          # tests/test_qwen_vit_gpu_parity.py: relative Frobenius error vs fp32


@pytest.fixture(scope="module")
def env():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    from flash_vstream_b200 import _lib
    _lib.load(build_if_missing=False)
    from flash_vstream_b200.qwen import offline, vision_tower, vstream_qwen2vl_model, vstream_qwen2vl_realtime
    towers, mergers = {}, {}
    for wdt in ("bf16", "f16"):
        towers[wdt] = vision_tower.QwenVisionBlocksB200(OI.tower_state_dict(wdt), depth=OI.TOWER["depth"],
                                                        heads=OI.TOWER["heads"], dtype=DT[wdt])
        w = OI.merger_weights(wdt)
        mergers[wdt] = vstream_qwen2vl_realtime.PatchMerger.from_weights(
            {"ln_w": w["ln_q.weight"], "ln_b": w["ln_q.bias"], "fc1_w": w["mlp.0.weight"], "fc1_b": w["mlp.0.bias"],
             "fc2_w": w["mlp.2.weight"], "fc2_b": w["mlp.2.bias"]})
    yield types.SimpleNamespace(lib=_lib.load(), of=offline, vt=vision_tower, M=vstream_qwen2vl_model,
                                rt=vstream_qwen2vl_realtime, towers=towers, mergers=mergers)
    for t in towers.values():
        t.close()


def _generators():
    from flash_vstream_b200.draws import GLOBAL
    GLOBAL.settle()
    return torch.get_rng_state(), torch.cuda.get_rng_state(), random.getstate()


def _same_generators(a, b):
    return torch.equal(a[0], b[0]) and torch.equal(a[1], b[1]) and a[2] == b[2]


def _inputs(fm, grids, seed, wdt):
    pool = fm.temporal_poolsize
    n_vis = [OI.n_visual(g, fm.temporal_length, fm.spatial_length, pool) for g in grids]
    pos, vis = OI.positions(n_vis)
    px = OI.pixels([(g, None) for g in grids], seed, wdt).cuda()
    return px, torch.tensor(grids).cuda(), pos.cuda(), vis.cuda()


def pruned_and_unpruned(env, fm_kw, grids, wdt="bf16", max_rows=None, seed=5):
    """(embeds, position ids, generator states) of the pruned, chunked forward and of the unpruned composition"""
    fm = env.M.FlashMemory(**fm_kw)
    kw = {} if max_rows is None else dict(offline_max_rows=max_rows)
    visual = env.rt.VisualB200(fm, env.mergers[wdt], encode_patches=env.towers[wdt], dtype=DT[wdt], **kw)
    px, thw, pos, vis = _inputs(fm, grids, seed, wdt)
    torch.manual_seed(seed)
    random.seed(seed)
    emb, new_pos = visual(px, thw, pos.clone(), vis)
    after = _generators()
    torch.manual_seed(seed)
    random.seed(seed)
    feats, _, small_thw = visual.forward_simple_not_merge(px, thw)
    mem, want_pos = fm.forward(feats, thw, small_thw, pos.clone(), vis)
    want = env.mergers[wdt](mem)
    return (emb, new_pos, after), (want, want_pos, _generators())


def assert_identical(got, want):
    (emb, pos, gen), (emb_w, pos_w, gen_w) = got, want
    assert emb.dtype == emb_w.dtype and emb.shape == emb_w.shape
    assert torch.equal(emb.view(torch.int16), emb_w.view(torch.int16)), \
        f"{(emb != emb_w).float().mean().item():.4f} of the embeddings differ"
    assert torch.equal(pos, pos_w)
    assert _same_generators(gen, gen_w), "the generators ended in different states"


S_CFG = dict(flash_memory_temporal_length=12, flash_memory_spatial_length=8)       # T0 = 6 centroids, S = 4 DAM frames
T0, S = 6, 4


# ------------------------------------------------------------------------------------------------ 1. bit-identical
@pytest.mark.parametrize("t", [1, S - 1, S, S + 1, T0 + 1, 2 * T0 + 3])
@pytest.mark.parametrize("wdt", ["bf16", "f16"])
def test_lengths_around_the_memory(env, t, wdt):
    assert_identical(*pruned_and_unpruned(env, S_CFG, [(t, 8, 8)], wdt))


@pytest.mark.parametrize("spatial", ["sample", "nearest", "klarge_retrieve", "klarge_retrieve_cos"])
@pytest.mark.parametrize("temporal", ["kmeans_ordered", "fast_kmeans_ordered", "sample"])
def test_methods(env, spatial, temporal):
    # 'sample' keeps no cluster weights, so (as in the reference) only 'sample' retrieval follows it past the CSM
    t = 2 * T0 + 3 if temporal != "sample" or spatial == "sample" else T0
    cfg = dict(S_CFG, flash_memory_temporal_method=temporal, flash_memory_spatial_method=spatial)
    assert_identical(*pruned_and_unpruned(env, cfg, [(t, 8, 12)]))


@pytest.mark.parametrize("t", [1, S + 1, 2 * T0 + 3])
def test_no_second_resolution(env, t):
    assert_identical(*pruned_and_unpruned(env, dict(S_CFG, flash_memory_temporal_poolsize=1), [(t, 8, 8)],
                                          max_rows=128))


@pytest.mark.parametrize("cfg", [dict(S_CFG, flash_memory_spatial_length=0),
                                 dict(S_CFG, flash_memory_temporal_length=0, flash_memory_spatial_method="sample")],
                         ids=["no_DAM", "no_CSM"])
def test_empty_memories(env, cfg):
    assert_identical(*pruned_and_unpruned(env, cfg, [(2 * T0 + 3, 8, 8)], max_rows=64))


@pytest.mark.parametrize("grids", [[(9, 8, 8), (15, 8, 8)], [(7, 8, 8), (20, 8, 8), (11, 8, 8)]], ids=["two", "three"])
@pytest.mark.parametrize("wdt", ["bf16", "f16"])
def test_mixed_batch(env, grids, wdt):
    assert_identical(*pruned_and_unpruned(env, S_CFG, grids, wdt, max_rows=192))


@pytest.mark.parametrize("grid", sorted({(T0 + 3, h, w) for *_, (_, h, w), _ in REAL_GRIDS}))
def test_real_grids(env, grid):
    assert_identical(*pruned_and_unpruned(env, S_CFG, [grid]))


@pytest.mark.parametrize("max_rows", [64, 16, 100, 128, 300, 10 ** 6])
def test_budgets(env, max_rows):
    """64: one full-resolution patch (four half-resolution ones) a call; 16: one half-resolution patch a call (only
    without a full-resolution pass); 100 and 300: budgets that are no multiple of a patch; 10**6: one call"""
    cfg = dict(S_CFG, flash_memory_spatial_length=0) if max_rows < 64 else S_CFG
    assert_identical(*pruned_and_unpruned(env, cfg, [(2 * T0 + 3, 8, 8)], max_rows=max_rows))


def test_from_reference_module(env):
    """from_reference over a transformers Qwen2-VL vision tower with the reference's flash_memory attribute: the same
    tower, memory and merger as building the parts by hand, so the same bits"""
    from transformers.models.qwen2_vl import modeling_qwen2_vl as HF
    from transformers.models.qwen2_vl.configuration_qwen2_vl import Qwen2VLVisionConfig
    c = OI.TOWER
    cfg = Qwen2VLVisionConfig(depth=c["depth"], embed_dim=c["embed"], hidden_size=OI.MERGER_OUT, num_heads=c["heads"],
                              mlp_ratio=4, in_channels=3, patch_size=14, spatial_merge_size=2, temporal_patch_size=2)
    ref = HF.Qwen2VisionTransformerPretrainedModel(cfg)
    sd = dict(OI.tower_state_dict("bf16"))
    sd.update({"merger." + k: v for k, v in OI.merger_weights("bf16").items()})
    missing, unexpected = ref.load_state_dict({k: v.float() for k, v in sd.items()}, strict=False)
    assert not missing and not unexpected
    ref = ref.to(torch.bfloat16)
    ref.flash_memory = types.SimpleNamespace(config=dict(OI.GOLDEN_FM, **S_CFG))
    visual = env.rt.VisualB200.from_reference(ref, offline_max_rows=256)
    assert visual.flash_memory.config == ref.flash_memory.config and visual.get_dtype() == torch.bfloat16
    grids = [(2 * T0 + 3, 8, 8)]
    px, thw, pos, vis = _inputs(visual.flash_memory, grids, 8, "bf16")
    torch.manual_seed(8)
    random.seed(8)
    emb, new_pos = visual(px, thw, pos.clone(), vis)
    hand = pruned_and_unpruned(env, dict(OI.GOLDEN_FM, **S_CFG), grids, seed=8)
    assert torch.equal(emb, hand[0][0]) and torch.equal(new_pos, hand[0][1])
    visual.encode_patches.close()


# ------------------------------------------------------------------------------------------------ 2. the golden
@pytest.mark.parametrize("name", list(OI.GOLDEN_CASES))
def test_matches_the_reference_forward(env, name):
    g = np.load(G)
    videos = OI.GOLDEN_CASES[name]
    grids = [grid for grid, _ in videos]
    fm = env.M.FlashMemory(**OI.GOLDEN_FM)
    visual = env.rt.VisualB200(fm, env.mergers["bf16"], encode_patches=env.towers["bf16"], dtype=torch.bfloat16)
    px = OI.pixels(videos, int(g[f"{name}_seed"])).cuda()
    pos, vis = OI.positions([OI.n_visual(grid, fm.temporal_length, fm.spatial_length) for grid in grids])
    opt = lambda a: a if len(a) else None
    draws = [dict(init_idx=opt(g[f"{name}_v{b}_init"]), refill_idx=g[f"{name}_v{b}_refill"],
                  ts_order=opt(g[f"{name}_v{b}_ts_order"]), weight_order=opt(g[f"{name}_v{b}_weight_order"]))
             for b in range(len(videos))]
    picks = []
    spatial_picks = fm.spatial_picks
    fm.spatial_picks = lambda *a, **k: picks.append(spatial_picks(*a, **k)) or picks[-1]
    emb, new_pos = visual(px, torch.tensor(grids).cuda(), pos.clone().cuda(), vis.cuda(), draws=draws)
    assert np.array_equal(new_pos.cpu().numpy(), g[f"{name}_pos"])
    for b, p in enumerate(picks):
        assert np.array_equal(p.cpu().numpy(), g[f"{name}_v{b}_picks"])
    # timestamps: the CSM tokens' temporal ids, after the DAM block
    for b, (t, h, w) in enumerate(grids):
        n_dam, n_csm = min(t, fm.spatial_length) * h * w // 4, min(t, fm.temporal_length) * h * w // 16
        csm = new_pos[0, b, OI.PREFIX + n_dam: OI.PREFIX + n_dam + n_csm].cpu().numpy()[:: h * w // 16]
        assert np.array_equal(csm - OI.PREFIX - n_dam, np.round(g[f"{name}_v{b}_ts"]))
    assert list(emb.shape) == g[f"{name}_rows"].tolist()
    ours, want = emb.float().cpu()[OI.GOLDEN_ROWS].double(), torch.from_numpy(g[f"{name}_emb32"]).double()
    err = float((ours - want).norm() / want.norm())
    print(f"\n[{name}] video_embeds rel vs the reference's fp32 run: {err:.3e}")
    assert err < TOL["bf16"]


# ------------------------------------------------------------------------------------------------ 3. work pruned
def test_full_resolution_rows_encoded(env):
    fm = env.M.FlashMemory(**S_CFG)
    rows = {}
    tower = env.towers["bf16"]

    def counting(x, grids):
        for t, h, w in grids:
            rows[(h, w)] = rows.get((h, w), 0) + t * h * w
        return tower(x, grids)
    visual = env.rt.VisualB200(fm, env.mergers["bf16"], encode_patches=counting, offline_max_rows=128)
    for grids in ([(1, 8, 8)], [(S, 8, 8)], [(2 * T0 + 3, 8, 8)], [(40, 16, 8)], [(9, 8, 8), (15, 8, 8)]):
        rows.clear()
        px, thw, pos, vis = _inputs(fm, grids, 3, "bf16")
        visual(px, thw, pos, vis)
        h, w = grids[0][1:]
        assert rows[(h, w)] == sum(min(t, S) * h * w for t, _, _ in grids)
        assert rows[(h // 2, w // 2)] == sum(t * h * w // 4 for t, _, _ in grids)


# ------------------------------------------------------------------------------------------------ 4. bounded memory
def test_long_video_memory_is_bounded(env):
    """320 temporal patches at 32x32 (the CLI's grid), the default memory lengths, a one-block tower, 8,192-row chunks.
    Peak = the half-resolution bank + the DAM rows + one chunk's workspace and activations + the memory's assembly
    (CSM rows, the concatenation, the merger's LayerNorm and fc1 outputs) + the k-means' fp32 view of the bank."""
    t, h, w, E, mlp, budget = 320, 32, 32, 1280, 5120, 8192
    sd = {k: v for k, v in OI.tower_state_dict("bf16").items() if not k.startswith("blocks.1.")}
    tower = env.vt.QwenVisionBlocksB200(sd, depth=1, heads=16, dtype=torch.bfloat16)
    fm = env.M.FlashMemory()
    visual = env.rt.VisualB200(fm, env.mergers["bf16"], encode_patches=tower, offline_max_rows=budget)
    px = (torch.randn(t * h * w, 1176, device="cuda") * 1.2).bfloat16()
    pos, vis = OI.positions([OI.n_visual((t, h, w), fm.temporal_length, fm.spatial_length)])
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    torch.cuda.reset_peak_memory_stats()
    emb, _ = visual(px, torch.tensor([[t, h, w]]).cuda(), pos.cuda(), vis.cuda())
    torch.cuda.synchronize()
    peak = torch.cuda.max_memory_allocated() - base
    b16 = 2
    bank = t * h * w // 4 * E * b16
    dam = fm.spatial_length * h * w * E * b16
    chunk = tower.lib.fvs_qwen_vit_workspace_bytes(tower._h, budget) + budget * (E + 1176) * b16
    mem_rows = fm.spatial_length * h * w + fm.temporal_length * h * w // 4
    assembly = fm.temporal_length * h * w // 4 * E * b16 + 4 * mem_rows * E * b16   # + concat, stack, LayerNorm, fc1
    kmeans = 2 * bank
    bound = bank + dam + chunk + assembly + kmeans
    unchunked = tower.lib.fvs_qwen_vit_workspace_bytes(tower._h, t * (h * w + h * w // 4))
    print(f"\n[long video] peak {peak / 2**20:.0f} MiB, bound {bound / 2**20:.0f} MiB, the unpruned pass's workspace "
          f"alone {unchunked / 2**20:.0f} MiB")
    assert emb.shape == (mem_rows // 4, OI.MERGER_OUT)
    assert peak <= bound
    assert bound < unchunked / 4
    tower.close()


# ------------------------------------------------------------------------------------------------ 5. refusals
@pytest.mark.parametrize("cfg,grids,exc", [
    (S_CFG, [(9, 8, 8), (9, 6, 8)], NotImplementedError),
    (dict(S_CFG, flash_memory_temporal_poolsize=3), [(9, 8, 8)], AssertionError),
    (dict(S_CFG, flash_memory_temporal_method="gmm"), [(9, 8, 8)], NotImplementedError),
    (dict(S_CFG, flash_memory_spatial_method="far"), [(9, 8, 8)], ValueError),
])
def test_refusals_launch_nothing(env, cfg, grids, exc):
    fm = env.M.FlashMemory(**cfg)
    visual = env.rt.VisualB200(fm, env.mergers["bf16"], encode_patches=env.towers["bf16"])
    rows = sum(t * h * w for t, h, w in grids)
    px = torch.zeros(rows, 1176, dtype=torch.bfloat16, device="cuda")
    pos, vis = OI.positions([8] * len(grids))
    pos, vis, thw = pos.cuda(), vis.cuda(), torch.tensor(grids).cuda()
    torch.cuda.synchronize()
    before, n0 = _generators(), env.lib.fvs_launch_count()
    with pytest.raises(exc):
        visual(px, thw, pos, vis)
    torch.cuda.synchronize()
    assert env.lib.fvs_launch_count() == n0
    assert _same_generators(_generators(), before)
    with pytest.raises(ValueError, match="smaller than one temporal patch"):
        env.rt.VisualB200(env.M.FlashMemory(**S_CFG), env.mergers["bf16"], encode_patches=env.towers["bf16"],
                          offline_max_rows=63)(px[:9 * 64], thw[:1], pos[:, :1], vis[:1])
    assert env.lib.fvs_launch_count() == n0
