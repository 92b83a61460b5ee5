"""Fixtures and helpers of tests/test_qwen_mem_multi_gpu.py: the small-depth tower and merger, hosts, clips, streams
stepped alone through QwenStreamState (the single-stream memory path every pool stream is held against) and the
bit-for-bit comparison of two states."""
import pytest
import torch

from tests import qwen_rt_inputs as RI
from tests import qwen_vit_inputs as VI

D, DM = 1280, 512


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


def clip(seed, t, h=8, w=8, repeat=False, device="cuda:0"):
    """patch rows [t*h*w, 1176] (bf16, device) and the grid; `repeat`: the second temporal patch repeats the first"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(t, h * w, 1176, generator=g)
    if repeat:
        x[1] = x[0]
    return x.reshape(-1, 1176).bfloat16().to(device), torch.tensor([[t, h, w]])


def bits(t):
    t = t.cpu()
    return t.view(torch.int16) if t.dtype in (torch.bfloat16, torch.float16) else t


def same_rng(a, b):
    a.settle()
    b.settle()
    return torch.equal(a.cpu, b.cpu) and torch.equal(a.cuda, b.cuda) and a.py.getstate() == b.py.getstate()


def same(a, b):
    if a is None or b is None:
        return a is None and b is None
    if not torch.is_tensor(a):
        return a == b
    return a.dtype == b.dtype and a.shape == b.shape and torch.equal(bits(a), bits(b))


class Alone:
    """one stream stepped alone: the host's own tower pass (forward_simple_not_merge) and QwenStreamState.step"""

    def __init__(self, host, seed, device_frames=None, small_device_frames=None):
        from flash_vstream_b200.draws import DrawSource
        from flash_vstream_b200.qwen.stream_state import QwenStreamState
        v = host.visual
        self.visual = v
        self.st = QwenStreamState(v.flash_memory, v.merger, device_frames=device_frames,
                                  small_device_frames=small_device_frames)
        self.st.rng = DrawSource(seed, "cuda")

    def step(self, c):
        pix, thw = c
        t, h, w = (int(v) for v in thw[0])
        feats, _, _ = self.visual.forward_simple_not_merge(pix, thw)
        n = t * h * w
        self.st.step(feats[:n], feats[n: n + n // 4], t, (h, w), (h // 2, w // 2), self.st.n_frames)

    @staticmethod
    def compare(a, b, tag):
        """states a and b hold the same bits: counters, generators, the 13-item list, video_embeds, DAM and CSM"""
        for k in ("n_frames", "steps", "fast_steps", "redone_steps", "n_tem", "grid", "small_grid", "n_host", "n_small_host"):
            assert getattr(a, k) == getattr(b, k), (tag, k)
        assert same_rng(a.rng, b.rng), tag
        if a.n_frames == 0:
            return
        for i, (u, v) in enumerate(zip(a.as_list(), b.as_list())):
            assert same(u, v), (tag, i)
        for k in ("video_embeds", "spa_positions", "spa_x", "tem_x", "tem_weights", "tem_timestamp"):
            assert same(getattr(a, k), getattr(b, k)), (tag, k)


def run(pool, alone, rounds, tag, others=()):
    """rounds: [{sid: clip}]; the pool (and every pool in `others`) steps each round, the lone streams step the same
    clips, and every stream of every pool is compared with its lone twin after every round"""
    for r, rnd in enumerate(rounds):
        for p in (pool, *others):
            p.step(rnd)
        for sid, c in rnd.items():
            alone[sid].step(c)
        for p in (pool, *others):
            for sid in alone:
                Alone.compare(p.state(sid), alone[sid].st, (tag, r, sid, p.BATCH_MIN_JOBS))
