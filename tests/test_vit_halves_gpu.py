"""GPU tests of the ViT layer stack run as two concurrent half-batches (vit_engine.cu stack_launches): a micro-batch
encoded in one call, split or not, gives the same bits as the same frames encoded one at a time through a one-frame
workspace, which never splits.  Odd frame counts give unequal halves.  Each shape runs eagerly (first call), through the
captured graph and through the profiled graph (event-record nodes in both branches)."""
import ctypes as C

import pytest
import torch

from oracle import fvs_oracle as O
from tests import golden_inputs as GI
from tests.test_gpu_parity import fvs  # noqa: F401  (fixture)

pytestmark = pytest.mark.gpu

FRAMES = (2, 3, 5, 16, 17, 32)
SMALL = O.VitConfig(image_size=336, patch_size=14, hidden=256, heads=4, mlp=512, layers=3)   # 577 tokens: every nf splits
VIT_L = O.VitConfig(layers=3)


def engines(ops, cfg, dtype, max_batch):
    w = O.random_vit_weights(cfg, 21)
    mk = lambda mb: ops.VitEncoder(w, image_size=cfg.image_size, patch_size=cfg.patch_size, heads=cfg.heads,
                                   layers_run=cfg.layers - 1, dtype=dtype, max_batch=mb)
    return mk(max_batch), mk(1)


def pool3(ops, eng, pix, a, b):
    """fvs_vit_encode_pool3: the three pooled levels of every frame, (a x a, b x b, 1 x 1) x hidden"""
    F, D = pix.shape[0], eng.hidden
    outs = [torch.empty(F, n, D, dtype=torch.float16, device=pix.device) for n in (a * a, b * b, 1)]
    ops.L.check(eng.lib.fvs_vit_encode_pool3(eng._h, ops.L.ptr(pix), *[ops.L.ptr(o) for o in outs], F, a, b,
                                             ops.L.ptr(eng._ws), eng._ws.numel(), ops.L.cur_stream()),
                "fvs_vit_encode_pool3")
    return outs


def encode_all_ways(ops, run, nf):
    """run(nf) eagerly, captured, replayed, then captured and replayed as the profiled graph"""
    lib = ops.L.load()
    outs = [run(nf) for _ in range(3)]
    n = 4096
    bufs = ((C.c_int32 * n)(), (C.c_float * n)(), (C.c_double * n)())
    try:
        ops.L.check(lib.fvs_prof_enable(n))
        outs += [run(nf) for _ in range(2)]
        torch.cuda.synchronize()
        got = lib.fvs_prof_collect(*bufs, n)
    finally:
        lib.fvs_prof_enable(0)
    assert got > 0 and all(ms > 0 for ms in bufs[1][:got])
    return outs


@pytest.mark.parametrize("dtype", [torch.float16, torch.bfloat16])
def test_full_features_equal_one_frame_at_a_time(fvs, dtype):
    pkg, ops = fvs
    big, one = engines(ops, SMALL, dtype, 32)
    pix = (GI.vit_pixels(SMALL, 32, 5) * 0.5).to(dtype).cuda()
    want = one.encode(pix).clone()
    for nf in FRAMES:
        for out in encode_all_ways(ops, lambda k: big.encode(pix[:k]).clone(), nf):
            assert torch.equal(out, want[:nf]), nf


def test_pooled_tail_equals_one_frame_at_a_time(fvs):
    pkg, ops = fvs
    big, one = engines(ops, SMALL, torch.float16, 32)
    pix = (GI.vit_pixels(SMALL, 32, 6) * 0.5).half().cuda()
    want = [o.clone() for o in pool3(ops, one, pix, 4, 2)]
    for nf in FRAMES:
        for outs in encode_all_ways(ops, lambda k: [o.clone() for o in pool3(ops, big, pix[:k], 4, 2)], nf):
            for o, w in zip(outs, want):
                assert torch.equal(o, w[:nf]), nf


def test_vit_l_halves_split_and_keep_bits(fvs):
    """ViT-L/14-336 width (2 layers run): micro-batches from 2 frames on (32 in bench.py) run as two half-batches, twice
    the layer-stack launches of a single frame, and both tails equal one frame at a time"""
    pkg, ops = fvs
    big, one = engines(ops, VIT_L, torch.float16, 32)
    lib = ops.L.load()
    pix = (GI.vit_pixels(VIT_L, 32, 7) * 0.5).half().cuda()
    want = one.encode(pix).clone()
    want_pool = [o.clone() for o in pool3(ops, one, pix, 8, 4)]
    per_layer = 7                                                      # 2 LayerNorms, 4 GEMMs, attention
    stack = 2 + per_layer * (VIT_L.layers - 1)                         # + patch GEMM, pre-LayerNorm
    for nf, halves in ((1, 1), (2, 2), (17, 2), (32, 2)):
        n0 = lib.fvs_launch_count()
        first = big.encode(pix[:nf]).clone()                           # eager
        assert lib.fvs_launch_count() - n0 == 1 + halves * stack + 1, nf   # im2col, the stack, the tail
        assert torch.equal(first, want[:nf]), nf
        for out in encode_all_ways(ops, lambda k: big.encode(pix[:k]).clone(), nf):
            assert torch.equal(out, want[:nf]), nf
        for outs in encode_all_ways(ops, lambda k: [o.clone() for o in pool3(ops, big, pix[:k], 8, 4)], nf):
            for o, w in zip(outs, want_pool):
                assert torch.equal(o, w[:nf]), nf
