"""GPU tests of the frame pre-processing (fvs_preprocess / flash_vstream_b200.preprocess): both layouts bit-identical to
the numpy oracle and to the reference goldens, whatever the input size, the split of a clip across calls, or where the
frames come from; the towers and the streaming memory fed from them end bit-identical to feeding the oracle's pixels;
a refused call launches nothing."""
import random

import numpy as np
import pytest
import torch

from flash_vstream_b200 import preprocess as P
from tests import preprocess_inputs as PI
from tests import preprocess_oracle as O
from tests.test_gpu_parity import cu, fvs, make_model  # noqa: F401  (fvs is a fixture)
from tests.test_preprocess_host import GOLDEN, _clip_processor
from tests.test_stream_step_gpu import small_tower

pytestmark = pytest.mark.gpu

SHAPES = {"480p": (2, 480, 640), "720p": (2, 720, 1280), "1080p": (2, 1080, 1920), "portrait": (2, 1280, 720),
          "tiny_up": (2, 90, 100)}


def _frames(shape, seed=1):
    return PI.frames(seed, shape)


def _oracle_clip(proc, f):
    resized, crop = proc.sizes(*f.shape[1:3])
    return torch.from_numpy(O.clip_pixels(f, resized, crop, proc.table)).half()


def _oracle_qwen(proc, f):
    pix, grid = O.qwen_pixels(f, proc.resized(*f.shape[1:3]), proc.table)
    return torch.from_numpy(pix), torch.tensor([grid])


@pytest.mark.parametrize("name", list(SHAPES))
def test_clip_layout_equals_oracle(fvs, name):
    f = _frames(SHAPES[name])
    proc = P.CLIPFramePreprocessor(_clip_processor())
    got = proc(torch.from_numpy(f).cuda())
    assert got.dtype == torch.float16 and got.is_cuda and got.shape == (f.shape[0], 3, 336, 336)
    assert torch.equal(got.cpu(), _oracle_clip(proc, f))


@pytest.mark.parametrize("name", list(SHAPES))
@pytest.mark.parametrize("pool", [1, 2])
def test_qwen_layout_equals_oracle(fvs, name, pool):
    f = _frames(SHAPES[name])
    proc = P.Qwen2VLFramePreprocessor(additional_pool_size=pool)
    got = proc(torch.from_numpy(f).cuda())
    pix, grid = _oracle_qwen(proc, f)
    assert torch.equal(got["video_grid_thw"], grid) and got["video_grid_thw"].dtype == torch.int64
    assert got["pixel_values_videos"].is_cuda and torch.equal(got["pixel_values_videos"].cpu(), pix)


def test_qwen_one_frame_fills_both_temporal_slots(fvs):
    f = _frames((1, 720, 1280), 4)
    proc = P.Qwen2VLFramePreprocessor()
    got = proc(torch.from_numpy(f).cuda())
    pix, grid = _oracle_qwen(proc, f)
    assert grid[0, 0] == 1 and torch.equal(got["video_grid_thw"], grid) and torch.equal(got["pixel_values_videos"].cpu(), pix)
    with pytest.raises(ValueError, match="even"):
        proc(torch.from_numpy(_frames((3, 56, 56))).cuda())


def test_goldens(fvs):
    g = np.load(GOLDEN)
    for name, (seed, shape, se, crop) in PI.CLIP_CASES.items():
        got = P.CLIPFramePreprocessor(_clip_processor(se, crop))(torch.from_numpy(PI.frames(seed, shape)).cuda())
        assert torch.equal(got.cpu(), torch.from_numpy(g[f"clip_{name}"])), name
    for name, (seed, shape, mn, mx, pool) in PI.QWEN_CASES.items():
        got = P.Qwen2VLFramePreprocessor(mn, mx, pool)(torch.from_numpy(PI.frames(seed, shape)).cuda())
        assert torch.equal(got["pixel_values_videos"].cpu(), torch.from_numpy(g[f"qwen_{name}"])), name
        assert torch.equal(got["video_grid_thw"], torch.from_numpy(g[f"qwen_{name}_grid"]).reshape(1, 3)), name


def test_split_calls_and_host_input_give_the_same_bits(fvs):
    f = torch.from_numpy(_frames((8, 720, 1280), 6))
    clip, qwen = P.CLIPFramePreprocessor(_clip_processor()), P.Qwen2VLFramePreprocessor(additional_pool_size=2)
    whole = clip(f.cuda())
    parts = torch.cat([clip(f[i:i + n].cuda()) for i, n in ((0, 1), (1, 3), (4, 4))])
    assert torch.equal(whole, parts)
    assert torch.equal(whole, clip(f.pin_memory()))
    assert torch.equal(whole, clip(f.numpy()))                     # pageable host memory: copied, then processed
    q = qwen(f.cuda())["pixel_values_videos"]
    rows = q.shape[0] // 4
    assert torch.equal(q, torch.cat([qwen(f[i:i + 2].cuda())["pixel_values_videos"] for i in range(0, 8, 2)]))
    assert torch.equal(q[:rows], qwen(f[:2].pin_memory())["pixel_values_videos"])
    # caller-owned output and workspace: no allocation, the same bits
    out = torch.empty_like(whole)
    ws = torch.empty(clip.workspace_bytes(8, 720, 1280), dtype=torch.uint8, device="cuda")
    assert clip(f.cuda(), out=out, workspace=ws) is out and torch.equal(out, whole)


def test_refused_call_launches_nothing(fvs):
    pkg, ops = fvs
    lib = ops.L.load()
    clip = P.CLIPFramePreprocessor(_clip_processor(336, 400))      # a crop larger than the 336 resize
    qwen = P.Qwen2VLFramePreprocessor()
    n0 = lib.fvs_launch_count()
    for call, frames in ((clip, _frames((1, 480, 640))), (qwen, _frames((3, 56, 56))), (qwen, np.zeros((2, 56, 56, 4), np.uint8))):
        with pytest.raises(ValueError):
            call(torch.from_numpy(frames).cuda())
    with pytest.raises(ValueError, match="workspace"):
        P.CLIPFramePreprocessor(_clip_processor())(torch.from_numpy(_frames((2, 480, 640))).cuda(),
                                                   workspace=torch.empty(16, dtype=torch.uint8, device="cuda"))
    torch.cuda.synchronize()
    assert lib.fvs_launch_count() == n0


def test_streaming_banks_from_gpu_pixels_equal_oracle_pixels(fvs):
    """embed_video_streaming and StreamPool.step fed by the GPU pre-processing end bit-identical to the same calls fed the
    oracle's pixels (the tower takes 112 x 112 pixels: a 112 shortest-edge processor)"""
    pkg, ops = fvs
    cfg, tower = small_tower(pkg)
    D, seed = cfg.hidden, 33
    star = dict(compress_size=4, compress_long_memory_size=2)
    proc = P.CLIPFramePreprocessor(_clip_processor(112, 112))
    chunks = [1, 4, 8, 8, 3, 8]                                  # 32 frames: crosses the 25-slot warm-up
    f = _frames((sum(chunks), 360, 640), 8)
    gpu_model, ref_model = make_model(D, seed, pkg, tower=tower, **star), make_model(D, seed, pkg, tower=tower, **star)
    pool = pkg.StreamPool(make_model(D, seed, pkg, tower=tower, **star), chunk_cap=8)
    sid = pool.open()
    from tests.test_multistream_gpu import assert_same_stream, draws_for
    pos = 0
    for r, n in enumerate(chunks):
        pix_gpu = proc(torch.from_numpy(f[pos:pos + n]).cuda())
        pix_ref = _oracle_clip(proc, f[pos:pos + n]).cuda()
        assert torch.equal(pix_gpu, pix_ref)
        d = draws_for(ref_model._fvs_bank, n, seed * 10 + r) if r else None
        ref_model.embed_video_streaming(pix_ref.unsqueeze(0), draws=d)
        gpu_model.embed_video_streaming(pix_gpu.unsqueeze(0), draws=d)
        pool.step({sid: pix_gpu.unsqueeze(0)}, draws={sid: d} if d is not None else {})
        pos += n
        assert_same_stream(pool.bank(sid), ref_model, r)
        for a, b in zip(gpu_model.video_embedding_memory, ref_model.video_embedding_memory):
            assert torch.equal(a, b), r


def test_qwen_clip_state_from_gpu_pixels_equals_oracle_pixels(fvs):
    """embed_new_video_clip on the GPU pre-processing's dict == on the oracle's pixel_values_videos: all 13 items"""
    import flash_vstream_b200.qwen.vstream_qwen2vl_realtime as rt
    from flash_vstream_b200.qwen.vision_tower import QwenVisionBlocksB200
    from tests import qwen_rt_inputs as RI
    from tests import qwen_vit_inputs as VI
    from tests.test_qwen_rt_gpu_parity import cuda_w
    sd = VI.state_dict(dict(depth=1, embed=1280, heads=16, seed=97), "bf16")
    w = RI.merger_weights(1280, 256, "bf16", 98)

    def host():
        flash = rt.FlashMemory(flash_memory_temporal_length=6, flash_memory_spatial_length=4)
        tower = QwenVisionBlocksB200(sd, depth=1, heads=16, dtype=torch.bfloat16)
        return rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(flash, rt.PatchMerger.from_weights(cuda_w(w)),
                                                                encode_patches=tower))
    proc = P.Qwen2VLFramePreprocessor(max_pixels=112 * 112, additional_pool_size=2)
    clips = [_frames((2, 100, 120), 30 + i) for i in range(4)]          # upscaled to 112 x 112: grid 8 x 8
    states = []
    for feed in ("gpu", "oracle"):
        model = host()
        torch.manual_seed(11)
        random.seed(11)
        for s, f in enumerate(clips):
            if feed == "gpu":
                inputs = proc(torch.from_numpy(f).cuda())
            else:
                pix, grid = _oracle_qwen(proc, f)
                inputs = {"pixel_values_videos": pix, "video_grid_thw": grid}
            model.embed_new_video_clip(**inputs, start_idx=2 * s)
        states.append(model.get_video_embedding_memory_cuda_list())
    a, b = states
    assert len(a) == len(b) == 13
    for i, (x, y) in enumerate(zip(a, b)):
        if isinstance(x, torch.Tensor):
            assert x.dtype == y.dtype and torch.equal(x, y.to(x.device)), i
        else:
            assert x == y, i
