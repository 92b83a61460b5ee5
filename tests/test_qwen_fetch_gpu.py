"""GPU tests of the Qwen2-VL evaluation drivers' pre-processing on the device (preprocess.Qwen2VLVideoFetcher, the
two-stage jobs of fvs_preprocess_multi and install_qwen_fetch), byte- and bit-equal on every case of
tests/golden/qwen_fetch.npz: the fetched 8-bit video against the golden and Pillow called here; the processor's rows and
their codes against the golden and the oracle; one mixed-size call against the per-video calls; the drop-in against the
same rows; the single-stage path on the fetched video; and one offline vision pass fed either rows."""
import random
import types

import numpy as np
import pytest
import torch
from PIL import Image

from flash_vstream_b200 import preprocess as P
from tests import preprocess_oracle as O
from tests import qwen_fetch_inputs as QF
from tests.test_qwen_fetch_host import GOLDEN, case, digest, golden_pixels, golden_stage1

pytestmark = pytest.mark.gpu
NAMES = list(QF.CASES)


@pytest.fixture(scope="module")
def g():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    return np.load(GOLDEN)


def fetcher(pool):
    return P.Qwen2VLVideoFetcher(P.Qwen2VLFramePreprocessor(QF.PROC_MIN_PIXELS, QF.PROC_MAX_PIXELS, pool))


def element(name, kind="array", tmp_path=None):
    f, ele, pool = case(name)
    if kind == "pil":
        frames = [Image.fromarray(x) for x in f]
    elif kind == "path":
        frames = []
        for i, x in enumerate(f):
            Image.fromarray(x).save(tmp_path / f"{name}_{i}.png")
            frames.append(("file://" if i % 2 else "") + str(tmp_path / f"{name}_{i}.png"))
    else:
        frames = list(f)
    return f, dict(ele, video=frames), pool


@pytest.mark.parametrize("name", NAMES)
@pytest.mark.parametrize("kind", ["array", "pil", "path"])
def test_fetch_equals_golden_and_pillow(g, name, kind, tmp_path):
    f, ele, pool = element(name, kind, tmp_path)
    got = fetcher(pool).fetch(ele)
    want = golden_stage1(g, name)
    assert got.is_cuda and got.dtype == torch.uint8 and tuple(got.shape) == want.shape
    got = got.cpu().numpy()
    assert np.array_equal(got, want)
    h1, w1 = want.shape[1:3]
    picks = P.fetch_video_picks(len(f), ele)
    pil = np.stack([np.asarray(Image.fromarray(f[i]).convert("RGB").resize((w1, h1))) for i in picks])
    assert np.array_equal(got, pil)


@pytest.mark.parametrize("name", NAMES)
def test_rows_and_codes_equal_golden_and_oracle(g, name):
    f, ele, pool = element(name)
    fx = fetcher(pool)
    got = fx(ele)
    want = golden_pixels(g, name)
    pix = got["pixel_values_videos"]
    assert pix.is_cuda and pix.dtype == torch.float32
    assert digest(pix.cpu().numpy()) == str(g[f"{name}_pixels_sha256"])
    assert np.array_equal(pix.cpu().numpy().view(np.uint32), want.view(np.uint32))
    stage1 = golden_stage1(g, name)
    h2, w2 = fx.pre.resized(*stage1.shape[1:3])
    _, grid = O.qwen_pixels(stage1, (h2, w2), fx.pre.table)
    assert got["video_grid_thw"].dtype == torch.int64 and not got["video_grid_thw"].is_cuda
    assert got["video_grid_thw"].tolist() == [list(g[f"{name}_grid"])] == [list(grid)]
    codes = fx(ele, codes=True)["pixel_values_videos"]
    want_codes, _ = O.qwen_patchify(np.moveaxis(O.resize(stage1, h2, w2), -1, 1))      # the bytes before the table
    assert codes.dtype == torch.uint8 and np.array_equal(codes.cpu().numpy(), want_codes)


@pytest.mark.parametrize("name", NAMES)
def test_single_stage_on_the_fetched_video(g, name):
    """the second stage alone, Qwen2VLFramePreprocessor on the fetched video, gives the chain's rows"""
    _, ele, pool = element(name)
    fx = fetcher(pool)
    video = fx.fetch(ele)
    single = fx.pre(video)
    chain = fx(ele)
    assert torch.equal(single["pixel_values_videos"], chain["pixel_values_videos"])
    assert torch.equal(single["video_grid_thw"], chain["video_grid_thw"])


@pytest.mark.parametrize("pool", [1, 2])
def test_many_mixed_sizes_equals_per_video_calls(g, pool):
    eles = [element(n)[1] for n in NAMES] * 3          # more than 32 videos: two launch groups
    fx = fetcher(pool)
    got = fx.many(eles)
    one = [fx(e) for e in eles]
    assert torch.equal(got["pixel_values_videos"], torch.cat([o["pixel_values_videos"] for o in one]))
    assert torch.equal(got["video_grid_thw"], torch.cat([o["video_grid_thw"] for o in one]))


def _vision_utils():
    """a qwen_vl_utils stand-in with the names install_qwen_fetch reads (the path / image branches are not taken)"""
    def extract_vision_info(conversations):
        return [ele for msg in conversations for ele in msg["content"] if "video" in ele or "image" in ele]

    def untouched(_):
        raise AssertionError("a list-of-frames video went to the CPU fetch")
    return types.SimpleNamespace(__name__="qwen_vl_utils", extract_vision_info=extract_vision_info,
                                 fetch_image=untouched, fetch_video=untouched, process_vision_info=untouched)


class _ImageProcessor:
    """the attributes of the drivers' FlashVStreamQwen2VLImageProcessor that the GPU stand-in reads"""
    resample, do_resize, do_rescale, do_normalize, rescale_factor = 3, True, True, True, 1 / 255
    patch_size, merge_size, temporal_patch_size = 14, 2, 2
    min_pixels, max_pixels = QF.PROC_MIN_PIXELS, QF.PROC_MAX_PIXELS
    image_mean, image_std = P.OPENAI_CLIP_MEAN, P.OPENAI_CLIP_STD

    def __call__(self, **kw):
        raise AssertionError("a device video went to the CPU processor")


def test_drop_in(g):
    from flash_vstream_b200.install import install_qwen_fetch
    vu = _vision_utils()
    processor = types.SimpleNamespace(image_processor=_ImageProcessor())
    patched = install_qwen_fetch(processor, vision_utils=vu)
    assert patched == ["qwen_vl_utils.process_vision_info", "SimpleNamespace.image_processor"]
    assert processor.image_processor.merge_size == 2
    for pool in (1, 2):
        names = [n for n in NAMES if QF.CASES[n][3] == pool]
        messages = [{"role": "user", "content": [element(n)[1], {"type": "text", "text": "?"}]} for n in names]
        images, videos = vu.process_vision_info(messages)
        assert images is None and len(videos) == len(names)
        for n, v in zip(names, videos):
            assert v.is_cuda and np.array_equal(v.cpu().numpy(), golden_stage1(g, n))
        got = processor.image_processor(images=None, videos=videos, return_tensors="pt", additional_pool_size=pool)
        want = np.concatenate([golden_pixels(g, n) for n in names])
        assert got["pixel_values_videos"].is_cuda
        assert np.array_equal(got["pixel_values_videos"].cpu().numpy().view(np.uint32), want.view(np.uint32))
        assert got["video_grid_thw"].tolist() == [list(g[f"{n}_grid"]) for n in names]
        fx = fetcher(pool)
        assert torch.equal(got["pixel_values_videos"], fx.many([element(n)[1] for n in names])["pixel_values_videos"])


def test_offline_vision_pass_fed_the_device_rows(g):
    """VisualB200.forward (small tower) on the fetcher's rows equals the same pass on the CPU processor's rows (the
    oracle's, held to the reference's digest)"""
    from flash_vstream_b200.qwen import vision_tower, vstream_qwen2vl_model, vstream_qwen2vl_realtime
    from tests import qwen_offline_inputs as OI
    from tests.qwen_inputs import DT
    name = "up_up"                                                          # grid (1, 8, 8)
    tower = vision_tower.QwenVisionBlocksB200(OI.tower_state_dict("bf16"), depth=OI.TOWER["depth"],
                                              heads=OI.TOWER["heads"], dtype=DT["bf16"])
    w = OI.merger_weights("bf16")
    merger = vstream_qwen2vl_realtime.PatchMerger.from_weights(
        {"ln_w": w["ln_q.weight"], "ln_b": w["ln_q.bias"], "fc1_w": w["mlp.0.weight"], "fc1_b": w["mlp.0.bias"],
         "fc2_w": w["mlp.2.weight"], "fc2_b": w["mlp.2.bias"]})
    try:
        fm = vstream_qwen2vl_model.FlashMemory(flash_memory_temporal_length=12, flash_memory_spatial_length=8)
        visual = vstream_qwen2vl_realtime.VisualB200(fm, merger, encode_patches=tower, dtype=DT["bf16"])
        rows = fetcher(2)(element(name)[1])
        grid = tuple(int(v) for v in rows["video_grid_thw"][0])
        pos, vis = OI.positions([OI.n_visual(grid, fm.temporal_length, fm.spatial_length, fm.temporal_poolsize)])
        outs = []
        for px in (rows["pixel_values_videos"], torch.from_numpy(golden_pixels(g, name)).cuda()):
            torch.manual_seed(5)
            random.seed(5)
            outs.append(visual(px.to(DT["bf16"]), rows["video_grid_thw"].cuda(), pos.clone().cuda(), vis.cuda()))
        (a, pa), (b, pb) = outs
        assert torch.equal(a.view(torch.int16), b.view(torch.int16)) and torch.equal(pa, pb)
    finally:
        tower.close()
