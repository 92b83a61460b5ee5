"""The Qwen2-VL vision tower at the grids real videos produce (CPU).  A 4:3 or 16:9 frame gives a grid with h != w, and
there the two rotary axes and the (h/2, w/2, 2, 2) row layout stop being interchangeable: a kernel that mixed them up
would pass every square-grid test.  This file pins the table of real grids to the frame pre-processor, pins the fp32
oracle to transformers' own tower on non-square grids, and shows that the inputs used on the GPU
(test_qwen_vit_grids_gpu.py) separate the true positions from the two plausible mix-ups by far more than the tolerance."""
import pytest
import torch

from flash_vstream_b200.preprocess import Qwen2VLFramePreprocessor
from oracle import qwen_oracle as QO
from tests import qwen_vit_inputs as VI
from tests.test_qwen_vit_gpu_parity import TOL, hf_vision_blocks, rel

# The reference CLI's settings (max_pixels = 4*224*224, additional_pool_size = flash_memory_temporal_poolsize = 2) and
# the processor's default max_pixels: (frames, frame H, frame W, max_pixels) -> grid (t, h, w), pooled grid
# (t, h/2, w/2).  Tokens per temporal patch: h*w full resolution, h*w/4 pooled.
CLI_MAX_PIXELS = 4 * 224 * 224
REAL_GRIDS = [
    (4, 336, 336, CLI_MAX_PIXELS, (2, 24, 24), (2, 12, 12)),         # 576 / 144 tokens: the square control
    (4, 480, 640, CLI_MAX_PIXELS, (2, 24, 36), (2, 12, 18)),         # 864 / 216: 4:3 landscape
    (4, 640, 480, CLI_MAX_PIXELS, (2, 36, 24), (2, 18, 12)),         # 864 / 216: portrait
    (4, 720, 1280, CLI_MAX_PIXELS, (2, 24, 40), (2, 12, 20)),        # 960 / 240: 16:9
    (4, 360, 640, CLI_MAX_PIXELS, (2, 24, 40), (2, 12, 20)),
    (4, 1080, 1920, CLI_MAX_PIXELS, (2, 24, 40), (2, 12, 20)),
    (4, 240, 1280, CLI_MAX_PIXELS, (2, 12, 72), (2, 6, 36)),         # 864 / 216: extreme aspect
    (4, 720, 1280, 28 * 28 * 1280, (2, 52, 92), (2, 26, 46)),        # 4784 / 1196: the processor's default max_pixels
]


@pytest.mark.parametrize("frames,height,width,max_pixels,grid,pooled", REAL_GRIDS)
def test_real_grid_table_matches_the_preprocessor(frames, height, width, max_pixels, grid, pooled):
    proc = Qwen2VLFramePreprocessor(max_pixels=max_pixels, additional_pool_size=2)
    assert proc.grid_thw(frames, height, width) == grid
    t, h, w = grid
    assert pooled == (t, h // 2, w // 2) and h % 4 == 0 and w % 4 == 0        # the pooled grid is still 2x2-mergeable
    assert QO.temporal_pool(torch.zeros(t * h * w, 1176), list(grid))[1] == list(pooled)


# ------------------------------------------------------------------------------------ the oracle, restated with knobs
def grid_positions(h, w, mutation=None):
    """(hpos, wpos) of every row of one frame, rows ordered (h/2, w/2, 2, 2) as rot_pos_emb lays them out.
    mutation='swap': hpos and wpos exchanged, row layout kept; 'transpose': the layout of the transposed (w x h) frame,
    i.e. what a position kernel that took the block row length from h instead of w would produce."""
    if mutation == "transpose":
        h, w = w, h
    hp = torch.arange(h).unsqueeze(1).expand(-1, w).reshape(h // 2, 2, w // 2, 2).permute(0, 2, 1, 3).flatten()
    wp = torch.arange(w).unsqueeze(0).expand(h, -1).reshape(h // 2, 2, w // 2, 2).permute(0, 2, 1, 3).flatten()
    if mutation == "swap":
        hp, wp = wp, hp
    return torch.stack([hp, wp], dim=-1)


# Localised rotary mistakes (rope_mutation of vit_forward / rope_apply), each touching a few percent of q and k or less:
#   'sin_sign'        the sign of sin flipped in one 8-dim group (dims 8g..8g+7 and their partners +40) of one head;
#   'extra_unrotated' dims 32..39 and 72..79 of every head (the 16-dim "extra" block of the kernel's layout) not rotated;
#   'partner_shift'   every dim rotated against partner d + 39 (d < 40) / d - 39 instead of d + 40 / d - 40.
ROPE_MUTATIONS = ("sin_sign", "extra_unrotated", "partner_shift")
SIN_SIGN_HEAD, SIN_SIGN_GROUP = 5, 2


def rope_apply(v, cos, sin, rope_mutation=None):
    """apply_rotary_pos_emb_vision: v * cos + rotate_half(v) * sin on v [rows, heads, hd], cos / sin [rows, 1, hd]
    (cat([angles, angles])), optionally with one of ROPE_MUTATIONS"""
    hd = v.shape[-1]
    half = hd // 2
    if rope_mutation == "partner_shift":
        rot = torch.cat([-v[..., half - 1:hd - 1], v[..., 1:half + 1]], dim=-1)
    else:
        rot = torch.cat([-v[..., half:], v[..., :half]], dim=-1)
    if rope_mutation == "sin_sign":
        sin = sin.expand(-1, v.shape[1], -1).clone()
        for d0 in (8 * SIN_SIGN_GROUP, half + 8 * SIN_SIGN_GROUP):
            sin[:, SIN_SIGN_HEAD, d0:d0 + 8] *= -1
    elif rope_mutation == "extra_unrotated":
        cos, sin = cos.clone(), sin.clone()
        for d0 in (half - 8, hd - 8):
            cos[..., d0:d0 + 8], sin[..., d0:d0 + 8] = 1, 0
    else:
        assert rope_mutation in (None, "partner_shift"), rope_mutation
    return v * cos + rot * sin


def vit_forward(patch_rows, grids, sd, *, depth, heads=16, eps=1e-6, dtype=torch.float64, device="cpu", mutation=None,
                head_chunk=4, rope_mutation=None):
    """QO.qwen_vit_forward in any precision on any device (test_oracle_restatement_is_the_oracle pins the two), with
    the rotary positions optionally mutated (see grid_positions) or the rotary itself (one of ROPE_MUTATIONS).
    Attention runs per segment and `head_chunk` heads at a time, so that a 4784-token segment fits on the GPU in fp64."""
    f = lambda k: sd[k].to(device=device, dtype=dtype)
    E = sd["patch_embed.proj.weight"].shape[0]
    hd = E // heads
    x = patch_rows.to(device=device, dtype=dtype) @ f("patch_embed.proj.weight").reshape(E, -1).T
    dim = hd // 2
    inv_freq = 1.0 / (10000.0 ** (torch.arange(0, dim, 2, dtype=torch.float) / dim))    # fp32, as the model computes it
    pos, segs = [], []
    for t, h, w in grids:
        pos.append(grid_positions(h, w, mutation).repeat(t, 1))
        segs += [h * w] * t
    pos = torch.cat(pos)
    freqs = torch.outer(torch.arange(int(max(max(g[1], g[2]) for g in grids)), dtype=torch.float), inv_freq)
    rot = freqs[pos].flatten(1)
    emb = torch.cat([rot, rot], dim=-1).to(device=device, dtype=dtype)
    cos, sin = emb.cos()[:, None, :], emb.sin()[:, None, :]

    def rope(v):
        return rope_apply(v, cos, sin, rope_mutation)

    ln = torch.nn.functional.layer_norm
    for i in range(depth):
        p = f"blocks.{i}."
        y = ln(x, (E,), f(p + "norm1.weight"), f(p + "norm1.bias"), eps)
        qkv = (y @ f(p + "attn.qkv.weight").T + f(p + "attn.qkv.bias")).reshape(-1, 3, heads, hd)
        q, k, v = rope(qkv[:, 0]), rope(qkv[:, 1]), qkv[:, 2]
        ctx, r0 = [], 0
        for n in segs:
            parts = []
            for h0 in range(0, heads, head_chunk):
                qs, ks, vs = (z[r0:r0 + n, h0:h0 + head_chunk].transpose(0, 1) for z in (q, k, v))
                parts.append(torch.softmax(qs @ ks.transpose(1, 2) * hd ** -0.5, dim=-1) @ vs)
            ctx.append(torch.cat(parts).transpose(0, 1).reshape(n, E))
            r0 += n
        x = x + torch.cat(ctx) @ f(p + "attn.proj.weight").T + f(p + "attn.proj.bias")
        y = ln(x, (E,), f(p + "norm2.weight"), f(p + "norm2.bias"), eps)
        hmid = y @ f(p + "mlp.fc1.weight").T + f(p + "mlp.fc1.bias")
        hmid = hmid * torch.sigmoid(1.702 * hmid)
        x = x + hmid @ f(p + "mlp.fc2.weight").T + f(p + "mlp.fc2.bias")
    return x


def clip_rows(c, wdt):
    """[full-resolution rows ; temporal_pool rows] of a seeded clip, pooled in the model dtype like the product"""
    px = VI.pixels(c, wdt)
    small, small_thw = QO.temporal_pool(px, [c["t"], c["h"], c["w"]])
    return torch.cat([px, small]), [(c["t"], c["h"], c["w"]), tuple(small_thw)]


def narrow(t, h, w, depth=1, embed=160, seed=301):
    return dict(depth=depth, embed=embed, heads=embed // 80, t=t, h=h, w=w, seed=seed)


# (case, grids evaluated in one call): landscape, portrait, extreme aspect, a real grid, and several grids at once
ORACLE_CASES = {
    "land_2x4x6": (narrow(2, 4, 6, depth=2), None),
    "port_1x6x4": (narrow(1, 6, 4, depth=2), None),
    "land_2x12x18": (narrow(2, 12, 18, embed=320), None),
    "wide_1x12x72": (narrow(1, 12, 72), None),
    "land_2x24x36": (narrow(2, 24, 36), None),
    "several": (narrow(0, 0, 0, depth=2), [(2, 4, 6), (1, 6, 4), (1, 12, 18), (2, 8, 2), (1, 2, 10)]),
}


def case_rows(c, grids, wdt):
    """the clip and its pooled grid when temporal_pool can pool it (h/2, w/2 even), else the grid alone"""
    if grids is None:
        if c["h"] % 4 == 0 and c["w"] % 4 == 0:
            return clip_rows(c, wdt)
        return VI.pixels(c, wdt), [(c["t"], c["h"], c["w"])]
    n = sum(t * h * w for t, h, w in grids)
    g = torch.Generator().manual_seed(c["seed"] + 7)
    return (torch.randn(n, 1176, generator=g) * 1.2).to(VI.DT[wdt]), grids


@pytest.mark.parametrize("name", list(ORACLE_CASES))
def test_oracle_matches_transformers_on_non_square_grids(name):
    c, grids = ORACLE_CASES[name]
    sd = VI.state_dict(c, "bf16")
    rows, grids = case_rows(c, grids, "bf16")
    want = hf_vision_blocks(sd, c, rows, grids, torch.float32, "cpu").float()
    got = QO.qwen_vit_forward(rows, grids, sd, depth=c["depth"], heads=c["heads"])
    err = rel(got, want)
    print(f"\n[{name}] oracle vs transformers fp32: {err:.2e}")
    assert err < 2e-5


def test_oracle_restatement_is_the_oracle():
    """vit_forward (fp32, no mutation) is QO.qwen_vit_forward: the GPU tests may use it in fp64 as the oracle"""
    c, grids = ORACLE_CASES["several"]
    sd = VI.state_dict(c, "f16")
    rows, grids = case_rows(c, grids, "f16")
    a = QO.qwen_vit_forward(rows, grids, sd, depth=c["depth"], heads=c["heads"])
    b = vit_forward(rows, grids, sd, depth=c["depth"], heads=c["heads"], dtype=torch.float32)
    assert rel(b, a) < 1e-6
    assert rel(vit_forward(rows, grids, sd, depth=c["depth"], heads=c["heads"]), a) < 2e-5


def test_positions_are_the_references():
    """grid_positions without a mutation is transformers' rot_pos_emb ordering; the mutations really differ from it"""
    from transformers.models.qwen2_vl import modeling_qwen2_vl as M
    from transformers.models.qwen2_vl.configuration_qwen2_vl import Qwen2VLVisionConfig
    cfg = Qwen2VLVisionConfig(depth=0, embed_dim=160, hidden_size=256, num_heads=2)
    model = M.Qwen2VisionTransformerPretrainedModel(cfg)
    for t, h, w in ((1, 4, 6), (2, 12, 72), (1, 36, 24)):
        freqs = model.rot_pos_emb(torch.tensor([[t, h, w]]))
        inv = model.rotary_pos_emb.inv_freq
        want = torch.stack([freqs[:, 0] / inv[0], freqs[:, inv.numel()] / inv[0]], dim=-1).round().long()
        assert torch.equal(grid_positions(h, w).repeat(t, 1), want)
        for m in ("swap", "transpose"):
            assert not torch.equal(grid_positions(h, w, m), grid_positions(h, w))


# The cases of test_qwen_vit_grids_gpu.py: (embed, depth, grids); the weights there are VI.state_dict at full width.
# Here the same grids at a narrow width show that a position mix-up moves the output by far more than the GPU tolerance
# (the GPU file checks the same at full width with its own fp64 references).
TEETH_CASES = {
    "land_864": [(2, 24, 36), (2, 12, 18)],
    "port_864": [(2, 36, 24), (2, 18, 12)],
    "wide_960": [(2, 24, 40), (2, 12, 20)],
    "wide_864": [(2, 12, 72), (2, 6, 36)],
    "many": [(1, 2, 4), (1, 4, 2), (2, 2, 6), (1, 6, 2), (1, 4, 8), (2, 8, 4), (1, 2, 10), (1, 10, 4), (1, 6, 8),
             (2, 8, 6), (1, 4, 12), (1, 12, 2), (1, 2, 16), (1, 16, 6), (2, 6, 10), (1, 10, 12)],
}


@pytest.mark.parametrize("wdt", ["f16", "bf16"])
@pytest.mark.parametrize("name", list(TEETH_CASES))
def test_position_mixups_are_far_outside_the_tolerance(name, wdt):
    grids = TEETH_CASES[name]
    c = narrow(0, 0, 0, depth=1, seed=311)
    sd = VI.state_dict(c, wdt)
    n = sum(t * h * w for t, h, w in grids)
    rows = (torch.randn(n, 1176, generator=torch.Generator().manual_seed(5)) * 1.2).to(VI.DT[wdt])
    true = vit_forward(rows, grids, sd, depth=1, heads=c["heads"], dtype=torch.float32)
    for m in ("swap", "transpose"):
        d = rel(vit_forward(rows, grids, sd, depth=1, heads=c["heads"], dtype=torch.float32, mutation=m), true)
        print(f"\n[{name} {wdt}] {m}: {d:.3f} (> {10 * TOL[wdt]:.3f} required)")
        assert d > 10 * TOL[wdt], (m, d)
