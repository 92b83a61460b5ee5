"""CPU: the pieces test_vit_block_stages_gpu.py stands on.  The restated perm_col is a bijection that keeps every rotary
pair (d, d + 40) in one aligned 8-column group, as qwen_rope_kernel assumes; the packed positions are transformers'
rot_pos_emb ids for every grid the GPU file encodes; the inv_freq = 0 companion's rotary is exact; and the rotary bound
accepts a CPU fp32 simulation of the kernel's arithmetic while rejecting the same simulation of each localised mistake."""
import pytest
import torch

from tests.test_kernel_bounds_gpu import DTYPES, check
from tests.test_qwen_vit_grids_host import ROPE_MUTATIONS, rope_apply
from tests.test_vit_block_stages_gpu import (GRIDS, HALF, HD, INV_FREQ, MIXED16, QWEN_CALLS, SEG_MOVE_GRID,
                                             packed_positions, perm_cols, rope_bound, to_natural, to_permuted)


def test_the_calls_cover_every_grid():
    assert len(MIXED16) == 16 and set(GRIDS) <= {g for c in QWEN_CALLS.values() for g in c}
    assert MIXED16[SEG_MOVE_GRID][0] == 2 and SEG_MOVE_GRID > 0


@pytest.mark.parametrize("heads", [1, 2, 16])
@pytest.mark.parametrize("sections", [1, 3])
def test_perm_cols_is_a_bijection_that_keeps_rotary_pairs_in_aligned_groups(heads, sections):
    perm = perm_cols(heads, sections)
    n = sections * heads * HD
    assert torch.equal(perm.sort().values, torch.arange(n))
    t = torch.randn(3, n)
    assert torch.equal(to_natural(to_permuted(t, heads, sections), heads, sections), t)
    p = perm.view(sections, heads, HD)
    lo, hi = p[..., :HALF], p[..., HALF:]
    d = torch.arange(HALF)
    is_main = d < 32
    # the partner sits 32 columns further in the main block, 8 in the extra block, at the same offset in its group
    assert torch.equal(hi - lo, torch.where(is_main, 32, 8).expand_as(lo))
    assert torch.equal(lo % 8, (d % 8).expand_as(lo))
    # dims 8g .. 8g + 7 fill one aligned 8-column group: the 16-byte vector the kernel rotates with one cos / sin slice
    groups = lo.view(sections, heads, 5, 8)
    assert torch.equal(groups - groups[..., :1], torch.arange(8).expand_as(groups))
    assert bool((groups[..., 0] % 8 == 0).all())
    # the kernel takes the angle of a main column from its offset in the head's 64, of an extra one from 32 + offset in 16
    main_base = (torch.arange(sections)[:, None] * heads + torch.arange(heads)[None, :]) * 64
    extra_base = sections * heads * 64 + (torch.arange(sections)[:, None] * heads + torch.arange(heads)[None, :]) * 16
    angle = torch.where(is_main, lo - main_base[..., None], 32 + lo - extra_base[..., None])
    assert torch.equal(angle, d.expand_as(lo))


def test_packed_positions_are_rot_pos_emb():
    """pos as the GPU test unpacks it equals transformers' rot_pos_emb ids, for every grid and for the 16-grid call"""
    from transformers.models.qwen2_vl import modeling_qwen2_vl as M
    from transformers.models.qwen2_vl.configuration_qwen2_vl import Qwen2VLVisionConfig
    model = M.Qwen2VisionTransformerPretrainedModel(Qwen2VLVisionConfig(depth=0, embed_dim=160, hidden_size=256,
                                                                        num_heads=2))
    inv = model.rotary_pos_emb.inv_freq
    for grids in [[g] for g in GRIDS] + [MIXED16]:
        freqs = model.rot_pos_emb(torch.tensor(grids))
        ids = torch.stack([freqs[:, 0] / inv[0], freqs[:, inv.numel()] / inv[0]], dim=-1).round().long()
        pos = packed_positions(grids)
        assert torch.equal(torch.stack([pos >> 16, pos & 0xFFFF], -1).long(), ids), grids


def test_rope_identity_companion_is_exact():
    """inv_freq = 0: cosf(0) = 1 and sinf(0) = 0 exactly, and fl(fl(x * 1) + fl(-y * 0)) rounds back to x for every
    finite f16 / bf16 x and y, up to the sign of a zero"""
    for dtype in (torch.float16, torch.bfloat16):
        v = torch.arange(-2 ** 15, 2 ** 15, dtype=torch.int32).to(torch.int16).view(dtype)
        x, y = v.float(), v.flip(0).float()
        r = (x * 1.0 + (-y) * 0.0).to(dtype)
        fin = torch.isfinite(x) & torch.isfinite(y)
        assert torch.equal(r[fin], v[fin])


def simulate_rope(pre, pos, rope_mutation=None):
    """qwen_rope_kernel's arithmetic on the CPU: fp32 angle, cos and sin, fp32 products and sum as separate roundings
    (no FMA), round to nearest even into the 16-bit dtype"""
    rows = pre.shape[0]
    p = torch.stack([pos >> 16, pos & 0xFFFF], -1).float()
    ang = (p[:, :, None] * INV_FREQ[None, None, :]).reshape(rows, HALF)
    a = torch.cat([ang, ang], -1)[:, None, :]
    x = pre.float()
    out = torch.stack([rope_apply(x[:, i], a.cos(), a.sin(), rope_mutation) for i in range(2)], 1)
    return out.to(pre.dtype)


@pytest.mark.parametrize("dt", list(DTYPES))
def test_rope_bound_accepts_the_kernel_arithmetic_and_rejects_each_mistake(dt):
    dtype = DTYPES[dt]
    grids = [(1, 24, 36), (1, 12, 72), (1, 2, 2), (1, 52, 92)]
    pos = packed_positions(grids)
    g = torch.Generator().manual_seed(7)
    pre = (torch.randn(pos.numel(), 2, 16, HD, generator=g) * 2).to(dtype)
    out = simulate_rope(pre, pos)
    ref, bound, rounding = rope_bound(pre, pos, INV_FREQ, out)
    check(f"rotary {dt} fp32 simulation", out, ref, bound, rounding)
    err = (out.double() - ref).abs()
    before = float(((err - rounding).clamp(min=0) / (bound - rounding)).max())
    assert before < 0.5, before
    for m in ROPE_MUTATIONS:
        wrong = simulate_rope(pre, pos, m)
        with pytest.raises(AssertionError):
            check(f"rotary {dt} fp32 simulation of mistake '{m}' (must fail)", wrong, *rope_bound(pre, pos, INV_FREQ, wrong))
