"""GPU: fvs_attention / fvs_attention80 at shapes that exercise the persistent schedule (one CTA per SM walking many
(query block, head, frame) tiles) and both sides of the narrow last KV tile (16 valid keys: m64n16 path, 17: full width),
against fp32 torch attention and bit for bit against a second launch.  The shared helpers and tolerances are those of
test_attention_variants_gpu.py."""
import pytest
import torch

from tests.test_attention_variants_gpu import REL_TOL, reference, rel, run

pytestmark = pytest.mark.gpu

CASES = [  # (head_dim, dtype, frames, tokens, heads)
    (64, torch.float16, 32, 577, 16),     # the bench shape: 2560 tiles, ~19 per persistent CTA
    (64, torch.float16, 8, 592, 16),      # last KV tile with 16 valid keys: narrow
    (64, torch.bfloat16, 8, 593, 16),     # 17 valid keys: full width
    (80, torch.bfloat16, 8, 592, 16),
    (80, torch.float16, 8, 593, 16),
    (80, torch.bfloat16, 40, 16, 16),     # a single KV tile that is narrow
    (64, torch.bfloat16, 2, 300, 16),     # 96 tiles: fewer than the SMs
    (64, torch.float16, 7, 577, 16),      # 560 tiles: not a multiple of the grid
    (80, torch.float16, 3, 593, 16),      # 240 tiles: one wave plus part of a second
]


@pytest.mark.parametrize("hd,dtype,frames,tokens,heads", CASES)
def test_attention_persistent_matches_fp32_and_is_deterministic(hd, dtype, frames, tokens, heads):
    from flash_vstream_b200 import ops
    g = torch.Generator().manual_seed(frames * 1000 + tokens + hd)
    nat = torch.randn(frames * tokens, 3 * heads * hd, generator=g).to(dtype).cuda()
    ref = reference(nat, frames, tokens, heads, hd)
    first = run(ops, nat, frames, tokens, heads, hd)
    second = run(ops, nat, frames, tokens, heads, hd)
    tol = REL_TOL if dtype == torch.float16 else 8e-3
    assert rel(first.float(), ref) < tol
    assert rel(second.float(), ref) < tol
    assert torch.equal(first, second)
