"""Host: the shape derivations of tests/vit_kernel_edges.py give every schedule the GPU sweep promises, and its guard
checker reports a flipped guard bit and an unwritten output element (the harness is shown to bite before it is trusted)."""
import math

import pytest
import torch

from tests import vit_kernel_edges as VE

SM_COUNTS = [132, 114]                       # H100 SXM and H100 PCIe


@pytest.mark.parametrize("bn", [128, 256])
@pytest.mark.parametrize("n_sms", SM_COUNTS)
def test_gemm_sweep_covers_every_schedule(n_sms, bn):
    stages = VE.K_STAGES[bn]
    for n in VE.SWEEP_N[bn]:
        num_n = -(-n // bn)
        g = math.gcd(num_n, n_sms)
        sched = [VE.gemm_schedule(n_sms, m, n_, k, bn) for m, n_, k, _ in VE.gemm_sweep_shapes(n_sms, n, bn)]
        assert all(n_ == n and m > 0 and k % 8 == 0 for m, n_, k, _ in VE.gemm_sweep_shapes(n_sms, n, bn))
        # last waves: empty, the smallest and the fullest partial one, each after one and after >= 20 full waves
        for waves in (1, VE.MANY):
            got = {r for tiles, grid, r, per, kb in sched if tiles > waves * grid}
            assert {0, g, n_sms - g} <= got, (n, waves, got)
        # tiles per CTA: exactly 1 on a single wave with every CTA busy but < num_n idle, exactly 2, and >= 20
        per_cta = {per for *_, per, kb in sched}
        assert {1, 2} <= per_cta and max(per_cta) >= VE.MANY, (n, per_cta)
        assert any(per == 1 and grid > n_sms - num_n for tiles, grid, r, per, kb in sched)
        # the K loop below, at and above the ring depth, on a single wave and with >= 20 tiles per CTA
        for lo, hi in ((1, 1), (2, 2), (VE.MANY, 10 ** 9)):
            kbs = {kb for tiles, grid, r, per, kb in sched if lo <= per <= hi}
            assert min(kbs) < stages and stages in kbs, (n, lo, kbs)
            if hi < VE.MANY:
                assert max(kbs) > stages, (n, lo, kbs)
        # M: full last row blocks and last blocks of 1 and of 64 rows
        assert {m % VE.BM for m, *_ in VE.gemm_sweep_shapes(n_sms, n, bn)} >= {0, 1, 64}
    # at each width one N gives last waves of exactly 1 and SMs - 1 tiles
    exact = [n for n in VE.SWEEP_N[bn] if math.gcd(-(-n // bn), n_sms) == 1]
    assert exact, (bn, n_sms)
    for n in exact:
        rs = {VE.gemm_schedule(n_sms, m, n, k, bn)[2] for m, _, k, _ in VE.gemm_sweep_shapes(n_sms, n, bn)}
        assert {0, 1, n_sms - 1} <= rs


def test_gemm_sweep_k_tails():
    """K % 64 in {8, 0} among the sweep's K, 56 among the guard shapes' (tests/test_vit_kernel_edges_gpu.py)"""
    for bn in (128, 256):
        assert {k % 64 for k in VE.sweep_ks(bn)} >= {0, 8}


@pytest.mark.parametrize("n_sms", SM_COUNTS)
@pytest.mark.parametrize("tokens", [65, 129, 577, 36, 100])
def test_attention_sweep_covers_every_last_wave(n_sms, tokens):
    heads = 5
    per_frame = -(-tokens // VE.BM) * heads
    g = math.gcd(per_frame, n_sms)
    got = []
    for frames, _ in VE.attention_sweep_frames(n_sms, tokens, heads):
        tiles = per_frame * frames
        grid = min(n_sms, tiles)
        got.append((tiles % grid, -(-tiles // grid), tiles > grid))
    assert {r for r, _, more in got if more} >= {0, g, n_sms - g}
    assert {per for _, per, _ in got} >= {1, 2}
    if g == 1:
        assert {r for r, _, more in got if more} >= {0, 1, n_sms - 1}


def harness_catches_planted_faults(device):
    """For every sentinel (input quiet NaN, output marked NaN) and dtype: a clean guarded buffer reports nothing; one
    flipped low bit in a guard row, in a pitch column, and one output element left at the sentinel are each reported.
    A flipped low bit keeps the guard a NaN, so only the bitwise comparison can see it."""
    for kind, table in (("in", VE.IN_BITS), ("out", VE.OUT_BITS)):
        for dtype, bits in table.items():
            ib = {2: torch.int16, 4: torch.int32}[torch.empty((), dtype=dtype).element_size()]
            payload = torch.randn(5, 24, generator=torch.Generator().manual_seed(3)).to(dtype).to(device)
            tag = f"{kind} {dtype}"
            buf, view = VE.guarded(payload, 3, 8, bits)
            assert VE.report(tag, buf, 5, 24, bits) == [], tag
            assert torch.equal(view, payload), tag
            for r, c in ((6, 2), (1, 27)):                    # a row past the payload, a pitch column
                buf, view = VE.guarded(payload, 3, 8, bits)
                buf.view(ib)[r, c] ^= 1
                assert torch.isnan(buf[r, c]), tag
                probs = VE.report(tag, buf, 5, 24, bits)
                assert len(probs) == 1 and "guard" in probs[0] and f"[{r}, {c}]" in probs[0], (tag, probs)
            buf, view = VE.guarded(payload, 3, 8, bits)
            view.view(ib)[2, 5] = bits                       # an element the kernel "never wrote"
            probs = VE.report(tag, buf, 5, 24, bits)
            assert len(probs) == 1 and "1 of them still the sentinel" in probs[0], (tag, probs)
            assert VE.report(tag, buf, 5, 24, bits, written=False) == [], tag
            buf, view = VE.blank(5, 24, dtype, 3, 8, bits, device)
            assert "120 of them still the sentinel" in VE.report(tag, buf, 5, 24, bits)[0], tag


def test_guard_checker_reports_planted_faults():
    harness_catches_planted_faults("cpu")
