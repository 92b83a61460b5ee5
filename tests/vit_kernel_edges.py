"""Shape derivations and guard-banded buffers for tests/test_vit_kernel_edges_gpu.py (pure: no CUDA needed, so the
host tests can check both).

Scheduler sweep.  fvs_linear runs min(SMs, tiles) persistent CTAs over tiles = ceil(M / 128) * ceil(N / BN), tile t on
CTA t mod grid; fvs_attention likewise over tiles = ceil(tokens / 128) * heads * frames.  The shapes below set the tile
count T so that the last wave (T mod grid) is empty, as small as it can be, or one short of full, and so that a CTA runs
1 tile, 2 tiles, or 20 and more.  Only M (frames) moves, so T is a multiple of the tiles per M block (per frame), and T
mod SMs is a multiple of g = gcd(that count, SMs): the smallest non-empty last wave is g tiles and the fullest is SMs - g
(exactly 1 and SMs - 1 when g = 1: N = 1280 at width 256, N = 1664 at width 128).

Guards.  `guarded` puts a payload in the top-left corner of a larger buffer filled with a sentinel bit pattern: the
extra rows stand for rows past M (past the last frame, past aux_period), the extra columns for a row pitch.  Inputs get
a quiet NaN, so a stray read turns an output into NaN (NaN * 0 is NaN where a zero-filled W tail would hide finite
padding); outputs get a distinctive NaN, so a stray write changes a guard and an element the kernel never wrote is still
NaN.  `report` compares the guards as integers, bit for bit."""
import math

import torch

BM = 128                                   # GEMM tile rows; attention query rows per tile
K_STAGES = {128: 6, 256: 4}                # gemm_sm90.cu Cfg<kBN>::kStages
# N per tile width: 1280 and 5120 at both; at width 128 both have an even number of column tiles, so 1664 (13 tiles)
# gives last waves of exactly 1 and SMs - 1 there
SWEEP_N = {128: (1280, 1664, 5120), 256: (1280, 5120)}
MANY = 20                                  # "many tiles per CTA"

IN_BITS = {torch.float16: 0x7E00, torch.bfloat16: 0x7FC0, torch.float32: 0x7FC00000}        # quiet NaN
OUT_BITS = {torch.float16: 0x7FA5, torch.bfloat16: 0x7FA5, torch.float32: 0x7FC0A5A5}      # NaN with a marked payload
_INT = {2: torch.int16, 4: torch.int32}


def _tiles_with_residue(sms, per_block, r, at_least):
    """the smallest multiple T of per_block with T >= at_least and T mod sms == r"""
    t = -(-at_least // per_block) * per_block
    while t % sms != r:
        t += per_block
    return t


def wave_targets(sms, per_block):
    """[(label, tiles)]: a single wave (every CTA one tile), two tiles per CTA, then last waves of 0, g and sms - g tiles
    after at least one full wave, then the same after at least MANY full waves"""
    g = math.gcd(per_block, sms)
    out = [("1 tile/CTA", per_block * (sms // per_block)), ("2 tiles/CTA", per_block * (2 * sms // per_block))]
    for waves in (1, MANY):
        for r in (0, g, sms - g):
            out.append((f"r={r} after >={waves} waves", _tiles_with_residue(sms, per_block, r, waves * sms + 1)))
    return out


def sweep_ks(bn):
    """K with num_kb = 1 (K % 64 = 8 and 0), 2, kStages and 19 (above): below, at and above the ring depth"""
    return (8, 64, 72, 64 * K_STAGES[bn], 1176)


def gemm_sweep_shapes(sms, n, bn):
    """[(M, N, K, label)] for fvs_linear at tile width bn on `sms` SMs.  The single- and two-wave shapes cross every K of
    sweep_ks; the shapes with a partial last wave take one K each, the large ones only K <= 64 * kStages (num_kb <=
    kStages: the producer laps the consumers across tile boundaries).  M alternates between full last row blocks and
    last blocks of 1 and 64 rows."""
    num_n = -(-n // bn)
    ks = sweep_ks(bn)
    shapes = []
    for i, (label, tiles) in enumerate(wave_targets(sms, num_n)):
        num_m = tiles // num_n
        tail = (0, 127, 64)[i % 3] if num_m > 1 else 0
        m = num_m * BM - tail
        if i < 2:
            shapes += [(m, n, k, label) for k in ks]
        elif i < 5:
            shapes.append((m, n, (ks[2], ks[3], ks[4])[i - 2], label))
        else:
            shapes.append((m, n, (ks[0], ks[2], ks[3])[i - 5], label))
    return shapes


def gemm_schedule(sms, m, n, k, bn):
    """(tiles, grid, last wave, most tiles on one CTA, num_kb) of fvs_linear at tile width bn"""
    tiles = -(-m // BM) * -(-n // bn)
    grid = min(sms, tiles)
    return tiles, grid, tiles % grid, -(-tiles // grid), -(-k // 64)


def attention_sweep_frames(sms, tokens, heads):
    """[(frames, label)] for fvs_attention at `tokens` and `heads`: the wave targets of wave_targets, without the
    >= MANY-wave ones (the fp64 reference loops over frames and heads)"""
    per_frame = -(-tokens // BM) * heads
    return [(t // per_frame, label) for label, t in wave_targets(sms, per_frame)[:5]]


def guarded(payload, g_rows, g_cols, bits):
    """(buffer, view): a [rows + g_rows, cols + g_cols] buffer of `bits` with `payload` in its top-left [rows, cols]"""
    rows, cols = payload.shape
    buf = torch.empty(rows + g_rows, cols + g_cols, dtype=payload.dtype, device=payload.device)
    buf.view(_INT[buf.element_size()]).fill_(bits)
    view = buf[:rows, :cols]
    view.copy_(payload)
    return buf, view


def blank(rows, cols, dtype, g_rows, g_cols, bits, device):
    """(buffer, view) like `guarded`, the view holding the sentinel as well (an output no kernel has written yet)"""
    buf = torch.empty(rows + g_rows, cols + g_cols, dtype=dtype, device=device)
    buf.view(_INT[buf.element_size()]).fill_(bits)
    return buf, buf[:rows, :cols]


def report(name, buf, rows, cols, bits, written=True):
    """the problems of a guarded buffer: guard elements whose bits are no longer `bits`, and (written=True) elements of
    the [rows, cols] view that are not finite, of which how many still hold the sentinel (never written)"""
    ib = buf.view(_INT[buf.element_size()])
    probs = []
    bad_rows = int((ib[rows:] != bits).sum())
    bad_pitch = int((ib[:rows, cols:] != bits).sum())
    if bad_rows or bad_pitch:
        where = (ib != bits)
        where[:rows, :cols] = False
        r, c = (int(v) for v in where.nonzero()[0])
        probs.append(f"{name}: {bad_rows} guard elements past row {rows} and {bad_pitch} in the pitch past column {cols} "
                     f"changed (first at [{r}, {c}])")
    if written:
        view = buf[:rows, :cols]
        nf = int((~torch.isfinite(view)).sum())
        if nf:
            left = int((ib[:rows, :cols] == bits).sum())
            probs.append(f"{name}: {nf} output elements not finite, {left} of them still the sentinel (never written)")
    return probs
