"""GPU: what the ViT kernels read and write OUTSIDE their operands, how their persistent tile schedulers cover the grid,
and whether their bits depend on the GEMM tile width or on programmatic dependent launch (PDL).

test_kernel_bounds_gpu.py bounds every output element of fvs_linear, fvs_attention / fvs_attention80 and fvs_layernorm
/ fvs_add_layernorm, but its operands are exactly the tensors the kernel should touch, filled with finite values: a read
of A's pitch padding past K meets W's zero-filled tail (finite * 0 = 0), a store past M or into the pitch lands outside
anything it checks, and an element the kernel never writes keeps the randn it was filled with.  Here every operand lives
in a guard-banded buffer (tests/vit_kernel_edges.py): inputs are surrounded by quiet NaN (rows past M, N, aux_period or
the last frame, and the row pitch), outputs are filled with a marked NaN before the call.  After each call every guard
must hold its sentinel bit for bit, every output element must be finite (so written), and the element-wise bound of
test_kernel_bounds_gpu.py must hold.

The tile-scheduler sweep derives M (frames) from the SM count so that the last wave of tiles is empty, as small as it can
be, or one short of full, with 1, 2 and >= 20 tiles per CTA, and K so that the K loop is shorter than, as long as and
longer than the TMA ring.  The GEMM sweep runs in two child processes, one per tile width (FVS_GEMM_BN is read once per
process); both must produce the same bits as each other and as this process, whose outputs meet the bound.  The PDL
chain runs one ViT block's seven launches back to back without a synchronize, with PDL and (in a child) without it, and
one synchronized launch at a time: all bit-identical.  Each group prints its largest err / bound, and the module its wall
time."""
import hashlib
import os
import subprocess
import sys
import time

import numpy as np
import pytest
import torch

from tests import vit_kernel_edges as VE
from tests.test_kernel_bounds_gpu import DTYPES, EPI, attention_bound, check, layernorm_bound, linear_bound, linear_raw, \
    ln_input
from tests.test_vit_kernel_edges_host import harness_catches_planted_faults

pytestmark = pytest.mark.gpu

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
G_ROWS = 128     # guard rows past M, past aux_period, past the last frame or LayerNorm row: one whole tile of rows
G_COLS = 64      # pitch guard: one whole 64-column K block or output chunk
G_W = 256        # W rows past N and bias elements past N: one whole 256-wide tile
CHILD_TIMEOUT = 1200
WORST = {}


def note(group, worst):
    WORST[group] = max(WORST.get(group, 0.0), worst)


@pytest.fixture(scope="module")
def L():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    from flash_vstream_b200 import _lib
    _lib.load(build_if_missing=False)
    t0 = time.perf_counter()
    yield _lib
    print("\n[vit kernel edges] largest err/bound per group: " + ", ".join(f"{g} {w:.3f}" for g, w in WORST.items()))
    print(f"[vit kernel edges] wall time {time.perf_counter() - t0:.1f} s")


def sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def digest(buf):
    return hashlib.sha256(buf.contiguous().cpu().view(torch.uint8).numpy().tobytes()).hexdigest()


def child(mode, out_path, **env):
    """runs this module as a child process (`mode` below) with extra environment variables; it writes `out_path`"""
    r = subprocess.run([sys.executable, "-m", "tests.test_vit_kernel_edges_gpu", mode, str(out_path)], cwd=ROOT,
                       env=dict(os.environ, **env), capture_output=True, text=True, timeout=CHILD_TIMEOUT)
    assert r.returncode == 0, f"child {mode} {env}: exit {r.returncode}\n{r.stdout[-3000:]}\n{r.stderr[-5000:]}"
    return torch.load(out_path)


# ------------------------------------------------------------------------------------------------------------ GEMM
def epi_code(L, epi):
    return {"bias": L.EPI_BIAS, "quickgelu": L.EPI_BIAS_QUICKGELU, "gelu": L.EPI_BIAS_GELU,
            "residual": L.EPI_BIAS_RESIDUAL, "residual_alias": L.EPI_BIAS_RESIDUAL, "rowtable": L.EPI_ROWTABLE,
            "residual_f32": L.EPI_BIAS_RESIDUAL_F32, "residual_f32_alias": L.EPI_BIAS_RESIDUAL_F32}[epi]


def gemm_operands(epi, dtype, M, N, K, seed):
    """{name: (guarded buffer, view)} for one fvs_linear call and its aux_period.  A and out (and a residual, which
    shares out's pitch) have G_COLS pitch columns and G_ROWS rows past M; W has G_W rows past N, bias G_W elements past
    N, the row table G_ROWS rows past aux_period.  An in-place (_alias) out starts as the residual; any other out starts
    as the sentinel.  The payloads are a function of `seed` alone (the same in every process)."""
    g = torch.Generator(device="cuda").manual_seed(seed)

    def rnd(*shape, scale=1.0, dt=dtype):
        return (torch.randn(*shape, generator=g, device="cuda") * scale).to(dt)

    odt = torch.float32 if epi.startswith("residual_f32") else dtype
    t = {"A": VE.guarded(rnd(M, K, scale=1.5), G_ROWS, G_COLS, VE.IN_BITS[dtype]),
         "W": VE.guarded(rnd(N, K, scale=K ** -0.5), G_W, 0, VE.IN_BITS[dtype])}
    if epi != "rowtable":
        t["bias"] = VE.guarded(rnd(1, N, scale=0.5), 0, G_W, VE.IN_BITS[dtype])
    period = 0
    if epi == "rowtable":
        period = 577 if M > 577 else M // 2 + 1
        t["aux"] = VE.guarded(rnd(period, N), G_ROWS, 0, VE.IN_BITS[dtype])
    elif epi in ("residual", "residual_f32"):
        t["aux"] = VE.guarded(rnd(M, N, dt=odt), G_ROWS, G_COLS, VE.IN_BITS[odt])
    if epi.endswith("_alias"):
        t["out"] = VE.guarded(rnd(M, N, dt=odt), G_ROWS, G_COLS, VE.OUT_BITS[odt])
    else:
        t["out"] = VE.blank(M, N, odt, G_ROWS, G_COLS, VE.OUT_BITS[odt], "cuda")
    return t, period


def aux_before(epi, t):
    """the epilogue's aux input as it is before the call (fp64), or None"""
    if epi.endswith("_alias"):
        return t["out"][1].double()
    return t["aux"][1].double() if "aux" in t else None


def gemm_run(L, epi, t, period):
    out = t["out"][1]
    aux = out if epi.endswith("_alias") else (t["aux"][1] if "aux" in t else None)
    linear_raw(L, t["A"][1], t["W"][1], t["bias"][1] if "bias" in t else None, aux, out, epi_code(L, epi), period)
    torch.cuda.synchronize()


def gemm_problems(name, t):
    probs = []
    for key, (buf, view) in t.items():
        bits = (VE.OUT_BITS if key == "out" else VE.IN_BITS)[buf.dtype]
        probs += VE.report(f"{name} {key}", buf, *view.shape, bits, written=key == "out")
    return probs


def gemm_bound_check(name, epi, t, aux_in):
    y, bound, rounding = linear_bound(t["A"][1], t["W"][1], t["bias"][1] if "bias" in t else None, epi, aux_in,
                                      t["out"][1])
    return check(name, t["out"][1], y, bound, rounding)


# K % 64 in {0, 8, 56, 24}; M below, at and past one 128-row block; N one to five 256-wide tiles, partial ones included
GUARD_SHAPES = [(1, 128, 120), (65, 64, 72), (129, 320, 56), (300, 1280, 64), (700, 640, 1176), (257, 1280, 8)]


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("epi", EPI)
def test_linear_guards(L, epi, dt):
    """NaN in A's pitch past K and rows past M, W's rows past N, bias past N, the residual's pitch and rows, the row
    table's rows past aux_period; a marked NaN in out's pitch and rows past M and (unless in place) in out itself"""
    dtype = DTYPES[dt]
    for i, (M, N, K) in enumerate(GUARD_SHAPES):
        t, period = gemm_operands(epi, dtype, M, N, K, 100 * EPI.index(epi) + 10 * i + len(dt))
        aux_in = aux_before(epi, t)
        gemm_run(L, epi, t, period)
        name = f"linear guards {epi} {dt} M{M} N{N} K{K}"
        probs = gemm_problems(name, t)
        assert not probs, "\n".join(probs)
        note("linear guards", gemm_bound_check(name, epi, t, aux_in))


def sweep_cases(n_sms):
    """[(epi, dt, M, N, K, label)]: the shapes of VE.gemm_sweep_shapes at both widths, the epilogues and dtypes in turn"""
    cases = []
    for bn, ns in VE.SWEEP_N.items():
        for n in ns:
            for M, N, K, label in VE.gemm_sweep_shapes(n_sms, n, bn):
                i = len(cases)
                cases.append((EPI[i % len(EPI)], ("f16", "bf16")[(i // len(EPI)) % 2], M, N, K, f"{label} at width {bn}"))
    return cases


def run_sweep(L, each):
    """runs every sweep case in this process; each(i, case, operands, aux_in) sees the result"""
    for i, case in enumerate(sweep_cases(sms())):
        epi, dt, M, N, K, _ = case
        t, period = gemm_operands(epi, DTYPES[dt], M, N, K, 1000 + i)
        aux_in = aux_before(epi, t)
        gemm_run(L, epi, t, period)
        each(i, case, t, aux_in)
        del t, aux_in


def test_linear_sweep_both_tile_widths_bitwise(L, tmp_path):
    """every sweep case at width 128 and at width 256 (one child process each): the guards hold in both, the outputs
    (guards included) are bit-identical to each other and to this process's, and this process's meet the bound"""
    runs = {bn: child("sweep", tmp_path / f"bn{bn}.pt", FVS_GEMM_BN=str(bn)) for bn in (128, 256)}
    cases = sweep_cases(sms())
    for bn, res in runs.items():
        assert len(res) == len(cases), bn
        bad = [p for r in res for p in r["problems"]]
        assert not bad, f"width {bn}:\n" + "\n".join(bad[:20])

    def each(i, case, t, aux_in):
        epi, dt, M, N, K, label = case
        name = f"linear sweep {epi} {dt} M{M} N{N} K{K} ({label})"
        probs = gemm_problems(name, t)
        assert not probs, "\n".join(probs)
        h = digest(t["out"][0])
        assert runs[128][i]["digest"] == runs[256][i]["digest"], f"{name}: widths 128 and 256 give different bits"
        assert h == runs[128][i]["digest"], f"{name}: this process and the forced widths give different bits"
        note("linear sweep", gemm_bound_check(name, epi, t, aux_in))
    run_sweep(L, each)
    print(f"\n[linear sweep] {len(cases)} cases on {sms()} SMs, bit-identical at widths 128 and 256")


def _child_sweep(L, out_path):
    res = []

    def each(i, case, t, aux_in):
        res.append({"digest": digest(t["out"][0]), "problems": gemm_problems(f"case {i} {case}", t)})
    run_sweep(L, each)
    torch.save(res, out_path)


# ------------------------------------------------------------------------------------------------------- attention
ATTN_TOKENS = [65, 129, 577, 36, 100]        # none a multiple of the 64-key tile but 64 * 9 + 1; 36 and 100 < 128
SWEEP_HEADS = 5                              # 5 * ceil(tokens / 128) tiles per frame: coprime to 132 and 114 but for 129


def attention_case(L, hd, dtype, frames, tokens, heads, seed, name):
    """fvs_attention / fvs_attention80 through the C entry point on a qkv with G_ROWS NaN rows past the last frame and a
    ctx filled with the sentinel and G_ROWS guard rows; returns the largest err / bound"""
    from flash_vstream_b200 import ops
    lib = L.load()
    g = torch.Generator(device="cuda").manual_seed(seed)
    rows = frames * tokens
    nat = torch.randn(rows, 3 * heads * hd, generator=g, device="cuda").to(dtype)
    qkv_buf, qkv = VE.guarded(nat if hd == 64 else ops.split_heads_80(nat, heads, 3), G_ROWS, 0, VE.IN_BITS[dtype])
    ctx_buf, ctx = VE.blank(rows, heads * hd, dtype, G_ROWS, 0, VE.OUT_BITS[dtype], "cuda")
    fn = lib.fvs_attention if hd == 64 else lib.fvs_attention80
    scale = 0.125 if hd == 64 else float(np.float32(80 ** -0.5))
    L.check(fn(L.ptr(qkv), L.ptr(ctx), frames, tokens, heads, scale, L.dtype_code(dtype), L.cur_stream()), name)
    torch.cuda.synchronize()
    probs = VE.report(f"{name} qkv", qkv_buf, *qkv.shape, VE.IN_BITS[dtype], written=False) + \
        VE.report(f"{name} ctx", ctx_buf, *ctx.shape, VE.OUT_BITS[dtype])
    assert not probs, "\n".join(probs)
    out = ctx if hd == 64 else ops.merge_heads_80(ctx, heads)
    ref, bound, rounding = attention_bound(nat, frames, tokens, heads, hd, scale)
    return check(name, out.view(frames, tokens, heads, hd), ref, bound, rounding)


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("hd", [64, 80])
def test_attention_guards(L, hd, dt):
    for tokens in ATTN_TOKENS:
        note("attention guards", attention_case(L, hd, DTYPES[dt], 3, tokens, 16, tokens * 7 + hd + len(dt),
                                                f"attention guards hd{hd} {dt} 3x{tokens} h16"))


@pytest.mark.parametrize("hd", [64, 80])
@pytest.mark.parametrize("tokens", ATTN_TOKENS)
def test_attention_scheduler_sweep(L, tokens, hd):
    """frames such that the (query block, head, frame) tiles fill one wave, two, or leave a last wave of 0, g or SMs - g
    tiles (VE.attention_sweep_frames), f16 and bf16 in turn, with the guards of test_attention_guards"""
    for i, (frames, label) in enumerate(VE.attention_sweep_frames(sms(), tokens, SWEEP_HEADS)):
        dt = ("f16", "bf16")[i % 2]
        note("attention sweep", attention_case(L, hd, DTYPES[dt], frames, tokens, SWEEP_HEADS, 7 * tokens + i + hd,
                                               f"attention sweep hd{hd} {dt} {frames}x{tokens} h{SWEEP_HEADS} ({label})"))


# ------------------------------------------------------------------------------------------------------- LayerNorm
LN_DIMS = [256, 1280, 2048]
LN_ROWS = [1, 7, 9, 263]                     # one warp per row, 8 rows per block: a partial last block, and full ones


def ln_params(dim, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    gamma = VE.guarded((1 + 0.1 * torch.randn(1, dim, generator=g)).to(dtype).cuda(), 0, 256, VE.IN_BITS[dtype])
    beta = VE.guarded((0.05 * torch.randn(1, dim, generator=g)).to(dtype).cuda(), 0, 256, VE.IN_BITS[dtype])
    return gamma, beta


@pytest.mark.parametrize("ykind", ["y16", "y32"])
@pytest.mark.parametrize("xkind", ["x16", "x32"])
@pytest.mark.parametrize("dt", list(DTYPES))
def test_layernorm_guards(L, dt, xkind, ykind):
    """NaN rows past the last row of x, NaN past gamma and beta; y filled with the sentinel, with guard rows"""
    dtype = DTYPES[dt]
    xdt = dtype if xkind == "x16" else torch.float32
    ydt = dtype if ykind == "y16" else torch.float32
    lib = L.load()
    for dim in LN_DIMS:
        gamma, beta = ln_params(dim, dtype, dim)
        for rows in LN_ROWS:
            x_buf, x = VE.guarded(ln_input(rows, dim, dim + rows).to(xdt).cuda(), G_ROWS, 0, VE.IN_BITS[xdt])
            y_buf, y = VE.blank(rows, dim, ydt, G_ROWS, 0, VE.OUT_BITS[ydt], "cuda")
            L.check(lib.fvs_layernorm(L.ptr(x), L.ptr(gamma[1]), L.ptr(beta[1]), L.ptr(y), rows, dim, 1e-5,
                                      L.dtype_code(dtype), L.dtype_code(xdt), L.dtype_code(ydt), L.cur_stream()),
                    "fvs_layernorm")
            torch.cuda.synchronize()
            name = f"layernorm guards {dim} {dt} {xkind} {ykind} rows {rows}"
            probs = VE.report(f"{name} x", x_buf, rows, dim, VE.IN_BITS[xdt], written=False) + \
                VE.report(f"{name} y", y_buf, rows, dim, VE.OUT_BITS[ydt])
            for key, (buf, view) in (("gamma", gamma), ("beta", beta)):
                probs += VE.report(f"{name} {key}", buf, 1, dim, VE.IN_BITS[dtype], written=False)
            assert not probs, "\n".join(probs)
            ref, bound, rounding = layernorm_bound(x, gamma[1][0], beta[1][0], float(np.float32(1e-5)), y)
            note("layernorm guards", check(name, y, ref, bound, rounding))


@pytest.mark.parametrize("dt", list(DTYPES))
def test_add_layernorm_guards(L, dt):
    """x (fp32) += delta in place: the rows of x past the last one (NaN) stay untouched bit for bit, as do delta's;
    y is filled with the sentinel and has guard rows"""
    dtype = DTYPES[dt]
    lib = L.load()
    for dim in LN_DIMS:
        gamma, beta = ln_params(dim, dtype, dim + 1)
        g = torch.Generator().manual_seed(dim)
        for rows in LN_ROWS:
            x_buf, x = VE.guarded(ln_input(rows, dim, 3 * dim + rows).cuda(), G_ROWS, 0, VE.IN_BITS[torch.float32])
            d_buf, delta = VE.guarded(torch.randn(rows, dim, generator=g).to(dtype).cuda(), G_ROWS, 0,
                                      VE.IN_BITS[dtype])
            y_buf, y = VE.blank(rows, dim, dtype, G_ROWS, 0, VE.OUT_BITS[dtype], "cuda")
            want_x = x + delta.float()
            L.check(lib.fvs_add_layernorm(L.ptr(x), L.ptr(delta), L.ptr(gamma[1]), L.ptr(beta[1]), L.ptr(y), rows, dim,
                                          1e-6, L.dtype_code(dtype), L.cur_stream()), "fvs_add_layernorm")
            torch.cuda.synchronize()
            name = f"add_layernorm guards {dim} {dt} rows {rows}"
            probs = VE.report(f"{name} x", x_buf, rows, dim, VE.IN_BITS[torch.float32]) + \
                VE.report(f"{name} delta", d_buf, rows, dim, VE.IN_BITS[dtype], written=False) + \
                VE.report(f"{name} y", y_buf, rows, dim, VE.OUT_BITS[dtype])
            assert not probs, "\n".join(probs)
            assert torch.equal(x.view(torch.int32), want_x.view(torch.int32)), name
            ref, bound, rounding = layernorm_bound(x, gamma[1][0], beta[1][0], float(np.float32(1e-6)), y)
            note("add_layernorm guards", check(name, y, ref, bound, rounding))


# ------------------------------------------------------------------------------------------------------- PDL chain
# One Qwen2-VL vision block's launches: LN1, QKV GEMM, attention80, out-proj reduce-add into x, add-LayerNorm (x += ctx,
# y = LN2(x)), fc1 quick-GELU, fc2 reduce-add into x.  Each launch reads what the one before it wrote.
CE, CHEADS, CMLP, CFRAMES, CTOKENS = 1280, 16, 5120, 2, 577
CHAIN_OUT = ("h", "qkv", "ctx", "y", "act", "x")


def chain_tensors(dtype, seed):
    g = torch.Generator(device="cuda").manual_seed(seed)
    rows = CFRAMES * CTOKENS

    def rnd(*shape, scale=1.0, dt=dtype):
        return (torch.randn(*shape, generator=g, device="cuda") * scale).to(dt)

    p = {"x": rnd(rows, CE, dt=torch.float32), "g1": 1 + rnd(CE, scale=0.1), "b1": rnd(CE, scale=0.05),
         "wqkv": rnd(3 * CE, CE, scale=CE ** -0.5), "bqkv": rnd(3 * CE, scale=0.5), "wo": rnd(CE, CE, scale=CE ** -0.5),
         "bo": rnd(CE, scale=0.5), "g2": 1 + rnd(CE, scale=0.1), "b2": rnd(CE, scale=0.05),
         "w1": rnd(CMLP, CE, scale=CE ** -0.5), "bf1": rnd(CMLP, scale=0.5), "w2": rnd(CE, CMLP, scale=CMLP ** -0.5),
         "bf2": rnd(CE, scale=0.5)}
    for key, cols in (("h", CE), ("qkv", 3 * CE), ("ctx", CE), ("y", CE), ("act", CMLP)):
        p[key] = VE.blank(rows, cols, dtype, 0, 0, VE.OUT_BITS[dtype], "cuda")[1]
    return p


def run_chain(L, p, sync):
    """the seven launches on the current stream; sync: a synchronize after each, else queued behind a GPU spin so that
    each launch is issued while its predecessor is still running.  Returns the outputs on the host."""
    lib, s = L.load(), L.cur_stream()
    dc = L.dtype_code(p["h"].dtype)
    rows = CFRAMES * CTOKENS
    steps = [
        lambda: L.check(lib.fvs_layernorm(L.ptr(p["x"]), L.ptr(p["g1"]), L.ptr(p["b1"]), L.ptr(p["h"]), rows, CE, 1e-6,
                                          dc, L.F32, dc, s), "fvs_layernorm"),
        lambda: linear_raw(L, p["h"], p["wqkv"], p["bqkv"], None, p["qkv"], L.EPI_BIAS),
        lambda: L.check(lib.fvs_attention80(L.ptr(p["qkv"]), L.ptr(p["ctx"]), CFRAMES, CTOKENS, CHEADS,
                                            float(np.float32(80 ** -0.5)), dc, s), "fvs_attention80"),
        lambda: linear_raw(L, p["ctx"], p["wo"], p["bo"], p["x"], p["x"], L.EPI_BIAS_RESIDUAL_F32),
        lambda: L.check(lib.fvs_add_layernorm(L.ptr(p["x"]), L.ptr(p["ctx"]), L.ptr(p["g2"]), L.ptr(p["b2"]),
                                              L.ptr(p["y"]), rows, CE, 1e-6, dc, s), "fvs_add_layernorm"),
        lambda: linear_raw(L, p["y"], p["w1"], p["bf1"], None, p["act"], L.EPI_BIAS_QUICKGELU),
        lambda: linear_raw(L, p["act"], p["w2"], p["bf2"], p["x"], p["x"], L.EPI_BIAS_RESIDUAL_F32),
    ]
    torch.cuda.synchronize()
    if not sync:
        torch.cuda._sleep(50_000_000)
    for step in steps:
        step()
        if sync:
            torch.cuda.synchronize()
    torch.cuda.synchronize()
    return {k: p[k].cpu() for k in CHAIN_OUT}


def chain_all(L, sync):
    return {dt: run_chain(L, chain_tensors(dtype, 77 + len(dt)), sync) for dt, dtype in DTYPES.items()}


def test_pdl_chain_bitwise(L, tmp_path):
    """the chain with PDL, without it (FVS_PDL=0, a child process) and one synchronized launch at a time: same bits"""
    assert os.environ.get("FVS_PDL", "1")[:1] != "0", "this process must run with PDL on"
    pdl = chain_all(L, sync=False)
    synced = chain_all(L, sync=True)
    no_pdl = child("chain", tmp_path / "chain.pt", FVS_PDL="0")
    for dt in DTYPES:
        for key in CHAIN_OUT:
            a = pdl[dt][key]
            ib = torch.int32 if a.dtype == torch.float32 else torch.int16
            assert torch.isfinite(a).all(), f"{dt} {key}: the chain left non-finite elements"
            assert torch.equal(a.view(ib), synced[dt][key].view(ib)), f"{dt} {key}: PDL chain != synchronized launches"
            assert torch.equal(a.view(ib), no_pdl[dt][key].view(ib)), f"{dt} {key}: PDL chain != FVS_PDL=0 chain"
    print("\n[pdl chain] LN, QKV, attention80, out-proj, add-LN, fc1, fc2: bit-identical with PDL, without, synchronized")


# ------------------------------------------------------------------------------------------------ harness self-test
def test_guard_checker_reports_planted_faults(L):
    """on CUDA tensors the test builds itself (no kernel): a flipped guard bit and a left-over sentinel are reported"""
    harness_catches_planted_faults("cuda")


if __name__ == "__main__":      # child processes: python -m tests.test_vit_kernel_edges_gpu {sweep|chain} OUT.pt
    torch.set_grad_enabled(False)
    from flash_vstream_b200 import _lib
    _lib.load(build_if_missing=False)
    mode, out = sys.argv[1], sys.argv[2]
    if mode == "sweep":
        _child_sweep(_lib, out)
    elif mode == "chain":
        torch.save(chain_all(_lib, sync=False), out)
    else:
        raise SystemExit(f"unknown mode {mode}")
