"""GPU: element-wise error bounds for the ViT kernels (fvs_attention / fvs_attention80, fvs_linear with every epilogue,
fvs_layernorm / fvs_add_layernorm).  Every reference is evaluated in float64 from the kernel's own 16-bit inputs, every
bound is derived from the kernel's arithmetic (the rounding steps it performs, in its order), and EVERY output element
must lie within its bound.  A relative Frobenius norm over a whole output cannot see a wrong row edge, a wrong last
column chunk or the negative tail of an activation; an element-wise bound does.  Each case prints its largest
err / bound (the achieved margin, DESIGN.md §1)."""
import math

import numpy as np
import pytest
import torch

from tests.test_attention_variants_gpu import run as attn_run

pytestmark = pytest.mark.gpu

U32 = 2.0 ** -24                                         # fp32 unit roundoff (round to nearest)
U16 = {torch.float16: 2.0 ** -11, torch.bfloat16: 2.0 ** -8}
DTYPES = {"f16": torch.float16, "bf16": torch.bfloat16}


@pytest.fixture(scope="module")
def L():
    assert torch.cuda.is_available(), "gpu-marked tests need a CUDA device"
    from flash_vstream_b200 import _lib
    _lib.load(build_if_missing=False)
    return _lib


def half_ulp(out):
    """half an ulp of each rounded 16-bit value: round-to-nearest put the unrounded value within this of it"""
    fi = torch.finfo(out.dtype)
    a = out.double().abs()
    _, e = torch.frexp(a)                                 # |out| in [2^(e-1), 2^e)
    h = torch.ldexp(torch.full_like(a, fi.eps / 2), e - 1)
    sub = fi.tiny * fi.eps / 2                            # subnormal range (and 0): half the subnormal spacing
    return torch.where(a < fi.tiny, torch.full_like(a, sub), h)


def check(name, got, ref, bound, rounding=None):
    """asserts |got - ref| <= bound element-wise.  `rounding`: the part of the bound that is the final rounding to the
    output dtype; where it dominates, err/bound sits near 1 by construction, so the margin left over the arithmetic
    before that rounding, max((err - rounding)+ / (bound - rounding)), is printed as well."""
    err = (got.double() - ref).abs()
    ratio = err / bound
    worst = float(ratio.max())
    i = int(ratio.argmax())
    pre = "" if rounding is None else ", before the output rounding " \
        f"{float(((err - rounding).clamp(min=0) / (bound - rounding)).nan_to_num(nan=0.0, posinf=math.inf).max()):.3f}"
    print(f"\n[{name}] max err/bound {worst:.3f} (err {float(err.flatten()[i]):.3e}, bound {float(bound.flatten()[i]):.3e})"
          f"{pre}")
    assert torch.isfinite(got).all(), name
    assert worst <= 1.0, f"{name}: element {np.unravel_index(i, tuple(err.shape))} err/bound {worst:.3f}"
    return worst


# ------------------------------------------------------------------------------------------------------- attention
# The kernel computes O = sum_j P~_j v_j / sum_j P~_j with P~_j = exp2((s_j - m) * scale * log2e) rounded to the P dtype
# (the 16-bit A operand of P V) and the row sum taken over the same rounded P~ (attention_sm90.cu), both sums in fp32.
# Rounding P~_j = e_j (1 + d_j) with |e_j d_j| <= max(u_P e_j, s_P) moves O by sum_j e_j d_j (v_j - o) / sum_j e_j to
# first order; the denominator is >= 1 (the row maximum contributes e = 1), so per output element
#   |o - o_ref| <= sum_j max(u_P p_j, s_P) |v_j - o_ref| + u_out |o_ref| + 2^-20 max_j |v_j|
# with p the exact softmax, u_P the P dtype's unit roundoff, s_P = 2^-25 (half the fp16 subnormal spacing; 0 for bf16),
# u_out the output rounding and 2^-20 max|v| for the fp32 accumulation, ex2.approx and the rescales.
ATTN_TOKENS = [577, 864, 216, 960, 240, 4784, 1196, 1, 16, 17, 64, 65, 128, 129]
ATTN_CASES = [(n, 16) for n in ATTN_TOKENS] + [(577, 1), (864, 3), (129, 3), (65, 1)]


def attention_bound_check(name, nat, out, frames, tokens, heads, hd, scale):
    ref, bound, rounding = attention_bound(nat, frames, tokens, heads, hd, scale)
    return check(name, out.view(frames, tokens, heads, hd), ref, bound, rounding)


def attention_bound(nat, frames, tokens, heads, hd, scale):
    """fp64 reference, element-wise bound and its output-rounding part, each [frames, tokens, heads, hd], for the
    attention of the natural-layout qkv rows `nat` [frames * tokens, 3 * heads * hd]"""
    dt = nat.dtype
    u, s_p = U16[dt], (2.0 ** -25 if dt == torch.float16 else 0.0)
    q, k, v = nat.double().view(frames, tokens, 3, heads, hd).unbind(2)
    ref_all = torch.empty(frames, tokens, heads, hd, dtype=torch.float64, device=nat.device)
    bound_all, round_all = torch.empty_like(ref_all), torch.empty_like(ref_all)
    for f in range(frames):
        for h in range(heads):
            qh, kh, vh = q[f, :, h], k[f, :, h], v[f, :, h]
            p = torch.softmax(qh @ kh.T * scale, dim=-1)
            o = p @ vh
            w = (u * p).clamp(min=s_p)
            ch = max(1, (1 << 24) // (tokens * hd))
            b = torch.empty_like(o)
            for r0 in range(0, tokens, ch):
                r1 = min(tokens, r0 + ch)
                b[r0:r1] = (w[r0:r1, :, None] * (vh[None] - o[r0:r1, None, :]).abs()).sum(1)
            b += u * o.abs() + 2.0 ** -20 * vh.abs().amax(0)
            ref_all[f, :, h], bound_all[f, :, h], round_all[f, :, h] = o, b, u * o.abs()
    return ref_all, bound_all, round_all


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("hd", [64, 80])
@pytest.mark.parametrize("tokens,heads", ATTN_CASES)
def test_attention_elementwise_bound(L, tokens, heads, hd, dt):
    from flash_vstream_b200 import ops
    dtype = DTYPES[dt]
    frames = 1 if tokens > 2000 else 3
    g = torch.Generator().manual_seed(tokens * 31 + heads * 7 + hd)
    nat = torch.randn(frames * tokens, 3 * heads * hd, generator=g).to(dtype).cuda()
    out = attn_run(ops, nat, frames, tokens, heads, hd)
    scale = 0.125 if hd == 64 else float(np.float32(80 ** -0.5))      # the fp32 scale the kernel is handed
    attention_bound_check(f"attention hd{hd} {dt} {frames}x{tokens} h{heads}", nat, out, frames, tokens, heads, hd, scale)


@pytest.mark.parametrize("hd", [64, 80])
def test_attention_elementwise_bound_growing_keys(L, hd):
    """test_attention_large_scores_rescale_path's input: keys grow along the sequence, every KV tile rescales O and L"""
    from flash_vstream_b200 import ops
    frames, tokens, heads = 4, 577, 16
    g = torch.Generator().manual_seed(11)
    nat = torch.randn(frames * tokens, 3 * heads * hd, generator=g)
    ramp = torch.linspace(0.2, 3.0, tokens).repeat(frames)[:, None]
    nat[:, heads * hd:2 * heads * hd] *= ramp
    nat = nat.half().cuda()
    out = attn_run(ops, nat, frames, tokens, heads, hd)
    scale = 0.125 if hd == 64 else float(np.float32(80 ** -0.5))
    attention_bound_check(f"attention hd{hd} f16 growing keys", nat, out, frames, tokens, heads, hd, scale)


# ------------------------------------------------------------------------------------------------------------ GEMM
# acc = sum_k a_k w_k in fp32 on the tensor cores: the products of 16-bit values are exact, the K additions are bounded by
# gamma * sum_k |a_k w_k| with gamma = K * 2^-23 (2^-23 rather than 2^-24: the tensor cores' fp32 accumulation may
# truncate instead of rounding).  The epilogue then rounds in fp32 (acc + bias, the activation, + residual) and once more
# to the 16-bit output (half an ulp of the result).  An activation multiplies the error it is handed by its Lipschitz
# constant: 1.0998 for quick-GELU x*sigmoid(1.702 x) (= SiLU's), 1.1289 for the erf GELU.
EPS_TANH = 2.0 ** -10.987     # PTX ISA, tanh: tanh.approx.f32 has a maximum relative error of 2^-10.987 (|tanh| <= 1)
LIP_QUICKGELU, LIP_GELU = 1.0998, 1.1290
C_0851 = float(np.float32(0.851))
C_SQRT1_2 = float(np.float32(0.70710678118654752))
ERFF_ULP = 2                  # CUDA Math API: erff has a maximum error of 2 ulp

EPI = ["bias", "quickgelu", "gelu", "residual", "residual_alias", "rowtable", "residual_f32", "residual_f32_alias"]
BIG = [(2160, 1280, 1176), (2160, 3840, 1280), (2160, 1280, 1280), (2160, 5120, 1280), (2160, 1280, 5120)]
SMALL = [(m, n, k) for m in (1, 65, 129) for n in (64, 320) for k in (8, 56, 72)]


def switch_shapes():
    """M on both sides of linear_tile_n's 128/256 switch for N = 1280: 2 * tiles256 <= SMs -> 128-wide tiles"""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    m_blocks = sms // (2 * 5)                                  # 5 = ceil(1280 / 256)
    return [(m_blocks * 128, 1280, 72), (m_blocks * 128 + 1, 1280, 72)]


def linear_raw(L, A, W, bias, aux, out, epi_code, aux_period=0):
    """fvs_linear with the row pitches of A and out as they are (ops.linear would make a pitched A contiguous)"""
    M, K = A.shape
    L.check(L.load().fvs_linear(L.ptr(A), L.ptr(W), L.ptr(bias), L.ptr(aux), L.ptr(out), M, W.shape[0], K, A.stride(0),
                                out.stride(0), epi_code, aux_period, L.dtype_code(A.dtype), L.cur_stream()), "fvs_linear")


def pitched(rows, cols, dtype, pad, g, scale=1.0):
    """a [rows, cols] column slice (starting at column `pad`) of a [rows, cols + 2 * pad] tensor, filled with randn"""
    wide = (torch.randn(rows, cols + 2 * pad, generator=g) * scale).to(dtype).cuda()
    return wide[:, pad:pad + cols]


def gemm_case(L, epi, dtype, M, N, K, pad, g, tails):
    """one fvs_linear call; returns its max err/bound"""
    code = {"bias": L.EPI_BIAS, "quickgelu": L.EPI_BIAS_QUICKGELU, "gelu": L.EPI_BIAS_GELU, "residual": L.EPI_BIAS_RESIDUAL,
            "residual_alias": L.EPI_BIAS_RESIDUAL, "rowtable": L.EPI_ROWTABLE, "residual_f32": L.EPI_BIAS_RESIDUAL_F32,
            "residual_f32_alias": L.EPI_BIAS_RESIDUAL_F32}[epi]
    f32_out = epi.startswith("residual_f32")
    odt = torch.float32 if f32_out else dtype
    A = pitched(M, K, dtype, pad, g, 1.5)
    W = (torch.randn(N, K, generator=g) * K ** -0.5).to(dtype).cuda()
    bias = (torch.randn(N, generator=g) * 0.5).to(dtype).cuda() if epi != "rowtable" else None
    out = pitched(M, N, odt, pad, g)
    aux, period = None, 0
    if epi in ("residual", "residual_f32"):
        aux = pitched(M, N, odt, pad, g)                         # aux shares out's row pitch
        if pad == 0:
            aux = aux.contiguous()
    elif epi.endswith("_alias"):
        aux = out                                                # in place: out = out + epilogue
    elif epi == "rowtable":
        period = 577 if M > 577 else M // 2 + 1                  # < M and not a divisor of M (M >= 3)
        aux = (torch.randn(period, N, generator=g)).to(dtype).cuda()
    aux_in = aux.double().clone() if aux is not None else None
    linear_raw(L, A, W, bias, aux, out, code, period)
    parts = {}
    y, bound, rounding = linear_bound(A, W, bias, epi, aux_in, out, parts)
    name = f"linear {epi} {str(dtype)[6:]} M{M} N{N} K{K}{' pitched' if pad else ''}"
    worst = check(name, out, y, bound, rounding)
    if epi == "quickgelu":
        x, tanh_term = parts["x"], parts["tanh_term"]
        tail = (x >= -6) & (x <= -1)
        if bool(tail.any()):
            err = (out.double() - y).abs()
            tails.append((float(err[tail].max()), float(tanh_term[tail].min()), float((err / bound)[tail].max())))
    return worst


def linear_bound(A, W, bias, epi, aux, out, parts=None):
    """fp64 reference, element-wise bound and its output-rounding part (None for an fp32 out) of fvs_linear with the
    epilogue `epi` (an EPI name) on the 16-bit A [M, K], W [N, K], bias [N] or None and the epilogue's aux input as it was
    before the call: the residual [M, N] (fp32 for the _f32 epilogues) or the row table [period, N].  `out` is what the
    kernel wrote; its dtype selects the output rounding.  `parts`, a dict, receives the fp64 pre-activation "x" and the
    quick-GELU "tanh_term"."""
    M, K = A.shape
    f32_out = out.dtype == torch.float32
    Ad, Wd = A.double(), W.double()
    acc = Ad @ Wd.T
    e = K * 2.0 ** -23 * (Ad.abs() @ Wd.abs().T)                  # accumulation
    if bias is not None:
        x = acc + bias.double()
        e = e + U32 * (x.abs() + e)                               # fl(acc + bias)
    else:
        x = acc                                                   # acc + 0.f: exact
    aux_in = aux.double() if aux is not None else None
    if parts is not None:
        parts["x"] = x
    if epi == "quickgelu":
        xa = x.abs() + e
        y = x * torch.sigmoid(1.702 * x)                          # = 0.5 x (1 + tanh(0.851 x))
        dz = abs(C_0851 - 0.851) * xa + U32 * C_0851 * xa         # fl(0.851f * x) vs 0.851 x
        tanh_term = 0.5 * xa * EPS_TANH
        e = LIP_QUICKGELU * e + tanh_term + 0.5 * xa * dz         # tanh.approx error; tanh is 1-Lipschitz
        e = e + U32 * (y.abs() + e)                               # fmaf(h, t, h)
        if parts is not None:
            parts["tanh_term"] = tanh_term
    elif epi == "gelu":
        xa = x.abs() + e
        y = 0.5 * x * (1 + torch.erf(x / math.sqrt(2)))
        dz = abs(C_SQRT1_2 - 0.5 ** 0.5) * xa + U32 * C_SQRT1_2 * xa
        d_erf = 2 / math.sqrt(math.pi) * dz + ERFF_ULP * 2.0 ** -23   # erf Lipschitz 2/sqrt(pi); erff's ulps (|erf| <= 1)
        e = LIP_GELU * e + 0.5 * xa * (d_erf + 2 * U32)           # fl(1 + erf), |1 + erf| <= 2: one rounding
        e = e + U32 * (y.abs() + e)                               # (0.5 x) * (1 + erf): one rounding
    elif epi == "rowtable":
        y = x + aux_in[torch.arange(M, device=x.device) % aux_in.shape[0]]
        e = e + U32 * (y.abs() + e)
    elif aux is not None:
        y = x + aux_in
        e = e + U32 * (y.abs() + e)                               # the residual add (fp32; the TMA reduce-add for _f32)
    else:
        y = x
    rounding = None if f32_out else half_ulp(out)
    bound = e if f32_out else e + rounding
    return y, bound, rounding


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("epi", EPI)
def test_linear_elementwise_bound(L, epi, dt):
    dtype = DTYPES[dt]
    g = torch.Generator().manual_seed(EPI.index(epi) * 10 + len(dt))
    shapes = BIG + SMALL + switch_shapes()
    worst, tails = 0.0, []
    for i, (M, N, K) in enumerate(shapes):
        pad = 64 if i % 2 else 0                                 # every other shape with a pitched A and out
        worst = max(worst, gemm_case(L, epi, dtype, M, N, K, pad, g, tails))
    print(f"\n[linear {epi} {dt}] largest err/bound over {len(shapes)} shapes: {worst:.3f}")
    if epi == "quickgelu":
        e_max, t_min, r_max = max(t[0] for t in tails), min(t[1] for t in tails), max(t[2] for t in tails)
        print(f"[linear quickgelu {dt}] negative tail x in [-6, -1]: largest err {e_max:.3e}; the tanh.approx term "
              f"0.5 |x| eps_tanh alone is >= {t_min:.3e} there; largest err/bound {r_max:.3f}")


# ------------------------------------------------------------------------------------------------------- LayerNorm
# One warp per row: each lane adds its 8 * kChunks values sequentially, then 5 butterfly levels; mean = sum * fp32(1/dim);
# the variance sums fma(d, d, q) of d = fl(x - mean) the same way; rstd = 1 / sqrtf(var + eps) (IEEE sqrt and division);
# y = fma(fl(d * rstd), gamma, beta), rounded once more to a 16-bit y.  So the gamma of both sums is that of
# 8 * kChunks + 5 additions, not of dim.
def layernorm_bound(v, gamma, beta, eps, out):
    """fp64 reference, element-wise bound and its output-rounding part (None for an fp32 y) for the kernel's LayerNorm
    of the fp32 values v [rows, dim]"""
    rows, dim = v.shape
    depth = 8 * (dim // 256) + 5
    gam = depth * U32 / (1 - depth * U32)
    v, g, b = v.double(), gamma.double(), beta.double()
    mu = v.mean(1, keepdim=True)
    e_s = gam * v.abs().sum(1, keepdim=True)
    e_m = e_s / dim + 3 * U32 * (mu.abs() + e_s / dim)             # fl(1/dim) and the product
    dev = (v - mu).abs()
    e_d = e_m + U32 * (dev + e_m)                                  # d = fl(x - mean)
    Q = (dev ** 2).sum(1, keepdim=True)
    e_Q = 2 * (dev * e_d).sum(1, keepdim=True) + (e_d ** 2).sum(1, keepdim=True)
    e_Q = e_Q + gam * (Q + e_Q)                                    # the fma chain and the butterfly
    e_var = e_Q / dim + 3 * U32 * (Q + e_Q) / dim
    V = Q / dim + eps
    e_V = e_var + U32 * (V + e_var)                                # fl(var + eps)
    rel_v = e_V / V
    rho = 0.5 * rel_v / (1 - rel_v) ** 1.5 + 2.01 * U32            # 1/sqrt of a perturbed input, sqrtf, the division
    rstd = V.rsqrt()
    e_t = e_d * rstd * (1 + rho) + dev * rstd * rho
    e_t = e_t + U32 * (dev + e_d) * rstd * (1 + rho)               # fl(d * rstd)
    ref = (v - mu) * rstd * g + b
    e = g.abs() * e_t
    e = e + U32 * (ref.abs() + e)                                  # the fma
    if out.dtype == torch.float32:
        return ref, e, None
    rounding = half_ulp(out)
    return ref, e + rounding, rounding


def ln_input(rows, dim, seed):
    """rows of three kinds: N(0, 1); a large common offset (mean ~ 1e3, std ~ 1); a few outlier dims (CLIP residual
    streams carry some hundreds-sized dims)"""
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(rows, dim, generator=g)
    kind = torch.arange(rows) % 3
    x[kind == 1] += 1e3
    cols = torch.tensor([3, dim // 3, dim // 2 + 1, dim - 2])
    out_rows = (kind == 2).nonzero().flatten()
    for r in out_rows.tolist():
        x[r, cols] = torch.tensor([120.0, -300.0, 45.0, 80.0]) * (1 + (r % 7) / 10)
    return x


LN_DIMS = [256 * c for c in range(1, 9)]
LN_ROWS = [1, 7, 8, 9, 2160]


@pytest.mark.parametrize("ykind", ["y16", "y32"])
@pytest.mark.parametrize("xkind", ["x16", "x32"])
@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("dim", LN_DIMS)
def test_layernorm_elementwise_bound(L, dim, dt, xkind, ykind):
    from flash_vstream_b200 import ops
    dtype = DTYPES[dt]
    g = torch.Generator().manual_seed(dim)
    gamma = (1 + 0.1 * torch.randn(dim, generator=g)).to(dtype).cuda()
    beta = (0.05 * torch.randn(dim, generator=g)).to(dtype).cuda()
    worst = 0.0
    for rows in LN_ROWS:
        x = ln_input(rows, dim, dim + rows).to(dtype if xkind == "x16" else torch.float32).cuda()
        y = ops.layernorm(x, gamma, beta, eps=1e-5, out_dtype=dtype if ykind == "y16" else torch.float32)
        ref, bound, rounding = layernorm_bound(x, gamma, beta, float(np.float32(1e-5)), y)
        worst = max(worst, check(f"layernorm {dim} {dt} {xkind} {ykind} rows {rows}", y, ref, bound, rounding))
    print(f"\n[layernorm {dim} {dt} {xkind} {ykind}] largest err/bound {worst:.3f}")


@pytest.mark.parametrize("dt", list(DTYPES))
@pytest.mark.parametrize("dim", LN_DIMS)
def test_add_layernorm_elementwise_bound(L, dim, dt):
    """x (fp32) += delta (16-bit) is written back bit for bit as x + float(delta); y meets the LayerNorm bound"""
    dtype = DTYPES[dt]
    g = torch.Generator().manual_seed(dim + 1)
    gamma = (1 + 0.1 * torch.randn(dim, generator=g)).to(dtype).cuda()
    beta = (0.05 * torch.randn(dim, generator=g)).to(dtype).cuda()
    lib = L.load()
    worst = 0.0
    for rows in LN_ROWS:
        x = ln_input(rows, dim, dim * 3 + rows).cuda()
        delta = torch.randn(rows, dim, generator=g).to(dtype).cuda()
        want_x = x + delta.float()
        y = torch.empty(rows, dim, dtype=dtype, device="cuda")
        L.check(lib.fvs_add_layernorm(L.ptr(x), L.ptr(delta), L.ptr(gamma), L.ptr(beta), L.ptr(y), rows, dim, 1e-6,
                                      L.dtype_code(dtype), L.cur_stream()), "fvs_add_layernorm")
        assert torch.equal(x.view(torch.int32), want_x.view(torch.int32)), (rows, dim)
        ref, bound, rounding = layernorm_bound(x, gamma, beta, float(np.float32(1e-6)), y)
        worst = max(worst, check(f"add_layernorm {dim} {dt} rows {rows}", y, ref, bound, rounding))
    print(f"\n[add_layernorm {dim} {dt}] largest err/bound {worst:.3f}")


@pytest.mark.parametrize("dim", [128, 300, 384, 2304, 4096])
def test_layernorm_refuses_unsupported_dims(L, dim):
    from flash_vstream_b200 import ops
    lib = L.load()
    x = torch.randn(4, dim, device="cuda").half()
    gamma, beta = torch.ones(dim, device="cuda").half(), torch.zeros(dim, device="cuda").half()
    y = torch.empty_like(x)
    torch.cuda.synchronize()
    n0 = lib.fvs_launch_count()
    with pytest.raises(ValueError, match="multiple of 256"):
        ops.layernorm(x, gamma, beta, out=y)
    xf = x.float()
    with pytest.raises(ValueError, match="multiple of 256"):
        L.check(lib.fvs_add_layernorm(L.ptr(xf), L.ptr(x), L.ptr(gamma), L.ptr(beta), L.ptr(y), 4, dim, 1e-6, L.F16,
                                      L.cur_stream()), "fvs_add_layernorm")
    assert lib.fvs_launch_count() == n0
