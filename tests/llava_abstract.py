"""The LLaVA abstract-memory update restated in the kernel's own order (csrc/mem_device.cuh: abs_proj_dot, abs_softmax_row,
abs_apply_elem), so the Turing rows of the fused step can be held bit for bit instead of to the few f16 ulp of
oracle.abstract_update (whose matmuls are fp64-accurate).

Every fmaf of those functions multiplies two f16-valued floats: the product is exact in fp32, so each chain is a chain of
plain fp32 additions in the kernel's lane order — reproduced here with numpy's IEEE fp32 arithmetic:
  * projection: lane l adds x[d] * w[d] for d = l, l + 32, ... from 0, the xor-butterfly (16, 8, 4, 2, 1), plus the bias,
    one f16 rounding;
  * score: sequential over h, f16, divided by sqrtf(H), f16; row max; e = expf(score - max); lane-strided sum over j
    (lane l owns j = l, l + 32), butterfly; w = f16(f16(e / sum) * ratio); decay = f16(lane-strided, butterflied sum of w);
  * output: f16(f16(m * f16(1 - decay)) + f16(sum_j w_j F[j, d] sequential in j)).
Only expf is not reproducible: the CUDA Math API bounds it by 2 ulp (exact at 0).  Here exp is correctly rounded to fp32,
and every e_j may lie within +-2 ulp of that value.  A weight w_j whose f16 roundings that interval leaves undetermined is
enumerated both (all) ways; rows are independent of each other (row i of the result depends on row i of the memory and on
the new rows only), so a row's candidates are the chain's values under every choice of its undetermined weights, carried
through every chunk of a step."""
from __future__ import annotations

import itertools

import numpy as np

F16, F32 = np.float16, np.float32
MAX_CANDIDATES = 256    # candidate rows per memory row and step; more would mean the interval is not doing its job


def _rh(x):
    return np.asarray(x, F32).astype(F16).astype(F32)


def _butterfly(acc):
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[..., lanes ^ o]
    return acc[..., 0]


def lane_strided_sum(terms):
    """terms [..., n] fp32 -> [...]: lane l adds terms l, l + 32, ... sequentially from 0, then the xor-butterfly"""
    terms = np.asarray(terms, F32)
    n = terms.shape[-1]
    acc = np.zeros(terms.shape[:-1] + (32,), F32)
    for base in range(0, n, 32):
        m = min(32, n - base)
        acc[..., :m] = acc[..., :m] + terms[..., base:base + m]
    return _butterfly(acc)


def proj(X, W, b):
    """abs_proj_dot for every (row of X, row of W): [R, D] x [H, D] -> [R, H] fp32 holding f16 values"""
    prods = X.astype(F32)[:, None, :] * W.astype(F32)[None, :, :]       # exact: products of two f16 values
    return _rh(lane_strided_sum(prods) + b.astype(F32)[None, :])


def scores(q, k):
    """[R, H] x [T2, H] -> f16(f16(q . k sequential in h) / sqrtf(H)) [R, T2]"""
    H = q.shape[1]
    acc = np.zeros((q.shape[0], k.shape[0]), F32)
    for h in range(H):
        acc = acc + q[:, h:h + 1] * k[None, :, h]
    return _rh(_rh(acc) / np.sqrt(F32(H)))


def exp_interval(x):
    """(nominal, lo, hi) fp32 of expf(x): exp correctly rounded to fp32, and +-2 ulp around it (exact at x == 0)"""
    x = np.asarray(x, F32)
    with np.errstate(over="ignore", under="ignore", invalid="ignore"):
        e = np.exp(x.astype(np.float64)).astype(F32)
    lo, hi = e.copy(), e.copy()
    for _ in range(2):
        lo = np.nextafter(lo, F32(-np.inf))
        hi = np.nextafter(hi, F32(np.inf))
    lo = np.maximum(lo, F32(0))
    exact = (x == 0) | np.isinf(x) | np.isnan(x)
    lo = np.where(exact, e, lo)
    hi = np.where(exact, e, hi)
    return e, lo, hi


def weights(q, k, ratio):
    """softmax * ratio of abs_softmax_row for rows q against k -> (nominal w, lo, hi) [R, T2] fp32 (f16 values)"""
    s = scores(q, k)
    mx = np.fmax.reduce(s, axis=1, initial=-np.inf)                     # fmaxf: NaN never wins
    with np.errstate(invalid="ignore"):
        e, lo, hi = exp_interval(s - mx[:, None])
    sm, slo, shi = lane_strided_sum(e), lane_strided_sum(lo), lane_strided_sum(hi)
    r = F32(ratio)
    with np.errstate(invalid="ignore", divide="ignore"):
        w = _rh(_rh(e / sm[:, None]) * r)
        wlo = _rh(_rh(lo / shi[:, None]) * r)
        whi = _rh(_rh(hi / slo[:, None]) * r)
    return w, wlo, whi


def apply_row(m, w, F):
    """abs_apply_elem over one row: m [D] f16, w [T2] fp32 (f16 values), F [T2, D] f16 -> [D] f16"""
    decay = _rh(lane_strided_sum(w))
    acc = np.zeros(F.shape[1], F32)
    for j in range(F.shape[0]):
        acc = acc + w[j] * F[j].astype(F32)
    keep = _rh(m.astype(F32) * _rh(F32(1.0) - decay))
    return (keep + _rh(acc)).astype(F16)


def _f16_range(lo, hi):
    """every f16 value in [lo, hi] (lo, hi f16 values of one sign, or equal)"""
    if lo == hi or np.isnan(lo) or np.isnan(hi):
        return [F32(lo)]
    a, b = np.array([lo, hi], F16).view(np.uint16).astype(np.int64)
    if lo >= 0:
        bits = range(int(a), int(b) + 1)
    else:
        bits = range(int(b), int(a) + 1)
    return [F32(np.array(v, np.uint16).view(F16)) for v in bits]


def chunk_candidates(M, F, Wq, bq, Wk, bk, ratio):
    """one chunk: M [R, D] f16 (candidate memory rows), F [T2, D] f16 -> (list of R arrays [n_r, D] f16, the nominal
    result [R, D] f16, number of undetermined weights)"""
    q, k = proj(M, Wq, bq), proj(F, Wk, bk)
    w, wlo, whi = weights(q, k, ratio)
    undet = (wlo.view(np.int32) != whi.view(np.int32))
    out, nominal = [], np.empty(M.shape, F16)
    for r in range(M.shape[0]):
        nominal[r] = apply_row(M[r], w[r], F)
        js = np.nonzero(undet[r])[0]
        if len(js) == 0:
            out.append(nominal[r][None])
            continue
        choices = [_f16_range(wlo[r, j], whi[r, j]) for j in js]
        n = int(np.prod([len(c) for c in choices]))
        assert n <= MAX_CANDIDATES, f"row {r}: {n} combinations of undetermined weights"
        rows = []
        for combo in itertools.product(*choices):
            wr = w[r].copy()
            wr[js] = combo
            rows.append(apply_row(M[r], wr, F))
        out.append(np.unique(np.stack(rows).view(np.uint16), axis=0).view(F16))
    return out, nominal, int(undet.sum())


def update_nominal(M, chunks, Wq, bq, Wk, bk, ratio):
    """the Turing update of one step with exp correctly rounded: M [T1, D] f16 folded with each F of `chunks` in turn"""
    for F in chunks:
        q, k = proj(M, Wq, bq), proj(F, Wk, bk)
        w, _, _ = weights(q, k, ratio)
        M = np.stack([apply_row(M[r], w[r], F) for r in range(M.shape[0])])
    return M


def update_candidates(M, chunks, Wq, bq, Wk, bk, ratio):
    """the Turing update of one step: memory M [T1, D] f16 folded with each F of `chunks` in turn.  Returns (cands: a
    list of T1 arrays [n_i, D] f16 — every result row the kernel may produce, the number of undetermined weights)."""
    cands = [M[i][None] for i in range(M.shape[0])]
    n_undet = 0
    for F in chunks:
        owner = np.concatenate([np.full(len(c), i) for i, c in enumerate(cands)])
        out, _, u = chunk_candidates(np.concatenate(cands), F, Wq, bq, Wk, bk, ratio)
        n_undet += u
        new = []
        for i in range(M.shape[0]):
            rows = np.concatenate([out[r] for r in np.nonzero(owner == i)[0]])
            rows = np.unique(rows.view(np.uint16), axis=0).view(F16)
            assert len(rows) <= MAX_CANDIDATES, f"row {i}: {len(rows)} candidate rows"
            new.append(rows)
        cands = new
    return cands, n_undet


def check_rows(got, cands):
    """got [T1, D] f16 (the device's rows) against the candidates of update_candidates -> number of elements decided by
    the expf rule (where a row's candidates disagree).  Raises AssertionError naming the first row that matches none."""
    got = np.ascontiguousarray(got, F16).view(np.uint16)
    n_rule = 0
    for i, c in enumerate(cands):
        cb = c.view(np.uint16)
        ok = (cb == got[i][None]).all(axis=1)
        assert ok.any(), (f"Turing row {i}: matches none of {len(c)} candidate(s); "
                          f"{int((cb[0] != got[i]).sum())} elements differ from the first")
        if len(c) > 1:
            n_rule += int((cb != cb[:1]).any(axis=0).sum())
    return n_rule
