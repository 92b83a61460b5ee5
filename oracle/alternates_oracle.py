"""CPU restatement of the alternate temporal compressors selectable through `video_sample_type`
(Flash-VStream-LLaVA/flash_vstream/model/vstream_arch.py:222-236, 626-637): drop_feature, merge_feature, kmeans_feature,
k_drop_feature, k_merge_feature of flash_vstream/model/compress_functions.py (:19, :57, :91, :170, :213).
TEST INFRASTRUCTURE — only tests/ may import this.  Pinned by tests/golden/alternates.npz, recorded by executing the
reference's own functions on CPU f16 tensors (tests/golden/make_golden_alternates.py).

f16 arithmetic contract (one rounding per PyTorch op, verified against ATen on CPU):
  ||v||      = f16( sqrt_f32( sum_f32( v_i * v_i ) ) )                    torch.linalg.vector_norm (products NOT rounded)
  cos(a, b)  = f16( sum_f32( f16( f16(a_i/||a||) * f16(b_i/||b||) ) ) )   F.cosine_similarity: normalise first, then dot
  normalize  = f16( v_i / ||v|| )                                         F.normalize(p=2)
  mm         = f16( sum_f32( a_i * b_i ) )                                torch.mm on f16
Every sum_f32 runs in the canonical slice order (fvs_oracle._slice_sum, slices added sequentially), which is what the CUDA
kernels implement; ATen's own order differs by fp32 rounding noise, so similarities can differ from the reference by one f16
ulp and an argmax between two near-equal similarities may resolve differently — the goldens use separated data, and the
kernels are bit-exact against THIS file.
RNG: random.randint coin flips (drop variants) and torch.randperm / random.randint (kmeans) are explicit inputs.
"""
from __future__ import annotations

from typing import List, Optional, Sequence

import numpy as np

from .fvs_oracle import F16, F32, _seq_sum, _slice_sum, argmin_first_nan, step_indices_from_labels

NEG = F32(-100.0)


def _h(x):
    return np.asarray(x, F32).astype(F16).astype(F32)


def _sum(terms: np.ndarray) -> np.ndarray:
    """canonical fp32 sum over the last axis (length % 1024 == 0)"""
    return _seq_sum(_slice_sum(np.ascontiguousarray(terms, dtype=F32)), -1)


def norm16(v: np.ndarray) -> np.ndarray:
    v = v.astype(F32)
    return _h(np.sqrt(_sum(v * v)))


def normalize16(v: np.ndarray) -> np.ndarray:
    """F.normalize(v, p=2, dim=-1) on f16 rows (eps 1e-12 underflows to 0 in f16: plain division)"""
    with np.errstate(divide="ignore", invalid="ignore"):
        return _h(v.astype(F32) / norm16(v)[..., None])


def dot16(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """torch.mm element: f16(sum_f32(a*b)) — f16 x f16 products are exact in fp32"""
    return _h(_sum(a.astype(F32) * b.astype(F32)))


def cos16(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """F.cosine_similarity(a, b, dim=-1) on f16"""
    return _h(_sum(_h(normalize16(a) * normalize16(b))))


def argmax_first_nan(v: np.ndarray) -> int:
    """torch.argmax on the flattened array: first maximal index, NaN is maximal"""
    v = np.asarray(v, F32).reshape(-1)
    return int(np.argmax(np.where(np.isnan(v), np.inf, v)))


def _adjacent_sims(F: np.ndarray, T0: int) -> List[np.float32]:
    return [cos16(F[i], F[i + 1]) for i in range(T0 - 1)]


# ---------------------------------------------------------------------------------------------------- drop_feature (:19-54)
def drop_feature(img_feature: np.ndarray, video_max_frames: int, img_similarity=None, *, coins: Sequence[int] = ()):
    T, P, D = img_feature.shape
    T0 = video_max_frames
    indices = [[i] for i in range(T)]
    if T <= T0:
        return img_feature, img_similarity, [indices]
    X = img_feature.reshape(T, P * D)
    kept = list(range(T0))                                   # frame index of every kept row
    sim = [F32(s) for s in img_similarity[:T0 - 1]] if img_similarity is not None else _adjacent_sims(X, T0)
    cur_indices = indices[:T0]
    steps = [cur_indices]
    for n, i in enumerate(range(T0, T)):
        new_sim = cos16(X[kept[-1]], X[i])
        allk = kept + [i]
        all_idx = cur_indices + [[i]]
        all_sim = sim + [new_sim]
        idx = argmax_first_nan(np.array(all_sim))
        if coins[n] > 0:
            idx += 1
        kept = allk[:idx] + allk[idx + 1:]
        if idx + 1 == T0 + 1:
            sim = all_sim[:T0 - 1]
            cur_indices = all_idx[:-1]
        elif idx == 0:
            sim = all_sim[1:]
            cur_indices = all_idx[1:]
        else:
            sim = all_sim[:idx] + all_sim[idx + 1:]
            sim[idx - 1] = cos16(X[allk[idx - 1]], X[allk[idx + 1]])
            cur_indices = all_idx[:idx] + all_idx[idx + 1:]
        steps.append(cur_indices)
    return X[kept].reshape(T0, P, D), np.array(sim, F32).astype(F16), steps


# ---------------------------------------------------------------------------------------------------- merge_feature (:57-88)
def merge_feature(img_feature: np.ndarray, video_max_frames: int, img_similarity=None):
    T, P, D = img_feature.shape
    T0 = video_max_frames
    indices = [[i] for i in range(T)]
    if T <= T0:
        return img_feature, img_similarity, [indices]
    X = img_feature.reshape(T, P * D)
    cur = [X[i].copy() for i in range(T0)]
    cur_indices = indices[:T0]
    steps = [cur_indices]
    sim = [F32(s) for s in img_similarity[:T0 - 1]] if img_similarity is not None else _adjacent_sims(X, T0)
    for i in range(T0, T):
        new_sim = cos16(cur[-1], X[i])
        allf = cur + [X[i].copy()]
        all_sim = sim + [new_sim]
        all_idx = cur_indices + [[i]]
        idx = argmax_first_nan(np.array(all_sim))
        allf[idx + 1] = (_h(allf[idx].astype(F32) + allf[idx + 1].astype(F32)) / F32(2.0)).astype(F16)
        all_idx[idx + 1] = all_idx[idx] + all_idx[idx + 1]
        cur = allf[:idx] + allf[idx + 1:]
        sim = all_sim[:idx] + all_sim[idx + 1:]
        cur_indices = all_idx[:idx] + all_idx[idx + 1:]
        if idx > 0:
            sim[idx - 1] = cos16(allf[idx - 1], allf[idx + 1])
        if idx + 1 < T0:
            sim[idx] = cos16(allf[idx + 1], allf[idx + 2])
        steps.append(cur_indices)
    return np.stack(cur).reshape(T0, P, D), np.array(sim, F32).astype(F16), steps


# ---------------------------------------------------------------------------------------------------- kmeans_feature (:91-127)
def cdist16(X: np.ndarray, C: np.ndarray, stats: Optional[list] = None) -> np.ndarray:
    """torch.cdist(X, C, p=2) on f16 with more than 25 rows on either side: ATen's matmul form (_euclidean_dist):
    [-2x, |x|^2, 1] . [c, 1, |c|^2] accumulated in fp32 as ONE dot product, rounded to f16, clamp_min(0), sqrt.
    |v|^2 = f16(sum_f32(f16(v_i^2))) (v.pow(2).sum(-1) on f16): +inf once the row's mean square passes 65504 / PD or
    one |v_i| >= 256, and then every distance of that row is inf (or NaN, which clamp_min keeps).
    stats: a list that gets the fraction of rows of X whose |x|^2 is inf."""
    Xf, Cf = X.astype(F32), C.astype(F32)
    xn = _h(_sum(_h(Xf * Xf)))
    cn = _h(_sum(_h(Cf * Cf)))
    if stats is not None:
        stats.append(float(np.isinf(xn).mean()))
    out = np.empty((X.shape[0], C.shape[0]), F32)
    for t in range(X.shape[0]):
        part = _seq_sum(_slice_sum((F32(-2.0) * Xf[t])[None, :] * Cf), -1)     # slices sequential
        tot = (part + xn[t]) + cn                                              # then the two appended columns
        out[t] = _h(np.sqrt(np.maximum(_h(tot), F32(0.0))))
    return out


def kmeans_feature(img_feature: np.ndarray, video_max_frames: int, img_similarity=None, *, init_idx: Sequence[int] = (),
                   refill_idx: Sequence[int] = (), max_iter: int = 10, tol: float = 1e-4, result: Optional[dict] = None):
    """result: a dict that gets labels, exit_step, refills and converged of the Lloyd loop, and per iteration whether some
    |x|^2 was inf (xn_inf) and some distance NaN (dist_nan)"""
    T, P, D = img_feature.shape
    T0 = video_max_frames
    if T <= T0:
        return img_feature, img_similarity, [[[i] for i in range(T)]]
    X = img_feature.reshape(T, P * D)
    C = X[np.asarray(init_idx[:T0], np.int64)].copy()
    tol_h = F32(F16(tol))
    pos = 0
    labels = np.zeros(T, np.int64)
    it, converged, xn_inf, dist_nan = 0, False, [], []
    for it in range(max_iter):
        dist = cdist16(X, C, stats=xn_inf)
        dist_nan.append(bool(np.isnan(dist).any()))
        labels = argmin_first_nan(dist, axis=1)
        new = np.empty_like(C)
        for j in range(T0):
            members = np.nonzero(labels == j)[0]
            if len(members) > 0:                                # cluster_points.mean(0): fp32 accumulate, / n, one rounding
                acc = np.zeros(P * D, F32)
                for t in members:
                    acc = acc + X[t].astype(F32)
                new[j] = (acc / F32(len(members))).astype(F16)
            else:
                new[j] = X[int(refill_idx[pos])]
                pos += 1
        d = _h(C.astype(F32) - new.astype(F32))
        nrm = _h(np.sqrt(_sum(d * d)))
        diff = _h(_seq_sum(nrm[None, :], -1)[0])
        if diff < tol_h:
            converged = True
            break
        C = new
    if result is not None:
        result.update(labels=labels, exit_step=it, refills=pos, converged=converged, xn_inf=xn_inf, dist_nan=dist_nan)
    return C.reshape(T0, P, D), img_similarity, step_indices_from_labels(labels, T0)


# ---------------------------------------------------------------------------------------------------- k_drop / k_merge
def _sim_matrix(N: np.ndarray) -> np.ndarray:
    n = N.shape[0]
    S = np.empty((n, n), F32)
    for i in range(n):
        S[i] = dot16(N[i][None, :], N)
    np.fill_diagonal(S, NEG)
    return S


def _extend_sim(S: np.ndarray, new_sim: np.ndarray) -> np.ndarray:
    n = S.shape[0]
    A = np.full((n + 1, n + 1), NEG, F32)
    A[:n, :n] = S
    A[:n, n] = new_sim
    A[n, :n] = new_sim
    return A


def k_drop_feature(img_feature: np.ndarray, video_max_frames: int, img_similarity=None, *, coins: Sequence[int] = ()):
    """:170-210"""
    T, P, D = img_feature.shape
    T0 = video_max_frames
    indices = [[i] for i in range(T)]
    if T <= T0:
        return img_feature, img_similarity, [indices]
    X = img_feature.reshape(T, P * D)
    kept = list(range(T0))
    N = normalize16(X[:T0]).astype(F16)
    S = _sim_matrix(N)
    cur_indices = indices[:T0]
    steps = [cur_indices]
    for n, i in enumerate(range(T0, T)):
        nn = normalize16(X[i]).astype(F16)
        A = _extend_sim(S, dot16(N, nn[None, :]))
        allk, all_idx = kept + [i], cur_indices + [[i]]
        allN = np.concatenate([N, nn[None, :]])
        flat = argmax_first_nan(A)
        left, right = flat // (T0 + 1), flat % (T0 + 1)
        idx = left if coins[n] > 0 else right
        kept = allk[:idx] + allk[idx + 1:]
        N = np.delete(allN, idx, axis=0)
        cur_indices = all_idx[:idx] + all_idx[idx + 1:]
        S = np.delete(np.delete(A, idx, axis=0), idx, axis=1)
        steps.append(cur_indices)
    return X[kept].reshape(T0, P, D), None, steps


def k_merge_feature(img_feature: np.ndarray, video_max_frames: int, img_similarity=None):
    """:213-260"""
    T, P, D = img_feature.shape
    T0 = video_max_frames
    indices = [[i] for i in range(T)]
    if T <= T0:
        return img_feature, img_similarity, [indices]
    X = img_feature.reshape(T, P * D)
    cur = X[:T0].copy()
    N = normalize16(cur).astype(F16)
    S = _sim_matrix(N)
    cur_indices = indices[:T0]
    steps = [cur_indices]
    for i in range(T0, T):
        nn = normalize16(X[i]).astype(F16)
        A = _extend_sim(S, dot16(N, nn[None, :]))
        allf = np.concatenate([cur, X[i][None, :]])
        allN = np.concatenate([N, nn[None, :]])
        all_idx = cur_indices + [[i]]
        flat = argmax_first_nan(A)
        left, right = flat // (T0 + 1), flat % (T0 + 1)
        allf[right] = (_h(allf[left].astype(F32) + allf[right].astype(F32)) / F32(2.0)).astype(F16)
        allN[right] = normalize16(allf[right]).astype(F16)
        all_idx[right] = all_idx[left] + all_idx[right]
        ns = dot16(allN, allN[right][None, :])
        A[right, :] = ns
        A[:, right] = ns
        A[right, right] = NEG
        cur = np.delete(allf, left, axis=0)
        N = np.delete(allN, left, axis=0)
        cur_indices = all_idx[:left] + all_idx[left + 1:]
        S = np.delete(np.delete(A, left, axis=0), left, axis=1)
        steps.append(cur_indices)
    return cur.reshape(T0, P, D), S.astype(F16), steps
