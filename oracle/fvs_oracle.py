"""fvs_oracle — CPU restatement of Flash-VStream's streaming hot path.  TEST INFRASTRUCTURE ONLY.

Only tests/, __graft_entry__.smoke() and bench.py's cpu_baseline / --impl reference legs may import this module;
the product (flash_vstream_b200) never does and has no CPU fallback.

Pinning status (DESIGN.md "Oracle"): the reference has NO tests or golden vectors (SURVEY.md §4, §8c).  This
restatement is pinned against outputs of the reference itself, executed in the build container from
/root/reference (tests/golden/make_golden.py -> tests/golden/*.npz).  The ViT arithmetic lives in the
un-vendored dependency `transformers` (pinned 4.31.0 by Flash-VStream-LLaVA/pyproject.toml:26; 5.5.0 is what
runs here): `vit_forward` restates CLIPVisionModel and is pinned against transformers' CLIPVisionModel on the
same seeded weights.

Each function cites the reference lines it follows.  Paths are relative to
/root/reference/Flash-VStream-LLaVA/flash_vstream/ .

Arithmetic conventions for the f16 consolidation functions (what "reference-exact" means here):
  * every f16 PyTorch op rounds once to binary16 (sub, mul/pow, reduction results, sqrt, div);
  * reductions accumulate in fp32; PyTorch does not specify the accumulation ORDER, so we fix a canonical
    one (`_slice_sum`) that the CUDA kernels reproduce operation for operation — kernel == oracle bit-for-bit;
    oracle == reference up to fp32-reassociation effects, measured on the golden vectors;
  * argmin = first minimal index, NaN wins (torch.argmin).
"""
from __future__ import annotations

import math
from typing import Optional, Sequence

import numpy as np

try:  # torch is only needed by the ViT restatement
    import torch
except Exception:  # pragma: no cover
    torch = None

F16 = np.float16
F32 = np.float32
SLICE = 1024


# ----------------------------------------------------------------------------------------------------------------
# canonical fp32 reductions (mirrored by csrc/mem_device.cuh: slice_sqdiff / butterfly_sum)
# ----------------------------------------------------------------------------------------------------------------
def _slice_sum(terms: np.ndarray) -> np.ndarray:
    """terms [..., n*1024] fp32 -> [..., n] fp32.  Within a 1024-slice lane l owns elements i*256 + l*8 + e
    (i<4, e<8) and adds them sequentially in (i, e) order from 0; the 32 lane sums are combined by an
    xor-butterfly with offsets 16, 8, 4, 2, 1."""
    assert terms.dtype == F32 and terms.shape[-1] % SLICE == 0
    shp = terms.shape[:-1]
    S = terms.shape[-1] // SLICE
    t = terms.reshape(*shp, S, 4, 32, 8)
    acc = np.zeros((*shp, S, 32), F32)
    for i in range(4):
        for e in range(8):
            acc = acc + t[..., i, :, e]
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[..., lanes ^ o]
    return acc[..., 0]


def _lane_sum(terms: np.ndarray) -> np.ndarray:
    """terms [..., n*256] fp32 -> [...] fp32: ONE warp pass over the whole vector — lane l owns elements
    i*256 + l*8 + e (i < n, e < 8), adds them sequentially in (i, e) order, then the xor-butterfly.  For n == 4 this
    equals one `_slice_sum` slice.  Used for the per-patch sums of key retrieval (D = 1024 -> n = 4)."""
    assert terms.dtype == F32 and terms.shape[-1] % 256 == 0
    shp = terms.shape[:-1]
    n = terms.shape[-1] // 256
    t = terms.reshape(*shp, n, 32, 8)
    acc = np.zeros((*shp, 32), F32)
    for i in range(n):
        for e in range(8):
            acc = acc + t[..., i, :, e]
    lanes = np.arange(32)
    for o in (16, 8, 4, 2, 1):
        acc = acc + acc[..., lanes ^ o]
    return acc[..., 0]


def _seq_sum(x: np.ndarray, axis: int = -1) -> np.ndarray:
    """sequential fp32 sum along `axis` starting from 0.0"""
    x = np.moveaxis(x.astype(F32, copy=False), axis, -1)
    acc = np.zeros(x.shape[:-1], F32)
    for i in range(x.shape[-1]):
        acc = acc + x[..., i]
    return acc


def _sqdiff_f16(a: np.ndarray, b: np.ndarray) -> np.ndarray:
    """f16(f16(a-b)^2) widened to fp32 — the per-element term of the reference's diff-form distance."""
    d = (a.astype(F32) - b.astype(F32)).astype(F16)
    return (d.astype(F32) * d.astype(F32)).astype(F16).astype(F32)


def argmin_first_nan(d: np.ndarray, axis: int) -> np.ndarray:
    """torch.argmin semantics: first minimal index; NaN is minimal."""
    d = np.asarray(d, dtype=F32)
    key = np.where(np.isnan(d), -np.inf, d)
    return np.argmin(key, axis=axis)  # numpy returns the first occurrence


# ----------------------------------------------------------------------------------------------------------------
# spatial pooling — model/vstream_arch.py:193-212 (compress_type='mean')
# ----------------------------------------------------------------------------------------------------------------
def spatial_pool(feat: np.ndarray, target: int) -> np.ndarray:
    """feat [T, g*g, D] f16 -> [T, target*target, D] f16.  avg_pool2d(kernel=stride=g//target) on the g x g token
    grid, or global mean when target == 1; fp32 window sum in (ky, kx) order, one division, one rounding."""
    assert feat.dtype == F16
    T, P, D = feat.shape
    g = round(math.sqrt(P))
    assert g * g == P, f"For ViT feature map, {g}*{g}={g*g} != {P}"      # vstream_arch.py:196
    if g == target:
        return feat                                                       # :197-198
    k = g // target                      # avg_pool2d kernel = stride = g // target, no padding (:207)
    c = g // k                           # output cells per side (== target when g % target == 0)
    x = feat.astype(F32).reshape(T, g, g, D)[:, :c * k, :c * k].reshape(T, c, k, c, k, D)
    acc = np.zeros((T, c, c, D), F32)
    for ky in range(k):
        for kx in range(k):
            acc = acc + x[:, :, ky, :, kx, :]
    out = (acc / F32(k * k)).astype(F16)
    return out.reshape(T, c * c, D)


def reshape_2x2(feat: np.ndarray) -> np.ndarray:
    """vstream_arch.py:163-172 (reshape_2x2_image_features): [B, g*g, D] -> [B, (g/2)^2, 4*D]; output token (y, x) holds
    the patches (2y+dy, 2x+dx) for (dy, dx) = (0,0), (0,1), (1,0), (1,1), each with its D channels, in that order."""
    B, P, D = feat.shape
    g = int(round(math.sqrt(P)))
    out = np.empty((B, (g // 2) ** 2, 4 * D), feat.dtype)
    grid = feat.reshape(B, g, g, D)
    for y in range(g // 2):
        for x in range(g // 2):
            for dy in range(2):
                for dx in range(2):
                    c = (dy * 2 + dx) * D
                    out[:, y * (g // 2) + x, c:c + D] = grid[:, 2 * y + dy, 2 * x + dx]
    return out


def spatial_pool3(feat: np.ndarray, a: int = 8, b: int = 4):
    """The STAR hierarchy of embed_video_streaming (vstream_arch.py:644,649,659-662): level a from the ViT output,
    then levels b and 1 from the ROUNDED level a."""
    la = spatial_pool(feat, a)
    return la, spatial_pool(la, b), spatial_pool(la, 1)


# ----------------------------------------------------------------------------------------------------------------
# weighted k-means — model/compress_functions.py:130-169
# ----------------------------------------------------------------------------------------------------------------
def weighted_kmeans(X: np.ndarray, weights: Optional[np.ndarray], init_idx: Sequence[int], refill_idx: Sequence[int],
                    K: int, max_iter: int = 10, tol: float = 1e-4, *, trace: Optional[list] = None,
                    chunk: Optional[int] = None):
    """Inner Lloyd loop `weighted_kmeans_torch` (compress_functions.py:133-157) on f16 data.
    X [T, PD] f16; weights [T] f16 or None (ones, :131-132); init_idx = randperm(T)[:K] (:134);
    refill_idx = the successive random.randint(0, T-1) draws (:152).
    Returns (centroids [K,PD] f16, labels [T] int64, weights_sum [K] f16, exit_step i, refills_consumed).
    trace: a list that gets one dict per iteration — it, diff (the f16 value compared with tol), stop (the loop broke
    there), empty (clusters refilled, in j order), refills (rows consumed), dist_inf / dist_nan (some distance was inf /
    NaN), c_inf / c_nan (some new centroid element was).  chunk: rows per distance batch (memory only, same bits);
    None keeps each batch's [rows, K, PD] fp32 terms near 64 MiB, at most 64 rows."""
    assert X.dtype == F16 and X.ndim == 2 and X.shape[1] % SLICE == 0
    T, PD = X.shape
    w = np.ones(T, F16) if weights is None else weights.astype(F16)
    C = X[np.asarray(init_idx[:K], dtype=np.int64)].copy()
    tol_h = F32(F16(tol))                      # `diff < tol` is evaluated in the tensor dtype (f16)
    pos = 0
    labels = np.zeros(T, np.int64)
    wsum = np.zeros(K, F16)
    it = 0
    rows = chunk if chunk is not None else max(1, min(64, (1 << 24) // max(1, K * PD)))
    for it in range(max_iter):
        # dists = ((X[:,None] - C[None])**2).sum(2).sqrt()                                       (:138)
        dist = np.empty((T, K), F32)
        for t0 in range(0, T, rows):                                  # chunked only to bound memory
            terms = _sqdiff_f16(X[t0:t0 + rows, None, :], C[None, :, :])  # [t, K, PD]
            part = _slice_sum(terms)                                  # [t, K, S]
            del terms
            tot = _seq_sum(part, -1).astype(F16)                      # f16(sum)
            dist[t0:t0 + rows] = np.sqrt(tot.astype(F32)).astype(F16).astype(F32)
        labels = argmin_first_nan(dist, axis=1)                                                   # (:141)
        # weighted centroid update                                                               (:142-149)
        newC = np.empty_like(C)
        n_empty = 0
        empty = []
        for j in range(K):
            members = np.nonzero(labels == j)[0]
            ws = F32(0)
            for t in members:
                ws = F32(ws + F32(w[t]))
            wsum[j] = F16(ws)
            if F32(wsum[j]) > 0:
                acc = np.zeros(PD, F32)
                for t in members:                                      # sequential in t, fp32
                    prod = (F32(w[t]) * X[t].astype(F32)).astype(F16)  # f16(w * x)
                    acc = acc + prod.astype(F32)
                newC[j] = (acc.astype(F16).astype(F32) / F32(wsum[j])).astype(F16)
            else:                                                      # fix nan centroids          (:150-152)
                newC[j] = X[int(refill_idx[pos + n_empty])]
                n_empty += 1
                empty.append(j)
        pos += n_empty
        # diff = torch.norm(C - newC, dim=1).sum()                                               (:153)
        d = (C.astype(F32) - newC.astype(F32)).astype(F16).astype(F32)
        nrm = np.sqrt(_seq_sum(_slice_sum(d * d), -1)).astype(F16)     # squares are NOT rounded to f16 by norm
        diff = F32(_seq_sum(nrm.astype(F32)[None, :], -1)[0].astype(F16))
        if trace is not None:
            nc = newC.astype(F32)
            trace.append(dict(it=it, diff=float(diff), stop=bool(diff < tol_h), empty=empty, refills=n_empty,
                              dist_inf=bool(np.isinf(dist).any()), dist_nan=bool(np.isnan(dist).any()),
                              c_inf=bool(np.isinf(nc).any()), c_nan=bool(np.isnan(nc).any())))
        if diff < tol_h:                                                                          # (:154-155)
            break                                                      # centroids stay the OLD ones
        C = newC                                                                                  # (:156)
    return C, labels, wsum.copy(), it, pos


def step_indices_from_labels(labels: np.ndarray, K: int):
    """compress_functions.py:166-169"""
    return [[[int(j) for j in np.nonzero(labels == i)[0]] for i in range(K)]]


def weighted_kmeans_feature(img_feature: np.ndarray, video_max_frames: int, weights=None, *, init_idx=None,
                            refill_idx=None, trace: Optional[list] = None, result: Optional[dict] = None):
    """compress_functions.py:130-169 incl. the T <= T0 pass-through (:160-161).  RNG draws are explicit inputs.
    trace: passed to weighted_kmeans; result: a dict that gets labels, exit_step and refills of the Lloyd loop."""
    T, P, D = img_feature.shape
    T0 = video_max_frames
    if weights is None:
        weights = np.ones(T, img_feature.dtype)
    if T <= T0:
        return img_feature, weights, [[[i] for i in range(T)]]
    C, labels, wsum, it, used = weighted_kmeans(img_feature.reshape(T, P * D), weights, init_idx, refill_idx, T0,
                                                trace=trace)
    if result is not None:
        result.update(labels=labels, exit_step=it, refills=used)
    return C.reshape(T0, P, D), wsum, step_indices_from_labels(labels, T0)


# ----------------------------------------------------------------------------------------------------------------
# abstract memory — model/vstream_arch.py:174-183 (attention) + :47-52 (NeuralTuringMachine.get_weight)
# and model/compress_functions.py:263-277 (attention_feature)
# ----------------------------------------------------------------------------------------------------------------
def abstract_update(M: np.ndarray, Fnew: np.ndarray, Wq, bq, Wk, bk, ratio: float = 0.2) -> np.ndarray:
    """M [T1,D], Fnew [T2,D] f16; Wq/Wk [H,D], bq/bk [H] f16.  f16 rounding after every PyTorch op, fp32 (here
    fp64-accurate) accumulation inside matmuls — GEMM accumulation order is library-defined, so this function
    is compared with a tolerance, not bit-exactly."""
    f = lambda a: np.asarray(a).astype(F16).astype(np.float64)
    H = Wq.shape[0]
    q = (f(M) @ f(Wq).T + f(bq)).astype(F16)                          # q_proj(x)            (:48)
    k = (f(Fnew) @ f(Wk).T + f(bk)).astype(F16)                       # k_proj(y)            (:49)
    s = (f(q) @ f(k).T).astype(F16)                                   # matmul               (:50)
    s = (s.astype(F32) / F32(math.sqrt(H))).astype(F16)               # / sqrt(output_dim)   (:50)
    s32 = s.astype(F32)
    e = np.exp(s32 - s32.max(axis=-1, keepdims=True))
    wgt = (e / e.sum(axis=-1, keepdims=True)).astype(F16)             # softmax              (:51)
    wgt = (wgt.astype(F32) * F32(ratio)).astype(F16)                  # * update_ratio       (:180)
    decay = wgt.astype(F32).sum(axis=1, keepdims=True).astype(F16)    # sum(dim=1)           (:181)
    keep = (M.astype(F32) * (F32(1.0) - decay.astype(F32)).astype(F16).astype(F32)).astype(F16)
    upd = (f(wgt) @ f(Fnew)).astype(F16)                              # torch.mm             (:182)
    return (keep.astype(F32) + upd.astype(F32)).astype(F16)


def attention_feature(img_feature: np.ndarray, video_max_frames: int, ntm, update_ratio: float = 0.2):
    """compress_functions.py:263-277; ntm = (Wq, bq, Wk, bk)."""
    T, P, D = img_feature.shape
    T0 = video_max_frames
    if T <= T0:
        return img_feature, None
    mem = img_feature[:T0].reshape(T0 * P, D)
    for i in range(T0, T, T0):
        j = min(i + T0, T)
        mem = abstract_update(mem, img_feature[i:j].reshape(-1, D), *ntm, ratio=update_ratio)
    return mem.reshape(T0, P, D), None


# ----------------------------------------------------------------------------------------------------------------
# key-frame retrieval — model/vstream_arch.py:261-268 (offline) / :681-688 (streaming)
# ----------------------------------------------------------------------------------------------------------------
def argsort_desc_stable(w: np.ndarray) -> np.ndarray:
    """Stable descending argsort, NaN first.  The reference's torch.argsort(weight, descending=True) (:261,:681) is
    unstable, so among equal weights ANY order is reference-conformant; ours is the stable one (tie contract)."""
    w = np.asarray(w, dtype=F32)
    key = np.where(np.isnan(w), np.inf, w)
    return np.argsort(-key, kind="stable").astype(np.int64)


def key_retrieve(long_mem: np.ndarray, order: np.ndarray, key_len: int = 3) -> np.ndarray:
    """long_mem [L,P,D] f16 -> idx [min(key_len, L)] int64:
    dists = ((long[:,None] - keyc[None])**2).sum(3).sum(2).sqrt(); argmin(dim=0)."""
    L, P, D = long_mem.shape
    kl = min(key_len, L)
    keyc = long_mem[np.asarray(order[:kl], dtype=np.int64)]
    terms = _sqdiff_f16(long_mem[:, None], keyc[None])                # [L, kl, P, D]
    per_patch = _lane_sum(terms).astype(F16)                           # .sum(dim=3) -> f16   [L, kl, P]
    tot = _seq_sum(per_patch.astype(F32), -1).astype(F16)              # .sum(dim=2) -> f16
    dist = np.sqrt(tot.astype(F32)).astype(F16).astype(F32)            # .sqrt()
    return argmin_first_nan(dist, axis=0).astype(np.int64)


# ----------------------------------------------------------------------------------------------------------------
# offline consolidation — model/vstream_arch.py:214-277 (compress_temporal_features), defaults of
# scripts/train_and_eval.sh:7-14
# ----------------------------------------------------------------------------------------------------------------
class StarConfig:
    def __init__(self, cur_len=1, cur_size=8, long_len=25, long_size=4, tur_len=25, tur_size=1, update_ratio=0.2,
                 key_length=3):
        self.cur_len, self.cur_size = cur_len, cur_size
        self.long_len, self.long_size = long_len, long_size
        self.tur_len, self.tur_size = tur_len, tur_size
        self.update_ratio, self.key_length = update_ratio, key_length


def _compress_long(long_: np.ndarray, cfg: StarConfig, compressor, init_idx, refill_idx, **kmeans_kw):
    """compress_fn(long_memory, video_long_memory_length) (:258, :679): weighted_kmeans_feature by default, or
    `compressor(long_, long_len) -> (long_c, weight, steps)`, e.g. an alternates_oracle function with its draws bound"""
    if compressor is None:
        return weighted_kmeans_feature(long_, cfg.long_len, init_idx=init_idx, refill_idx=refill_idx, **kmeans_kw)
    return compressor(long_, cfg.long_len)


def _weight_order(weight) -> np.ndarray:
    """sorted_indices = torch.argsort(weight, descending=True) followed by long_memory[sorted_indices] and the distance
    broadcast (:261-266, :681-686), raising where they raise for the weights the alternate compressors return: None
    (kdrop and kmeans always, every compressor's T <= T0 pass-through) -> TypeError from torch.argsort; k_merge's
    [T0, T0] similarity matrix -> long_memory[sorted_indices] is [T0, T0, P, D] and (long[:, None] - key[None]) does not
    broadcast for T > T0 >= 2 -> RuntimeError"""
    if weight is None:
        raise TypeError("argsort(): got (NoneType, descending=bool) as the weight to sort")
    w = np.asarray(weight)
    if w.ndim != 1:
        raise RuntimeError(f"a weight of shape {w.shape} gives key centroids that do not broadcast against the long memory")
    return argsort_desc_stable(w)


def compress_temporal_features(feat: np.ndarray, cfg: StarConfig, ntm, *, init_idx=None, refill_idx=None, order=None,
                               compressor=None):
    """feat [T, cur_size^2, D] f16 (already pooled to compress_size) -> (memory [<=681, D], debug dict).
    `order` optionally overrides the descending weight argsort (to replay the reference's unstable tie order).
    `compressor` replaces weighted_kmeans_feature (see _compress_long); its weight feeds the key retrieval."""
    T = feat.shape[0]
    cur_start = min(cfg.cur_len, T)                                                       # :240
    if cur_start == 0:
        cur, long_, tur = feat[:0], feat, feat
    else:
        cur, long_, tur = feat[-cur_start:], feat[:-cur_start], feat[:-cur_start]         # :246-250
    if cfg.long_size ** 2 != long_.shape[1]:
        long_ = spatial_pool(long_, cfg.long_size)                                        # :251-252
    if cfg.tur_size ** 2 != tur.shape[1]:
        tur = spatial_pool(tur, cfg.tur_size)                                             # :253-254
    dbg = {}
    if cfg.long_len == 0 or long_.shape[0] == 0:
        long_c = long_[:0]                                                                # :256-257
    else:
        long_c, weight, _ = _compress_long(long_, cfg, compressor, init_idx, refill_idx)  # :258
        if order is None:
            order = _weight_order(weight)                                                 # :261
        idx = key_retrieve(long_, order, cfg.key_length)                                  # :262-267
        cur = np.concatenate([feat[idx], cur], axis=0)                                    # :268-269
        dbg.update(weight=np.asarray(weight), order=np.asarray(order), key_idx=idx)
    if cfg.tur_len == 0 or tur.shape[0] == 0:
        tur_c = tur[:0]
    else:
        tur_c, _ = attention_feature(tur, cfg.tur_len, ntm, cfg.update_ratio)             # :274
    mem = np.concatenate([tur_c.reshape(-1, feat.shape[2]), long_c.reshape(-1, feat.shape[2]),
                          cur.reshape(-1, feat.shape[2])], axis=0)                        # :275
    return mem, dbg


# ----------------------------------------------------------------------------------------------------------------
# streaming step — model/vstream_arch.py:611-697 (embed_video_streaming), Appendix B of SURVEY.md
# ----------------------------------------------------------------------------------------------------------------
class StreamState:
    def __init__(self):
        self.cur = None   # [<=4, 64, D]
        self.long = None  # [<=25, 16, D]
        self.tur = None   # [<=25, 1, D]
        self.buf = None   # [n, 64, D]   (img_feature_buffer; CPU tensor in the reference)

    def prefix(self):
        """vstream_arch.py:483: cat([Turing, long, cur]) flattened"""
        D = self.cur.shape[-1]
        return np.concatenate([self.tur.reshape(-1, D), self.long.reshape(-1, D), self.cur.reshape(-1, D)], axis=0)


def stream_step(state: StreamState, feat_a: np.ndarray, cfg: StarConfig, ntm, *, init_idx=None, refill_idx=None,
                order=None, trace: Optional[list] = None, compressor=None):
    """One embed_video_streaming call after the encoder: feat_a [t, cur_size^2, D] f16 is the clip's pooled ViT
    output (already `.to(float16)`, :649).  Mutates and returns `state`; returns a debug dict too.
    `compressor` replaces weighted_kmeans_feature as in compress_temporal_features; where the key retrieval raises on its
    weight, `state` is left as it was (the reference publishes at the end of the call, :693-695).

    long_len == 0 switches the long memory and the key retrieval off from the first call on, behind the guard of the
    offline path (compress_temporal_features, :256-257); the reference's streaming branch has no such guard (its first
    call publishes the clip's long rows, its second runs a k-means with K = 0 and raises).

    trace: a list that gets one dict per call — T (long working-set rows), K, S (1024-element slices of a long row), kl
    (key frames retrieved), kmeans (whether the Lloyd loop ran), chunks (rows of each abstract-memory chunk folded in) and
    iters (the weighted_kmeans trace of the call)."""
    t = feat_a.shape[0]
    cur_start = min(cfg.cur_len, t)                                                       # :652
    cur = feat_a[:0] if cur_start == 0 else feat_a[-cur_start:]                           # :653-656
    long_new = spatial_pool(feat_a, cfg.long_size) if cfg.long_size ** 2 != feat_a.shape[1] else feat_a  # :659-660
    tur_new = spatial_pool(feat_a, cfg.tur_size) if cfg.tur_size ** 2 != feat_a.shape[1] else feat_a     # :661-662
    if cfg.long_len == 0:
        long_new = long_new[:0]
    dbg = {}
    S = long_new.shape[1] * long_new.shape[2] // SLICE
    if state.buf is None:                                                                 # first call: :669-672 skipped
        state.cur, state.long, state.tur, state.buf = cur, long_new, tur_new, feat_a
        if trace is not None:
            trace.append(dict(T=long_new.shape[0], K=cfg.long_len, S=S, kl=0, kmeans=False, chunks=[], iters=[]))
        return state, dbg
    buf = np.concatenate([state.buf, feat_a], axis=0)                                     # :676
    L = np.concatenate([state.long, long_new], axis=0)                                    # :678
    iters, res = [], {}
    if cfg.long_len == 0:
        long_c, idx = L, np.zeros(0, np.int64)
    else:
        kw = dict(trace=iters, result=res) if compressor is None else {}
        long_c, weight, _ = _compress_long(L, cfg, compressor, init_idx, refill_idx, **kw)  # :679
        if order is None:
            order = _weight_order(weight)                                                 # :681
        idx = key_retrieve(L, order, cfg.key_length)                                      # :682-687
        dbg.update(weight=np.asarray(weight), order=np.asarray(order))
    key = buf[idx]                                    # global buffer indexed by working-set indices (:688, quirk)
    cur = np.concatenate([key, cur], axis=0)                                              # :689
    Tm = np.concatenate([state.tur, tur_new], axis=0)                                     # :690
    tur_c, _ = attention_feature(Tm, cfg.tur_len, ntm, cfg.update_ratio)                  # :691
    dbg.update(key_idx=idx, **res)
    if trace is not None:
        T1 = cfg.tur_len
        chunks = [min(T1, Tm.shape[0] - i) for i in range(T1, Tm.shape[0], T1)] if Tm.shape[0] > T1 else []
        trace.append(dict(T=L.shape[0], K=cfg.long_len, S=S, kl=len(idx), kmeans=bool(res), chunks=chunks, iters=iters))
    state.cur, state.long, state.tur, state.buf = cur, long_c, tur_c, buf                 # :693-695
    return state, dbg


# ----------------------------------------------------------------------------------------------------------------
# ViT-L/14 encoder — multimodal_encoder/clip_encoder.py:31-53 over transformers CLIPVisionModel
# (modeling_clip.py: CLIPVisionEmbeddings, CLIPEncoderLayer, CLIPAttention, CLIPMLP; quick_gelu)
# ----------------------------------------------------------------------------------------------------------------
class VitConfig:
    def __init__(self, image_size=336, patch_size=14, hidden=1024, heads=16, mlp=4096, layers=24, select_layer=-2,
                 ln_eps=1e-5):
        self.image_size, self.patch_size, self.hidden, self.heads = image_size, patch_size, hidden, heads
        self.mlp, self.layers, self.select_layer, self.ln_eps = mlp, layers, select_layer, ln_eps

    @property
    def grid(self):
        return self.image_size // self.patch_size

    @property
    def tokens(self):
        return self.grid ** 2 + 1

    @property
    def layers_run(self):
        """hidden_states has layers+1 entries (index 0 = embeddings after pre-LN); hidden_states[select_layer] is the
        output of encoder layer (layers + select_layer) counted from 1, i.e. that many layers must run."""
        return self.layers + 1 + self.select_layer if self.select_layer < 0 else self.select_layer


def random_vit_weights(cfg: VitConfig, seed: int = 0, n_layers: Optional[int] = None):
    """Seeded synthetic weights (fp32 torch tensors).  Scales are chosen so attention logits have O(1) spread and
    activations stay well inside f16 range — parity is about arithmetic, not accuracy (no checkpoints offline)."""
    g = torch.Generator(device="cpu").manual_seed(seed)
    H, Mlp, P = cfg.hidden, cfg.mlp, cfg.patch_size
    rn = lambda *s, std=1.0: torch.randn(*s, generator=g) * std
    w = {
        "patch_w": rn(H, 3, P, P, std=0.02), "class_emb": rn(H, std=0.5), "pos_emb": rn(cfg.tokens, H, std=0.3),
        "pre_ln_w": 1 + rn(H, std=0.1), "pre_ln_b": rn(H, std=0.1), "layers": [],
    }
    for _ in range(cfg.layers if n_layers is None else n_layers):
        w["layers"].append({
            "ln1_w": 1 + rn(H, std=0.1), "ln1_b": rn(H, std=0.05),
            "q_w": rn(H, H, std=0.04), "q_b": rn(H, std=0.1), "k_w": rn(H, H, std=0.04), "k_b": rn(H, std=0.1),
            "v_w": rn(H, H, std=0.03), "v_b": rn(H, std=0.02), "o_w": rn(H, H, std=0.02), "o_b": rn(H, std=0.02),
            "ln2_w": 1 + rn(H, std=0.1), "ln2_b": rn(H, std=0.05),
            "fc1_w": rn(Mlp, H, std=0.03), "fc1_b": rn(Mlp, std=0.1), "fc2_w": rn(H, Mlp, std=0.015), "fc2_b": rn(H, std=0.02),
        })
    return w


def cast_weights(w, dtype):
    """round every weight to `dtype` and widen back to fp32 (what an f16 checkpoint holds)"""
    c = lambda t: t.to(dtype).to(torch.float32)
    out = {k: (c(v) if k != "layers" else [{kk: c(vv) for kk, vv in l.items()} for l in v]) for k, v in w.items()}
    return out


def vit_forward(pixels, w, cfg: VitConfig, layers_run: Optional[int] = None, round_dtype=None, residual_fp32=False,
                keep_cls=False):
    """pixels [B,3,S,S] fp32 torch -> hidden_states[select_layer][:, 1:]  [B, grid^2, hidden] fp32.
    round_dtype=torch.float16 emulates an f16 activation pipeline (rounding wherever the CUDA path stores a tensor)
    so tests can budget the tolerance; None = exact fp32 restatement."""
    rd = (lambda t: t.to(round_dtype).to(torch.float32)) if round_dtype is not None else (lambda t: t)
    rres = (lambda t: t) if residual_fp32 else rd
    B = pixels.shape[0]
    H, nh = cfg.hidden, cfg.heads
    hd = H // nh
    L = cfg.layers_run if layers_run is None else layers_run
    # CLIPVisionEmbeddings: conv(stride=patch, no bias) -> flatten -> [cls | patches] + position_embedding
    x = torch.nn.functional.conv2d(pixels, w["patch_w"], stride=cfg.patch_size)          # [B,H,g,g]
    x = x.flatten(2).transpose(1, 2)                                                     # [B,g*g,H]
    x = torch.cat([w["class_emb"].expand(B, 1, H), x], dim=1) + w["pos_emb"]
    x = rd(x)
    x = rres(torch.nn.functional.layer_norm(x, (H,), w["pre_ln_w"], w["pre_ln_b"], cfg.ln_eps))   # pre_layrnorm
    for l in range(L):
        p = w["layers"][l]
        y = rd(torch.nn.functional.layer_norm(x, (H,), p["ln1_w"], p["ln1_b"], cfg.ln_eps))
        q = rd(y @ p["q_w"].T + p["q_b"]).view(B, -1, nh, hd).transpose(1, 2)
        k = rd(y @ p["k_w"].T + p["k_b"]).view(B, -1, nh, hd).transpose(1, 2)
        v = rd(y @ p["v_w"].T + p["v_b"]).view(B, -1, nh, hd).transpose(1, 2)
        s = (q @ k.transpose(-1, -2)) * (hd ** -0.5)
        a = rd(torch.softmax(s, dim=-1))
        ctx = rd((a @ v).transpose(1, 2).reshape(B, -1, H))
        x = rres(x + ctx @ p["o_w"].T + p["o_b"])
        y = rd(torch.nn.functional.layer_norm(x, (H,), p["ln2_w"], p["ln2_b"], cfg.ln_eps))
        h = y @ p["fc1_w"].T + p["fc1_b"]
        h = rd(h * torch.sigmoid(1.702 * h))                                             # quick_gelu
        x = rres(x + h @ p["fc2_w"].T + p["fc2_b"])
    return rd(x if keep_cls else x[:, 1:])                # feature_select 'cls_patch' / 'patch' (clip_encoder.py:31-39)


def hf_state_dict(w, cfg: VitConfig):
    """Map our weight dict onto transformers.CLIPVisionModel parameter names (to run the reference's dependency
    on the same numbers)."""
    sd = {
        "vision_model.embeddings.class_embedding": w["class_emb"],
        "vision_model.embeddings.patch_embedding.weight": w["patch_w"],
        "vision_model.embeddings.position_embedding.weight": w["pos_emb"],
        "vision_model.pre_layrnorm.weight": w["pre_ln_w"], "vision_model.pre_layrnorm.bias": w["pre_ln_b"],
    }
    for i, p in enumerate(w["layers"]):
        b = f"vision_model.encoder.layers.{i}."
        sd.update({
            b + "layer_norm1.weight": p["ln1_w"], b + "layer_norm1.bias": p["ln1_b"],
            b + "self_attn.q_proj.weight": p["q_w"], b + "self_attn.q_proj.bias": p["q_b"],
            b + "self_attn.k_proj.weight": p["k_w"], b + "self_attn.k_proj.bias": p["k_b"],
            b + "self_attn.v_proj.weight": p["v_w"], b + "self_attn.v_proj.bias": p["v_b"],
            b + "self_attn.out_proj.weight": p["o_w"], b + "self_attn.out_proj.bias": p["o_b"],
            b + "layer_norm2.weight": p["ln2_w"], b + "layer_norm2.bias": p["ln2_b"],
            b + "mlp.fc1.weight": p["fc1_w"], b + "mlp.fc1.bias": p["fc1_b"],
            b + "mlp.fc2.weight": p["fc2_w"], b + "mlp.fc2.bias": p["fc2_b"],
        })
    return sd


# ----------------------------------------------------------------------------------------------------------------
# mm_projector — model/multimodal_projector/builder.py:35-51 ('mlpNx_gelu': Linear, then (GELU, Linear) x (N-1))
# ----------------------------------------------------------------------------------------------------------------
def mlp_gelu_projector(x, weights):
    """x [rows, in] fp32 torch; weights = [(W0, b0), (W1, b1), ...] fp32; exact (erf) GELU between layers."""
    for i, (W, b) in enumerate(weights):
        x = x @ W.T + b
        if i + 1 < len(weights):
            x = torch.nn.functional.gelu(x)
    return x
