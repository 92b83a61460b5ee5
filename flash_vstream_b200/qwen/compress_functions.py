"""Drop-in mirror of Flash-VStream-Qwen/models/compress_functions.py for the path the Qwen Flash Memory takes by default
(`flash_memory_temporal_method='kmeans_ordered'`): weighted_kmeans_ordered_feature (:181-298), on the sm_90a kernels.

RNG: default draws come from `draws.GLOBAL`, the global generators the reference draws from (contract in draws.py);
explicit draws (init_idx= / refill_idx= / order=) bypass it, which is what the parity tests do with the draws recorded
from the reference.
"""
from __future__ import annotations

from typing import Optional

import numpy as np
import torch

from . import ops as Q
from .. import _lib as L
from ..draws import GLOBAL, DrawSource, to_device

MAX_ITER = 10   # compress_functions.py:203 (max_iter=10)
TOL = 1e-4      # compress_functions.py:203 (tol=1e-4)


def weighted_kmeans_ordered_feature(img_feature: torch.Tensor, video_max_frames: int, weights: Optional[torch.Tensor] = None,
                                    times=None, *, init_idx=None, refill_idx=None, order=None, source: DrawSource = GLOBAL):
    """compress_functions.py:181-298.  img_feature [T, P, D] (f16 / bf16 / f32, CUDA); `source`: where the default draws
    come from.  Returns
    (sorted_reduced_feature [T0, P, D] in the input dtype, sorted_weights fp32 [T0], centroids_timestamp fp32 [T0],
    sorted_step_indices) — or, like the reference, the 3-tuple (img_feature.float(), weights, [[[0], [1], ...]]) when
    T <= T0 (:265-266).  `order` replays the reference's (unstable) torch.argsort(centroids_timestamp) permutation; the
    default is the stable order."""
    dtype = img_feature.dtype
    dev = img_feature.device
    T, P, D = img_feature.shape
    T0 = int(video_max_frames)
    if weights is None:
        weights = torch.ones(T, dtype=torch.float32, device=dev)
    if T <= T0:
        return img_feature.float(), weights, [[[i] for i in range(T)]]
    X = img_feature.reshape(T, P * D)
    uniq_idx, n_unique = Q.unique_rows(X)                              # torch.unique(X, dim=0), :204
    U = int(n_unique.item())
    w32 = weights.to(torch.float32)
    if U < T0:                                                         # :205-216 fewer distinct frames than clusters
        K = U
        C, _, labels, _ = Q.kmeans_ordered(X, w32, uniq_idx, torch.arange(U, dtype=torch.int32, device=dev),
                                           torch.zeros(1, dtype=torch.int32, device=dev), K, max_iter=0, tol=TOL)
        wsum = torch.ones(U, dtype=torch.float32, device=dev)
        exit_step = -1
        lab = labels.cpu().tolist()
    else:
        K = T0
        if init_idx is None:
            init_idx = source.randperm(U, dev)[:K]                      # :218
        init_idx = torch.as_tensor(init_idx).to(device=dev, dtype=torch.int32)
        if refill_idx is None:
            refill_dev, _ = source.refill_candidates(T, MAX_ITER * K, dev)    # :258, drawn ahead
        else:
            refill = list(int(v) for v in refill_idx)
            refill_dev = to_device(refill + [0] * (MAX_ITER * K - len(refill)), np.int32, dev)
        C, wsum, labels, info = Q.kmeans_ordered(X, w32, uniq_idx, init_idx, refill_dev, K, MAX_ITER, TOL)
        lab = labels.cpu().tolist()                                     # the member lists need the labels on the host
        info_h = info.cpu().tolist()
        exit_step = info_h[0]
        if refill_idx is None:                                          # leave `random` where the reference would
            source.consume(T, info_h[1])
    step_indices = [[] for _ in range(K)]
    for j, l in enumerate(lab):                                         # :274-277
        step_indices[l].append(j)
    ts = np.array([sum(m) / len(m) for m in step_indices], np.float32)  # :284-285 (ZeroDivisionError if a cluster is empty)
    if order is None:
        order = np.argsort(ts, kind="stable")                           # :287 torch.argsort(centroids_timestamp)
    order = [int(i) for i in order]
    sorted_idx = torch.tensor(order, dtype=torch.int64, device=dev)
    feat = Q.gather_rows_cast(C.view(K, P, D), sorted_idx, dtype)       # :288 + the final .to(dtype) (:297)
    sorted_weights = wsum[sorted_idx]
    timestamps = torch.from_numpy(ts[order]).to(dev)
    sorted_steps = [step_indices[i] for i in order]
    if exit_step == -1:                                                 # :291-296 pad with the first frames
        pad_len = T0 - K
        feat = torch.cat([img_feature[:pad_len], feat])
        sorted_weights = torch.cat([torch.ones(pad_len, device=dev), sorted_weights])
        timestamps = torch.cat([torch.arange(pad_len, device=dev), timestamps])
        sorted_steps = [[i] for i in range(pad_len)] + sorted_steps
    return feat, sorted_weights, timestamps, sorted_steps


class LazyMembers:
    """The `sorted_step_indices` list of weighted_kmeans_ordered_feature (:274-277, :288) as a sequence that is only
    materialised — one D2H copy of the labels and the cluster order — when somebody looks at it.  The streaming step passes
    it to spatial_enhance, which never does."""

    def __init__(self, labels: torch.Tensor, sorted_idx: torch.Tensor):
        self._labels, self._sorted_idx, self._lists = labels, sorted_idx, None

    def _get(self):
        if self._lists is None:
            lab, order = self._labels.cpu().tolist(), self._sorted_idx.cpu().tolist()
            members = [[] for _ in order]
            for j, l in enumerate(lab):
                members[l].append(j)
            self._lists = [members[i] for i in order]
            self._labels = self._sorted_idx = None
        return self._lists

    def __len__(self):
        return len(self._get())

    def __iter__(self):
        return iter(self._get())

    def __getitem__(self, i):
        return self._get()[i]

    def __eq__(self, other):
        return list(self._get()) == list(other)

    def __repr__(self):
        return repr(self._get())


def ordered_kmeans_enqueue_multi(reqs, video_max_frames: int, budget: int = 0):
    """The non-degenerate branch of weighted_kmeans_ordered_feature (:216-290: at least T0 distinct frames) for many
    streams at once (DESIGN.md §3.17), enqueued without a single host round trip: unique rows, the Lloyd loop, the
    timestamp / ordering bookkeeping (fvs_qwen_kmeans_finalize) and the sorted gather all stay on the device, and each of
    those four kernels runs once per launch group for all streams; a stream's bits do not depend on the other streams.
    reqs = [(img_feature [T, P, D], weights [T], init_idx, refill_idx, order or None)]: init_idx int32 [T0] indexes the
    unique-row list like `unique_X[indices]` (:219), refill_idx int32 [MAX_ITER * T0] are the candidate draws.
    Returns (outs, readback).  outs: per stream a dict of device tensors, feat [T0, P, D] (input dtype), weights /
    timestamps fp32 [T0], members (LazyMembers), and what the caller has to look at ONCE, after everything it wants has
    been enqueued, to know the result is valid: n_unique int32 [1] (must be >= T0, and == T when init_idx was drawn as
    randperm(T)), info int32 [4] ({last iteration, refills consumed, converged, 0}), flags int32 [1] (empty clusters:
    ZeroDivisionError in the reference).  readback: a device int32 [n, 8] holding each stream's n_unique, info[4] and
    flags in columns 0, 1-4 and 5 (the dicts' n_unique, info and flags are views of it), so the caller copies every
    stream's read-back at once."""
    n, K = len(reqs), int(video_max_frames)
    dev = reqs[0][0].device
    Ts = [r[0].shape[0] for r in reqs]
    rb = torch.zeros(n, 8, dtype=torch.int32, device=dev)
    uniq = torch.zeros(sum(Ts), dtype=torch.int32, device=dev)      # zero-filled, as unique_rows (ops.py) leaves it
    labels = torch.empty(sum(Ts), dtype=torch.int32, device=dev)
    small = torch.empty(n, 3, K, dtype=torch.float32, device=dev)     # wsum, timestamps, sorted weights
    sorted_idx = torch.empty(n, K, dtype=torch.int64, device=dev)
    lib = L.load()
    sizes = []
    for (x, *_), T in zip(reqs, Ts):
        PD = x[0].numel()
        sizes.append((Q._al(K * PD * 4), Q._al(lib.fvs_qwen_unique_workspace_bytes(T)),
                      Q._al(lib.fvs_qwen_kmeans_workspace_bytes(T, K, PD))))
    ws = Q._workspace(sum(map(sum, sizes)), dev, "mem_multi")
    jobs, outs, keep, o, t0 = [], [], [], 0, 0           # keep: converted inputs, alive until the calls are enqueued
    for i, ((x, w, init_idx, refill_idx, order), T, (nc, nu, nk)) in enumerate(zip(reqs, Ts, sizes)):
        assert T > K and init_idx.dtype == torch.int32 and refill_idx.dtype == torch.int32
        X, w32 = Q._c(x.reshape(T, -1)), Q._c(w.to(torch.float32))
        order = None if order is None else Q._c(order)
        init_idx, refill_idx = Q._c(init_idx), Q._c(refill_idx)
        keep.append((X, w32, order, init_idx, refill_idx))
        PD = X.shape[1]
        C = ws[o: o + K * PD * 4].view(torch.float32).view(K, PD)
        feat = torch.empty((K,) + tuple(x.shape[1:]), dtype=x.dtype, device=dev)
        lab = labels[t0: t0 + T]
        jobs.append(Q.mem_job(X, K, w=w32, init_idx=init_idx, refill_idx=refill_idx,
                              max_iter=MAX_ITER, tol=TOL, uniq_idx=uniq[t0: t0 + T], n_unique=rb[i, 0:1],
                              uniq_ws=ws[o + nc: o + nc + nu], C=C, wsum=small[i, 0], labels=lab, info=rb[i, 1:5],
                              km_ws=ws[o + nc + nu: o + nc + nu + nk], order=order,
                              sorted_idx=sorted_idx[i], ts=small[i, 1], w_sorted=small[i, 2], flags=rb[i, 5:6], out=feat))
        outs.append(dict(feat=feat, weights=small[i, 2], timestamps=small[i, 1], members=LazyMembers(lab, sorted_idx[i]),
                         n_unique=rb[i, 0:1], info=rb[i, 1:5], flags=rb[i, 5:6]))
        o += nc + nu + nk
        t0 += T
    arr = Q.mem_jobs(jobs)
    Q.unique_rows_multi(arr, budget)
    Q.kmeans_multi(arr, budget)
    Q.kmeans_finalize_multi(arr, budget)
    Q.gather_rows_cast_multi(arr, budget)
    return outs, rb


def fast_weighted_kmeans_ordered_feature(img_feature, video_max_frames, weights=None, *, init_idx=None, refill_idx=None,
                                         order=None):
    """compress_functions.py:301-386 ('fast_kmeans_ordered').  The reference's "fast" variant inlines the very same GEMM-form
    distance (A_2 + B_2.T - 2 * AB, :315-319 vs :196-200), draws the same RNG streams and orders the clusters by the same mean
    member index (:369 vs :278) as weighted_kmeans_ordered_feature — it only drops the unused `times` argument and the
    timing log — so it runs on the same kernels and returns the same four values."""
    return weighted_kmeans_ordered_feature(img_feature, video_max_frames, weights, None, init_idx=init_idx,
                                           refill_idx=refill_idx, order=order)


def _alternate(name, line):
    def fn(*a, **k):
        raise NotImplementedError(
            f"temporal method behind '{name}' (Flash-VStream-Qwen/models/compress_functions.py:{line}) is an alternate "
            f"compressor; only the default 'kmeans_ordered' path is built for sm_90a")
    fn.__name__ = name
    return fn


drop_feature = _alternate("drop_feature", 29)
merge_feature = _alternate("merge_feature", 67)
kmeans_feature = _alternate("kmeans_feature", 101)
weighted_kmeans_feature = _alternate("weighted_kmeans_feature", 139)
pca_weighted_kmeans_ordered_feature = _alternate("pca_weighted_kmeans_ordered_feature", 388)
# torchpca_kmeans_ordered (:479-577) projects every token onto the 32 eigenvectors of the 1280 x 1280 token covariance with the
# SMALLEST eigenvalues (eigh is ascending and the reference takes [:, :k]) before clustering.  That subspace is numerically
# degenerate noise: eigenvectors are defined up to sign and up to rotation inside (near-)equal eigenvalues, so two correct
# eigensolvers (LAPACK, cuSOLVER, any hand-written Jacobi) give different projections and different cluster assignments —
# there is no reference result to be identical to, which is the bar of this package.  Not built; the message says why.
torchpca_weighted_kmeans_ordered_feature = _alternate("torchpca_weighted_kmeans_ordered_feature", 479)
dbscan_feature = _alternate("dbscan_feature", 671)
gmm_feature = _alternate("gmm_feature", 704)
attention_feature = _alternate("attention_feature", 722)
k_drop_feature = _alternate("k_drop_feature", 580)
k_merge_feature = _alternate("k_merge_feature", 623)
