"""Drop-in mirror of flash_vstream.model.compress_functions (reference file, cited per function) running on the
sm_90a kernels.  Same names, argument meaning, return tuples and pass-through rules as the reference.

RNG: every default draw comes from `draws.GLOBAL`, the global generators the reference draws from (contract in
draws.py); explicit draws (init_idx= / refill_idx= / coins=) bypass it, which is what the parity tests do.
"""
from __future__ import annotations

from typing import Optional

import torch

from . import ops
from .draws import GLOBAL, DrawSource

MAX_ITER = 10      # compress_functions.py:133 (max_iter=10)
TOL = 1e-4         # compress_functions.py:133 (tol=1e-4)


def sync_rng():
    """Bring Python's `random` to the state the reference would have left: advance it by the refill draws the device
    consumed in the calls made so far.  Blocks on their (tiny) read-backs."""
    GLOBAL.settle()


def kmeans_draws(source: DrawSource, T: int, K: int, device):
    """(init_idx, refill_idx, Refills) for a weighted k-means over T rows, drawn from `source` as the reference draws them:
    torch.randperm on the rows' device (compress_functions.py:134) and random.randint refill candidates (:152)"""
    init_idx = source.randperm(T, device)[:K].to(torch.int32)
    refill_idx, refills = source.refill_candidates(T, MAX_ITER * K, device)
    return init_idx, refill_idx, refills


def weighted_kmeans_device(img_feature: torch.Tensor, video_max_frames: int, weights: Optional[torch.Tensor] = None,
                           init_idx: Optional[torch.Tensor] = None, refill_idx: Optional[torch.Tensor] = None):
    """Sync-free core: returns device tensors (centroids [T0,P,D], weights_sum [T0], labels int32 [T], info int32[4])
    or the pass-through tuple when T <= T0 (compress_functions.py:160-161)."""
    T, P, D = img_feature.shape
    T0 = video_max_frames
    if weights is None:
        weights_in = None
    else:
        weights_in = weights.to(img_feature.dtype)
    if T <= T0:
        w = weights if weights is not None else torch.ones(T, dtype=img_feature.dtype, device=img_feature.device)
        return img_feature, w, None, None
    refills = None
    if init_idx is None or refill_idx is None:
        init_idx, refill_idx, refills = kmeans_draws(GLOBAL, T, T0, img_feature.device)
    X = img_feature.reshape(T, P * D)
    C, wsum, labels, info = ops.weighted_kmeans(X, weights_in, init_idx, refill_idx, T0, MAX_ITER, TOL)
    if refills is not None:
        refills.consumed_from(info)
    return C.view(T0, P, D), wsum, labels, info


def weighted_kmeans_feature(img_feature, video_max_frames, weights=None, *, init_idx=None, refill_idx=None):
    """compress_functions.py:130-169.  Returns (reduced_feature [T0,P,D], weights [T0], [step_indices]).
    Building step_indices (nested Python lists, :166-169) needs the labels on the host: one small D2H copy."""
    T = img_feature.shape[0]
    T0 = video_max_frames
    feat, w, labels, _ = weighted_kmeans_device(img_feature, T0, weights, init_idx, refill_idx)
    if labels is None:
        return feat, w, [[[i] for i in range(T)]]
    lab = labels.cpu().tolist()
    sync_rng()
    step_indices = [[] for _ in range(T0)]
    for j, l in enumerate(lab):
        step_indices[l].append(j)
    return feat, w, [step_indices]


def attention_feature(img_feature, video_max_frames, attention_fn=None, update_ratio=0.2):
    """compress_functions.py:263-277: fold chunks of <= T0 new frames into the first T0 frames' memory."""
    T, P, D = img_feature.shape
    T0 = video_max_frames
    if T <= T0:
        return img_feature, None
    turing_memory = img_feature[:T0].reshape(T0 * P, D)
    for i in range(T0, T, T0):
        j = min(i + T0, T)
        new_feature = img_feature[i:j].reshape(-1, D)
        turing_memory = attention_fn(turing_memory, new_feature, update_ratio=update_ratio)
    return turing_memory.reshape(T0, P, D), None


def _coins(n, coins, device):
    """the random.randint(0, 1) flips of the drop variants (compress_functions.py:38, :194): exactly one per incoming frame,
    so drawing them ahead consumes Python's `random` stream exactly like the reference"""
    if coins is None:
        coins = GLOBAL.randints(0, 1, n)
    return torch.as_tensor(list(coins), dtype=torch.int32).to(device)


def drop_feature(img_feature, video_max_frames, img_similarity=None, *, coins=None):
    """compress_functions.py:19-54: keep T0 frames, dropping one of the most similar adjacent pair per incoming frame.
    One launch for the whole loop; returns (cur_feature [T0,P,D], cur_sim [T0-1], step_indices)."""
    T, P, D = img_feature.shape
    indices = [[i] for i in range(T)]
    T0 = video_max_frames
    if T <= T0:
        return img_feature, img_similarity, [indices]
    X = img_feature.reshape(T, P * D)
    kept, _, sim, pos = ops.alt_sequential(ops.ALT_DROP, X, T0, _coins(T - T0, coins, X.device), img_similarity)
    cur_indices = indices[:T0]
    step_indices = [cur_indices]
    for n, idx in enumerate(pos.cpu().tolist()):
        all_indices = cur_indices + [[T0 + n]]
        cur_indices = all_indices[:idx] + all_indices[idx + 1:]
        step_indices.append(cur_indices)
    return ops.gather_rows(img_feature, kept.long()), sim, step_indices


def merge_feature(img_feature, video_max_frames, img_similarity=None):
    """compress_functions.py:57-88: average the most similar adjacent pair per incoming frame."""
    T, P, D = img_feature.shape
    indices = [[i] for i in range(T)]
    T0 = video_max_frames
    if T <= T0:
        return img_feature, img_similarity, [indices]
    _, feat, sim, pos = ops.alt_sequential(ops.ALT_MERGE, img_feature.reshape(T, P * D), T0, None, img_similarity)
    cur_indices = indices[:T0]
    step_indices = [cur_indices]
    for n, idx in enumerate(pos.cpu().tolist()):
        all_indices = cur_indices + [[T0 + n]]
        all_indices[idx + 1] = all_indices[idx] + all_indices[idx + 1]
        cur_indices = all_indices[:idx] + all_indices[idx + 1:]
        step_indices.append(cur_indices)
    return feat.view(T0, P, D), sim, step_indices


def k_drop_feature(img_feature, video_max_frames, img_similarity=None, *, coins=None):
    """compress_functions.py:170-210: all-pairs cosine similarity; drop one frame of the most similar pair."""
    T, P, D = img_feature.shape
    indices = [[i] for i in range(T)]
    T0 = video_max_frames
    if T <= T0:
        return img_feature, img_similarity, [indices]
    X = img_feature.reshape(T, P * D)
    kept, _, _, pos = ops.alt_sequential(ops.ALT_KDROP, X, T0, _coins(T - T0, coins, X.device))
    cur_indices = indices[:T0]
    step_indices = [cur_indices]
    for n, idx in enumerate(pos.cpu().tolist()):
        all_indices = cur_indices + [[T0 + n]]
        cur_indices = all_indices[:idx] + all_indices[idx + 1:]
        step_indices.append(cur_indices)
    return ops.gather_rows(img_feature, kept.long()), None, step_indices


def k_merge_feature(img_feature, video_max_frames, img_similarity=None):
    """compress_functions.py:213-260: all-pairs cosine similarity; merge the most similar pair (left into right)."""
    T, P, D = img_feature.shape
    indices = [[i] for i in range(T)]
    T0 = video_max_frames
    if T <= T0:
        return img_feature, img_similarity, [indices]
    _, feat, sim, pos = ops.alt_sequential(ops.ALT_KMERGE, img_feature.reshape(T, P * D), T0)
    cur_indices = indices[:T0]
    step_indices = [cur_indices]
    for n, flat in enumerate(pos.cpu().tolist()):
        left, right = flat // (T0 + 1), flat % (T0 + 1)
        all_indices = cur_indices + [[T0 + n]]
        all_indices[right] = all_indices[left] + all_indices[right]
        cur_indices = all_indices[:left] + all_indices[left + 1:]
        step_indices.append(cur_indices)
    return feat.view(T0, P, D), sim, step_indices


def kmeans_feature(img_feature, video_max_frames, img_similarity=None, *, init_idx=None, refill_idx=None):
    """compress_functions.py:91-127: plain k-means (torch.cdist distances, unweighted means).  The reference draws
    torch.randperm(T) on the CPU generator (:93) and random.randint per empty cluster (:107)."""
    T, P, D = img_feature.shape
    T0 = video_max_frames
    if T <= T0:
        return img_feature, img_similarity, [[[i] for i in range(T)]]
    dev = img_feature.device
    if init_idx is None:
        init_idx = GLOBAL.randperm(T, "cpu")[:T0]
    if refill_idx is None:
        refill_dev, _ = GLOBAL.refill_candidates(T, MAX_ITER * T0, dev)
    else:
        refill = [int(v) for v in refill_idx]
        refill_dev = torch.tensor(refill + [0] * (MAX_ITER * T0 - len(refill)), dtype=torch.int32).to(dev)
    C, labels, info = ops.alt_kmeans(img_feature.reshape(T, P * D), torch.as_tensor(init_idx).to(device=dev, dtype=torch.int32),
                                     refill_dev, T0, MAX_ITER, TOL)
    lab = labels.cpu().tolist()
    if refill_idx is None:
        GLOBAL.consume(T, int(info[1]))                                  # what the reference would have drawn (:107)
    step_indices = [[j for j in range(T) if lab[j] == i] for i in range(T0)]
    return C.view(T0, P, D), img_similarity, [step_indices]
