"""Tensor-level wrappers over the fvs_qwen_* entry points of include/fvs_b200.h (no CPU path; torch = memory + streams)."""
from __future__ import annotations

import ctypes as C
from typing import NamedTuple, Optional

import torch

from .. import _lib as L
from ..host_tier import host_device_ptr, placement  # noqa: F401
from ..ops import _c, _chk_cuda

_ws_cache: dict = {}


def _workspace(need: int, dev, tag: str) -> torch.Tensor:
    key = (tag, dev.index, torch.cuda.current_stream().cuda_stream)
    ws = _ws_cache.get(key)
    if ws is None or ws.numel() < need:
        ws = torch.empty(max(need, 1 << 16), dtype=torch.uint8, device=dev)
        _ws_cache[key] = ws
    return ws


def temporal_pool(x: torch.Tensor, t: int, h: int, w: int) -> torch.Tensor:
    """FlashMemory.temporal_pool arithmetic (vstream_qwen2vl_model.py:113-142): [t*h*w, 1176] -> [t*(h/2)*(w/2), 1176]"""
    _chk_cuda(x)
    x = _c(x)
    assert x.shape == (t * h * w, 1176), f"x must be [t*h*w, 1176], got {tuple(x.shape)}"
    out = torch.empty(t * (h // 2) * (w // 2), 1176, dtype=x.dtype, device=x.device)
    L.check(L.load().fvs_qwen_temporal_pool(L.ptr(x), L.ptr(out), t, h, w, L.dtype_code(x.dtype), L.cur_stream()),
            "fvs_qwen_temporal_pool")
    return out


def unique_rows(X: torch.Tensor):
    """-> (uniq_idx int32 [T] (first n_unique entries valid), n_unique int32 [1]) on the device"""
    _chk_cuda(X)
    X = _c(X)
    T, PD = X.shape
    lib = L.load()
    ws = _workspace(lib.fvs_qwen_unique_workspace_bytes(T), X.device, "uniq")
    # zero-filled: the kernel defines the first n_unique entries, and a step that optimistically indexes the list before it
    # has read n_unique back (stream_state.py) must stay inside X whatever it finds in the rest
    idx = torch.zeros(T, dtype=torch.int32, device=X.device)
    n = torch.empty(1, dtype=torch.int32, device=X.device)
    L.check(lib.fvs_qwen_unique_rows(L.ptr(X), T, PD, L.dtype_code(X.dtype), L.ptr(idx), L.ptr(n), L.ptr(ws), ws.numel(),
                                     L.cur_stream()), "fvs_qwen_unique_rows")
    return idx, n


def kmeans_ordered(X: torch.Tensor, weights: torch.Tensor, uniq_idx: Optional[torch.Tensor], init_idx: torch.Tensor,
                   refill_idx: torch.Tensor, K: int, max_iter: int = 10, tol: float = 1e-4):
    """fp32 Lloyd loop on the device (no host synchronisation).  Returns (C fp32 [K, PD], wsum fp32 [K], labels int32 [T],
    info int32 [4])."""
    _chk_cuda(X, weights, uniq_idx, init_idx, refill_idx)
    X = _c(X)
    T, PD = X.shape
    dev = X.device
    lib = L.load()
    ws = _workspace(lib.fvs_qwen_kmeans_workspace_bytes(T, K, PD), dev, "km")
    assert weights.dtype == torch.float32 and init_idx.dtype == torch.int32 and refill_idx.dtype == torch.int32
    assert refill_idx.numel() >= max(1, max_iter * K)
    C = torch.empty(K, PD, dtype=torch.float32, device=dev)
    wsum = torch.empty(K, dtype=torch.float32, device=dev)
    labels = torch.empty(T, dtype=torch.int32, device=dev)
    info = torch.empty(4, dtype=torch.int32, device=dev)
    L.check(lib.fvs_qwen_kmeans(L.ptr(X), L.dtype_code(X.dtype), L.ptr(_c(weights)), L.ptr(uniq_idx), L.ptr(init_idx),
                                L.ptr(refill_idx), T, K, PD, max_iter, tol, L.ptr(C), L.ptr(wsum), L.ptr(labels),
                                L.ptr(info), L.ptr(ws), ws.numel(), L.cur_stream()), "fvs_qwen_kmeans")
    return C, wsum, labels, info


def kmeans_finalize(labels: torch.Tensor, wsum: torch.Tensor, order: Optional[torch.Tensor] = None):
    """device-side bookkeeping after kmeans_ordered (compress_functions.py:274-290): -> (sorted_idx int64 [K], timestamps
    fp32 [K], weights fp32 [K] — both already permuted —, flags int32 [1] = number of empty clusters).  order: the
    permutation to replay instead of the stable argsort of the timestamps."""
    _chk_cuda(labels, wsum, order)
    assert labels.dtype == torch.int32 and wsum.dtype == torch.float32 and (order is None or order.dtype == torch.int64)
    T, K = labels.numel(), wsum.numel()
    dev = labels.device
    sorted_idx = torch.empty(K, dtype=torch.int64, device=dev)
    ts = torch.empty(K, dtype=torch.float32, device=dev)
    w = torch.empty(K, dtype=torch.float32, device=dev)
    flags = torch.empty(1, dtype=torch.int32, device=dev)
    L.check(L.load().fvs_qwen_kmeans_finalize(L.ptr(_c(labels)), L.ptr(_c(wsum)), T, K, L.ptr(None if order is None else _c(order)),
                                              L.ptr(sorted_idx), L.ptr(ts), L.ptr(w), L.ptr(flags), L.cur_stream()),
            "fvs_qwen_kmeans_finalize")
    return sorted_idx, ts, w, flags


def gather_rows_cast(src: torch.Tensor, idx: torch.Tensor, dtype: torch.dtype, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _chk_cuda(src, idx, out)
    src = _c(src)
    assert src.dtype == torch.float32 and idx.dtype == torch.int64
    n, row = idx.numel(), src[0].numel()
    if out is None:
        out = torch.empty((n,) + tuple(src.shape[1:]), dtype=dtype, device=src.device)
    assert out.dtype == dtype and out.is_contiguous() and out.numel() == n * row
    L.check(L.load().fvs_gather_rows_cast(L.ptr(src), L.ptr(_c(idx)), L.ptr(out), n, row, L.dtype_code(dtype),
                                          L.cur_stream()), "fvs_gather_rows_cast")
    return out


# ---- the CSM chain of many streams (fvs_qwen_*_multi, DESIGN.md §3.17) ----------------------------------------------------
def mem_job(X: torch.Tensor, K: int, *, w=None, init_idx=None, refill_idx=None, max_iter: int = 10, tol: float = 1e-4,
            uniq_idx=None, n_unique=None, uniq_ws=None, C=None, wsum=None, labels=None, info=None, km_ws=None, order=None,
            sorted_idx=None, ts=None, w_sorted=None, flags=None, out=None) -> L.QwenMemJob:
    """one fvs_qwen_mem_job: X [T, PD] (contiguous, device) and whichever device tensors the calls it goes to read or write
    (workspaces: uint8 views of at least the fvs_qwen_*_workspace_bytes); the tensors must outlive the calls' enqueue"""
    _chk_cuda(X, w, init_idx, refill_idx, uniq_idx, n_unique, uniq_ws, C, wsum, labels, info, km_ws, order, sorted_idx, ts,
              w_sorted, flags, out)
    assert X.is_contiguous() and X.dim() == 2
    T, PD = X.shape
    nb = lambda t: 0 if t is None else t.numel() * t.element_size()
    return L.QwenMemJob(
        X=X.data_ptr(), T=T, K=int(K), PD=PD, x_dtype=L.dtype_code(X.dtype), w=L.ptr(w), init_idx=L.ptr(init_idx),
        refill_idx=L.ptr(refill_idx), max_iter=int(max_iter), tol=float(tol), uniq_idx=L.ptr(uniq_idx),
        n_unique=L.ptr(n_unique), uniq_workspace=L.ptr(uniq_ws), uniq_workspace_bytes=nb(uniq_ws), C=L.ptr(C),
        wsum=L.ptr(wsum), labels=L.ptr(labels), info=L.ptr(info), km_workspace=L.ptr(km_ws), km_workspace_bytes=nb(km_ws),
        order_in=L.ptr(order), sorted_idx=L.ptr(sorted_idx), ts=L.ptr(ts), w_sorted=L.ptr(w_sorted), flags=L.ptr(flags),
        out=L.ptr(out), out_dtype=L.dtype_code(out.dtype) if out is not None else 0)


def mem_jobs(jobs) -> "C.Array":
    return (L.QwenMemJob * len(jobs))(*jobs)


def mem_plan(jobs, budget: int = 0):
    """fvs_qwen_mem_plan (host arithmetic): -> (Lloyd-sweep blocks per job, launch group per job, number of groups)"""
    n = len(jobs)
    blocks, groups = (C.c_int32 * n)(), (C.c_int32 * n)()
    r = L.load().fvs_qwen_mem_plan(mem_jobs(jobs) if not isinstance(jobs, C.Array) else jobs, n, int(budget), blocks, groups)
    if r < 0:
        L.check(r, "fvs_qwen_mem_plan")
    return list(blocks), list(groups), r


def _multi(name: str, jobs, budget: int):
    arr = jobs if isinstance(jobs, C.Array) else mem_jobs(jobs)
    L.check(getattr(L.load(), name)(arr, len(arr), int(budget), L.cur_stream()), name)


def unique_rows_multi(jobs, budget: int = 0):
    """fvs_qwen_unique_rows per job (uniq_idx, n_unique, uniq_ws), in one launch pair per launch group"""
    _multi("fvs_qwen_unique_rows_multi", jobs, budget)


def kmeans_multi(jobs, budget: int = 0):
    """fvs_qwen_kmeans per job (C, wsum, labels, info, km_ws), each kernel of the Lloyd loop once per launch group"""
    _multi("fvs_qwen_kmeans_multi", jobs, budget)


def kmeans_finalize_multi(jobs, budget: int = 0):
    """fvs_qwen_kmeans_finalize per job (sorted_idx, ts, w_sorted, flags)"""
    _multi("fvs_qwen_kmeans_finalize_multi", jobs, budget)


def gather_rows_cast_multi(jobs, budget: int = 0):
    """fvs_gather_rows_cast(C, sorted_idx, out) per job"""
    _multi("fvs_gather_rows_cast_multi", jobs, budget)


def klarge_retrieve_multi(items, metric: str = "euclidean", want_dist: bool = False):
    """fvs_qwen_klarge_retrieve_multi: items = [(tem_x [st, PD], klarge_idx int64 [k <= 64], bank [t, PD])], every bank
    wholly in HBM and of one 16-bit dtype -> per item idx int64 [k] (and dist fp32 [k, t]), the bits klarge_retrieve
    gives each item alone"""
    code = {"euclidean": L.KLARGE_EUCLIDEAN, "cosine": L.KLARGE_COSINE}[metric]
    lib = L.load()
    keep, sizes = [], []
    for tem_x, klarge_idx, bank in items:
        _chk_cuda(tem_x, klarge_idx, bank)
        tem_x, klarge_idx, bank = _c(tem_x), _c(klarge_idx), _c(bank)
        assert klarge_idx.dtype == torch.int64 and tem_x.dtype == bank.dtype == items[0][2].dtype
        assert tem_x.shape[1] == bank.shape[1]
        keep.append((tem_x, klarge_idx, bank))
        sizes.append(_al(lib.fvs_qwen_klarge_workspace_bytes(klarge_idx.numel(), bank.shape[0], bank.shape[1])))
    dev = keep[0][0].device
    ws = _workspace(sum(sizes), dev, "klarge")         # klarge_retrieve's: a stream's bank may move between the two
    jobs, outs, o = [], [], 0
    for (tem_x, klarge_idx, bank), nb in zip(keep, sizes):
        k, t = klarge_idx.numel(), bank.shape[0]
        idx = torch.empty(k, dtype=torch.int64, device=dev)
        dist = torch.empty(k, t, dtype=torch.float32, device=dev) if want_dist else None
        jobs.append(L.QwenRetrieveJob(tem_x=tem_x.data_ptr(), klarge_idx=klarge_idx.data_ptr(), bank=bank.data_ptr(), k=k,
                                      t_total=t, n_dev=t, PD=bank.shape[1], idx_out=idx.data_ptr(), dist_out=L.ptr(dist),
                                      workspace=ws.data_ptr() + o, workspace_bytes=nb))
        outs.append((idx, dist) if want_dist else idx)
        o += nb
    arr = (L.QwenRetrieveJob * len(jobs))(*jobs)
    L.check(lib.fvs_qwen_klarge_retrieve_multi(arr, len(jobs), L.dtype_code(keep[0][2].dtype), code, L.cur_stream()),
            "fvs_qwen_klarge_retrieve_multi")
    return outs


def dam_gather_multi(calls):
    """fvs_qwen_dam_gather_multi: calls = [dict(picks, n_frames, prev (picks, x rows, merged rows or None) or None,
    fresh (plan int64, n_fresh, x rows, merged rows or None) or None, n_base (default: n_frames), dev_x, dev_merged,
    n_dev, chunks (device int64 table of the host chunks' mapped pointers), chunk_frames, x_frame_elems,
    merged_frame_elems, spa_x_out, merged_out, host_fetches (device int64 [1] counter or None))], one per stream, all
    outputs of one 16-bit dtype: spa_x_out[i] = x[picks[i]], merged_out[i] = merged[picks[i]], each read from the first
    of the previous DAM, the fresh rows, the device tier and the host chunks that holds the frame"""
    jobs, keep = [], []
    for a in calls:
        picks, prev, fresh, sx, mo = _c(a["picks"]), a.get("prev"), a.get("fresh"), a.get("spa_x_out"), a.get("merged_out")
        _chk_cuda(picks, a["dev_x"], a["dev_merged"], a["chunks"], sx, mo, a.get("host_fetches"))
        assert picks.dtype == torch.int64 and all(t is None or t.is_contiguous() for t in (sx, mo))
        m, pp, px, pm = 0, None, None, None
        if prev is not None and prev[0] is not None and prev[0].numel():
            pp, px, pm = prev
            _chk_cuda(pp, px, pm)
            pp = _c(pp)
            m = pp.numel()
        nf, fp, fx, fm = 0, None, None, None
        if fresh is not None and fresh[1]:
            fp, nf, fx, fm = fresh
            _chk_cuda(fp, fx, fm)
            assert fp.dtype == torch.int64 and fx.is_contiguous() and (fm is None or fm.is_contiguous())
        keep.append((picks, pp))
        jobs.append(L.QwenGatherJob(
            picks=picks.data_ptr(), n=picks.numel(), n_frames=int(a["n_frames"]), dev_x=L.ptr(a["dev_x"]),
            dev_merged=L.ptr(a["dev_merged"]), n_dev=int(a["n_dev"]), host_chunks=L.ptr(a["chunks"]),
            chunk_frames=int(a["chunk_frames"]), prev_picks=L.ptr(pp), m=m, prev_x=L.ptr(px), prev_merged=L.ptr(pm),
            x_frame_elems=int(a["x_frame_elems"]), merged_frame_elems=int(a["merged_frame_elems"]), spa_x_out=L.ptr(sx),
            merged_out=L.ptr(mo), host_fetches=L.ptr(a.get("host_fetches")), fresh_frames=L.ptr(fp), n_fresh=int(nf),
            fresh_x=L.ptr(fx), fresh_merged=L.ptr(fm), n_base=int(a.get("n_base", a["n_frames"]))))
    out0 = calls[0].get("spa_x_out") if calls[0].get("spa_x_out") is not None else calls[0].get("merged_out")
    arr = (L.QwenGatherJob * len(jobs))(*jobs)
    L.check(L.load().fvs_qwen_dam_gather_multi(arr, len(jobs), L.dtype_code(out0.dtype), L.cur_stream()),
            "fvs_qwen_dam_gather_multi")


def pick_plan_multi(jobs):
    """fvs_qwen_pick_plan_multi: jobs = [(picks int64 [n] or None for frames 0..n-1, n, frames uint8 [>= n_frames],
    n_frames, plan int64 [>= n], count address[, stored, prev_picks int64 [m] or None, re_encodes int64 [1] or None])],
    count address = an int: the mapped address of an int32 slot of pinned memory (host_device_ptr) or of a device int32.
    Plans the picks whose frame byte is below `stored` (1, the default: a bank's "not yet encoded"; 2 without a bank:
    not in the base bank) and that prev_picks does not hold, and sets the planned frames' bytes to 1.  A job of a
    stream with a bank gives the first six items only."""
    arr, keep = [], []
    for picks, n, frames, n_frames, plan, count, *rest in jobs:
        stored, prev, re_enc = rest or (1, None, None)
        _chk_cuda(picks, frames, prev, plan, re_enc)
        picks, prev = None if picks is None else _c(picks), None if prev is None or prev.numel() == 0 else _c(prev)
        assert picks is None or (picks.dtype == torch.int64 and picks.numel() >= n)
        assert frames.dtype == torch.uint8 and plan.dtype == torch.int64 and plan.numel() >= n
        assert prev is None or prev.dtype == torch.int64
        keep.append((picks, prev))
        arr.append(L.QwenPickPlanJob(picks=L.ptr(picks), n=int(n), n_frames=int(n_frames), frames=frames.data_ptr(),
                                     plan=plan.data_ptr(), count=int(count), prev_picks=L.ptr(prev),
                                     m=0 if prev is None else prev.numel(), re_encodes=L.ptr(re_enc), stored=int(stored)))
    L.check(L.load().fvs_qwen_pick_plan_multi((L.QwenPickPlanJob * len(arr))(*arr), len(arr), L.cur_stream()),
            "fvs_qwen_pick_plan_multi")


def pixel_gather_multi(jobs):
    """fvs_qwen_pixel_gather_multi: jobs = [(plan int64, n, n_frames, base, chunk table (device int64), chunk_frames,
    out [n, ...] of 16-bit rows, frame_elems, value table fp32 [3, 256] or None)], all outputs of one dtype and all jobs
    of one kind: chunks of rows of out's dtype (no table), or of uint8 codes decoded through the table in the same pass"""
    arr = []
    for plan, n, n_frames, base, chunks, cf, out, fe, table in jobs:
        _chk_cuda(plan, chunks, out, table)
        assert plan.dtype == torch.int64 and chunks.dtype == torch.int64 and out.is_contiguous() and out.numel() == n * fe
        assert table is None or (table.dtype == torch.float32 and table.is_contiguous() and table.numel() == 3 * 256)
        arr.append(L.QwenPixelJob(plan=plan.data_ptr(), n=int(n), n_frames=int(n_frames), base=int(base),
                                  host_chunks=chunks.data_ptr(), chunk_frames=int(cf), frame_elems=int(fe),
                                  out=out.data_ptr(), table=L.ptr(table)))
    L.check(L.load().fvs_qwen_pixel_gather_multi((L.QwenPixelJob * len(arr))(*arr), len(arr), L.dtype_code(jobs[0][6].dtype),
                                                 L.cur_stream()), "fvs_qwen_pixel_gather_multi")


def pixel_decode(codes: torch.Tensor, table: torch.Tensor, dtype: torch.dtype,
                 out: Optional[torch.Tensor] = None) -> torch.Tensor:
    """fvs_qwen_pixel_decode: codes uint8 [rows, 1176] -> dtype(table[column // 392][code]) [rows, 1176] (f16 / bf16),
    the bits of casting the fp32 rows the codes stand for (DESIGN.md §3.20)"""
    _chk_cuda(codes, table, out)
    codes, table = _c(codes), _c(table)
    assert codes.dtype == torch.uint8 and codes.dim() == 2 and codes.shape[1] == 1176, f"codes {codes.dtype} {tuple(codes.shape)}"
    assert table.dtype == torch.float32 and table.numel() == 3 * 256
    if out is None:
        out = torch.empty(codes.shape, dtype=dtype, device=codes.device)
    assert out.dtype == dtype and out.is_contiguous() and out.shape == codes.shape
    L.check(L.load().fvs_qwen_pixel_decode(codes.data_ptr(), codes.shape[0], table.data_ptr(), L.dtype_code(dtype),
                                           out.data_ptr(), L.cur_stream()), "fvs_qwen_pixel_decode")
    return out


def bank_scatter_multi(jobs):
    """fvs_qwen_bank_scatter_multi: jobs = [dict(plan, n, n_frames, x_rows, merged_rows, dev_x, dev_merged, n_dev, chunks,
    chunk_frames, x_frame_elems, merged_frame_elems)], every row tensor of one 16-bit dtype"""
    arr = []
    for a in jobs:
        _chk_cuda(a["plan"], a["x_rows"], a["merged_rows"], a["dev_x"], a["dev_merged"], a["chunks"])
        assert a["plan"].dtype == torch.int64 and a["x_rows"].is_contiguous()
        assert a["merged_rows"] is None or a["merged_rows"].is_contiguous()
        arr.append(L.QwenScatterJob(
            plan=a["plan"].data_ptr(), n=int(a["n"]), n_frames=int(a["n_frames"]), x_rows=a["x_rows"].data_ptr(),
            merged_rows=L.ptr(a["merged_rows"]), dev_x=L.ptr(a["dev_x"]), dev_merged=L.ptr(a["dev_merged"]),
            n_dev=int(a["n_dev"]), host_chunks=L.ptr(a["chunks"]), chunk_frames=int(a["chunk_frames"]),
            x_frame_elems=int(a["x_frame_elems"]), merged_frame_elems=int(a["merged_frame_elems"])))
    L.check(L.load().fvs_qwen_bank_scatter_multi((L.QwenScatterJob * len(arr))(*arr), len(arr),
                                                 L.dtype_code(jobs[0]["x_rows"].dtype), L.cur_stream()),
            "fvs_qwen_bank_scatter_multi")


def mem_workspace_bytes(T: int, K: int, PD: int) -> int:
    """bytes one job of the CSM chain needs besides its outputs: fp32 centroids, unique-rows and k-means workspaces"""
    lib = L.load()
    return _al(K * PD * 4) + _al(lib.fvs_qwen_unique_workspace_bytes(T)) + _al(lib.fvs_qwen_kmeans_workspace_bytes(T, K, PD))


def _al(v: int) -> int:
    return (v + 255) & ~255


class TieredBank(NamedTuple):
    """A bank of t_total rows of PD 16-bit elements in two tiers (DESIGN.md §3.13): rows [0, n_dev) are `dev` (HBM,
    [n_dev, PD], None when n_dev is 0); row n_dev + c * chunk_frames + r is row r of the pinned host chunk whose mapped
    device pointer (host_device_ptr) is chunks[c]."""
    dev: Optional[torch.Tensor]
    n_dev: int
    chunks: tuple
    chunk_frames: int
    t_total: int
    dtype: torch.dtype
    device: torch.device


def klarge_plan(t_total: int, n_dev: int, chunk_frames: int):
    """the row ranges a tiered klarge sweep launches over, as (chunk, t_first, rows): chunk -1 is the device rows (every
    row when n_dev >= t_total), chunk c >= 0 the c-th host chunk"""
    return [(c, s, cnt) for c, _, s, cnt in placement(0, t_total, n_dev, chunk_frames)]


def klarge_retrieve(tem_x: torch.Tensor, klarge_idx: torch.Tensor, bank, want_dist: bool = False,
                    metric: str = "euclidean"):
    """tem_x [st, PD], klarge_idx int64 [k], bank [t, PD] (16-bit) or a TieredBank of t rows -> idx int64 [k] (and the
    rounded distances — or, with metric="cosine" ('klarge_retrieve_cos'), similarities — fp32 [k, t]).  A tiered bank's
    host rows are read in place over PCIe (once per sweep; the cosine metric sweeps twice); the results are the bits of the
    same rows in HBM."""
    code = {"euclidean": L.KLARGE_EUCLIDEAN, "cosine": L.KLARGE_COSINE}[metric]
    tiered = isinstance(bank, TieredBank)
    rows = bank.dev if tiered else bank
    _chk_cuda(tem_x, klarge_idx, rows)
    tem_x, klarge_idx, rows = _c(tem_x), _c(klarge_idx), None if rows is None else _c(rows)
    assert klarge_idx.dtype == torch.int64 and tem_x.dtype == bank.dtype and (rows is None or tem_x.shape[1] == rows.shape[1])
    assert not tiered or (0 if rows is None else rows.shape[0]) == bank.n_dev
    k, t, PD = klarge_idx.numel(), bank.t_total if tiered else rows.shape[0], tem_x.shape[1]
    if k > 64:   # the kernel keeps <= 64 centroid slices in shared memory: sweep the bank once per group of 64
        parts = [klarge_retrieve(tem_x, klarge_idx[i:i + 64], bank, want_dist, metric) for i in range(0, k, 64)]
        return (torch.cat([p[0] for p in parts]), torch.cat([p[1] for p in parts])) if want_dist else torch.cat(parts)
    lib = L.load()
    dev = tem_x.device
    ws = _workspace(lib.fvs_qwen_klarge_workspace_bytes(k, t, PD), dev, "klarge")
    idx = torch.empty(k, dtype=torch.int64, device=dev)
    dist = torch.empty(k, t, dtype=torch.float32, device=dev) if want_dist else None
    if not tiered:
        L.check(lib.fvs_qwen_klarge_retrieve(L.ptr(tem_x), L.ptr(klarge_idx), L.ptr(rows), k, t, PD, L.dtype_code(rows.dtype),
                                             code, L.ptr(idx), L.ptr(dist), L.ptr(ws), ws.numel(), L.cur_stream()),
                "fvs_qwen_klarge_retrieve")
        return (idx, dist) if want_dist else idx
    n_chunks = sum(1 for c, _, _ in klarge_plan(t, bank.n_dev, bank.chunk_frames) if c >= 0)
    assert len(bank.chunks) >= n_chunks, f"a bank of {t} rows needs {n_chunks} host chunks, got {len(bank.chunks)}"
    table = (C.c_void_p * n_chunks)(*bank.chunks[:n_chunks]) if n_chunks else None     # host array, read at launch
    L.check(lib.fvs_qwen_klarge_retrieve_tiered(L.ptr(tem_x), L.ptr(klarge_idx), L.ptr(rows), int(bank.n_dev), table,
                                                int(bank.chunk_frames), k, t, PD,
                                                L.dtype_code(bank.dtype), code, L.ptr(idx), L.ptr(dist), L.ptr(ws),
                                                ws.numel(), L.cur_stream()), "fvs_qwen_klarge_retrieve_tiered")
    return (idx, dist) if want_dist else idx


def am_rope(spa_positions: torch.Tensor, spa_grid, tem_positions: torch.Tensor, tem_grid, visual_start_id: int,
            device) -> torch.Tensor:
    """-> [3, n] int64; *_grid = (t, h, w) in LLM tokens (h, w already halved)"""
    n = spa_grid[0] * spa_grid[1] * spa_grid[2] + tem_grid[0] * tem_grid[1] * tem_grid[2]
    out = torch.empty(3, n, dtype=torch.int64, device=device)
    if n == 0:
        return out
    sp = _c(spa_positions) if spa_grid[0] > 0 else None
    tp = _c(tem_positions) if tem_grid[0] > 0 else None
    _chk_cuda(sp, tp)
    assert (sp is None or sp.dtype == torch.int64) and (tp is None or tp.dtype == torch.int64)
    L.check(L.load().fvs_qwen_am_rope(L.ptr(sp), *spa_grid, L.ptr(tp), *tem_grid, int(visual_start_id), L.ptr(out),
                                      L.cur_stream()), "fvs_qwen_am_rope")
    return out
