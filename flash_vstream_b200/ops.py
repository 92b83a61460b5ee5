"""Tensor-level wrappers over the C ABI (include/fvs_b200.h).  torch is used only for device memory and streams;
every function here ends in a call into libfvs_b200.so and raises if that is impossible (no CPU fallback)."""
from __future__ import annotations

import ctypes as C
import math
from typing import Optional

import torch

from . import _lib as L
from . import host_tier as HT


def _chk_cuda(*ts):
    for t in ts:
        if t is not None and not t.is_cuda:
            raise L.FvsError("flash_vstream_b200 has no CPU path: tensors must live on a CUDA device")


def _c(t: Optional[torch.Tensor]) -> Optional[torch.Tensor]:
    return None if t is None else (t if t.is_contiguous() else t.contiguous())


def require_inference(*tensors, what="flash_vstream_b200"):
    """The kernels write into torch.empty outputs through the C ABI: there is no autograd graph behind them.  Training
    through an install()'d process would silently detach the projector / attention model, so refuse instead."""
    if torch.is_grad_enabled():
        for t in tensors:
            if t is not None and t.requires_grad:
                raise RuntimeError(f"{what} is inference-only (no autograd): call it under torch.no_grad() / "
                                   f"torch.inference_mode(), or keep the reference's own module for training")


# --------------------------------------------------------------------------------------------- ViT building blocks
def linear(A, W, bias=None, *, epilogue=L.EPI_BIAS, aux=None, aux_period=0, out=None):
    """out = epilogue(A @ W^T); see fvs_linear in include/fvs_b200.h"""
    _chk_cuda(A, W, bias, aux, out)
    A, W = _c(A), _c(W)
    M, K = A.shape
    N = W.shape[0]
    if out is None:
        out = torch.empty(M, N, dtype=torch.float32 if epilogue == L.EPI_BIAS_RESIDUAL_F32 else A.dtype, device=A.device)
    rc = L.load().fvs_linear(L.ptr(A), L.ptr(W), L.ptr(_c(bias)), L.ptr(aux), L.ptr(out), M, N, K, A.stride(0),
                             out.stride(0), epilogue, aux_period, L.dtype_code(A.dtype), L.cur_stream())
    L.check(rc, "fvs_linear")
    return out


def attention(qkv, frames, tokens, heads, scale=0.125, out=None):
    _chk_cuda(qkv, out)
    qkv = _c(qkv)
    if out is None:
        out = torch.empty(frames * tokens, heads * 64, dtype=qkv.dtype, device=qkv.device)
    L.check(L.load().fvs_attention(L.ptr(qkv), L.ptr(out), frames, tokens, heads, scale, L.dtype_code(qkv.dtype),
                                   L.cur_stream()), "fvs_attention")
    return out


def split_heads_80(t: torch.Tensor, heads: int, sections: int) -> torch.Tensor:
    """[rows, sections*heads*80] in the natural (section, head, dim) order -> the [main | extra] column layout of
    fvs_attention80 (index plumbing; the engine gets this layout for free from permuted weights)"""
    rows = t.shape[0]
    v = t.view(rows, sections, heads, 80)
    return torch.cat([v[..., :64].reshape(rows, -1), v[..., 64:].reshape(rows, -1)], dim=1).contiguous()


def merge_heads_80(t: torch.Tensor, heads: int, sections: int = 1) -> torch.Tensor:
    """inverse of split_heads_80"""
    rows = t.shape[0]
    main = t[:, : sections * heads * 64].view(rows, sections, heads, 64)
    extra = t[:, sections * heads * 64:].view(rows, sections, heads, 16)
    return torch.cat([main, extra], dim=-1).reshape(rows, -1).contiguous()


def attention80(qkv, frames, tokens, heads, scale=80 ** -0.5, out=None):
    """head_dim-80 attention over the [main | extra] layout (see fvs_attention80)"""
    _chk_cuda(qkv, out)
    qkv = _c(qkv)
    if out is None:
        out = torch.empty(frames * tokens, heads * 80, dtype=qkv.dtype, device=qkv.device)
    L.check(L.load().fvs_attention80(L.ptr(qkv), L.ptr(out), frames, tokens, heads, scale, L.dtype_code(qkv.dtype),
                                     L.cur_stream()), "fvs_attention80")
    return out


def layernorm(x, gamma, beta, eps=1e-5, out=None, out_dtype=None):
    """x may be f16/bf16 (same as gamma) or f32; the output dtype defaults to gamma's"""
    _chk_cuda(x, gamma, beta, out)
    x = _c(x)
    rows, dim = x.shape
    if out is None:
        out = torch.empty(rows, dim, dtype=out_dtype or gamma.dtype, device=x.device)
    L.check(L.load().fvs_layernorm(L.ptr(x), L.ptr(_c(gamma)), L.ptr(_c(beta)), L.ptr(out), rows, dim, eps,
                                   L.dtype_code(gamma.dtype), L.dtype_code(x.dtype), L.dtype_code(out.dtype),
                                   L.cur_stream()), "fvs_layernorm")
    return out


class VitEncoder:
    """fvs_vit_* handle: ViT-L/14 frame encoder (CLIPVisionTower.forward + feature_select, clip_encoder.py:31-53).

    `weights` uses the layout of oracle-free plain dicts: patch_w [H,3,P,P], class_emb [H], pos_emb [T,H],
    pre_ln_w/b, layers = list of {ln1_w, ln1_b, q_w,q_b,k_w,k_b,v_w,v_b, o_w,o_b, ln2_w,ln2_b, fc1_w,fc1_b, fc2_w,fc2_b}
    (exactly the tensors of transformers.CLIPVisionModel).  Only the first `layers_run` layers are kept."""

    def __init__(self, weights: dict, *, image_size=336, patch_size=14, heads=16, layers_run=23, ln_eps=1e-5,
                 dtype=torch.float16, device="cuda", max_batch=32, keep_cls=False):
        dev = torch.device(device)
        if dev.type != "cuda":
            raise L.FvsError("VitEncoder needs a CUDA device (no CPU fallback)")
        self.lib = L.load()
        self._ctor = dict(image_size=image_size, patch_size=patch_size, heads=heads, layers_run=layers_run, ln_eps=ln_eps,
                          dtype=dtype, device=str(dev), max_batch=max_batch, keep_cls=keep_cls)
        self.dtype, self.device = dtype, dev
        cv = lambda t: t.detach().to(device=dev, dtype=dtype).contiguous()
        H = weights["class_emb"].numel()
        self.hidden, self.heads, self.patch, self.image = H, heads, patch_size, image_size
        self.grid = image_size // patch_size
        self.tokens = self.grid ** 2 + 1
        self.mlp = weights["layers"][0]["fc1_w"].shape[0] if weights["layers"] else 4 * H
        self.layers_run = layers_run
        assert len(weights["layers"]) >= layers_run, "not enough encoder layers in the weight dict"
        self._keep = []  # device tensors referenced by raw pointers inside the handle
        k = lambda t: (self._keep.append(cv(t)), self._keep[-1])[1]
        self._w = {"class_emb": None, "layers": []}     # the prepared device tensors in weight-dict form (for pickling)
        self.patch_w = k(weights["patch_w"].reshape(H, -1))
        self.class_emb, self.pos_emb = k(weights["class_emb"]), k(weights["pos_emb"])
        self.pre_w, self.pre_b = k(weights["pre_ln_w"]), k(weights["pre_ln_b"])
        arr = (L.VitLayerWeights * max(layers_run, 1))()
        for i in range(layers_run):
            p = weights["layers"][i]
            qkv_w = k(p["qkv_w"] if "qkv_w" in p else torch.cat([p["q_w"], p["k_w"], p["v_w"]], dim=0))
            qkv_b = k(p["qkv_b"] if "qkv_b" in p else torch.cat([p["q_b"], p["k_b"], p["v_b"]], dim=0))
            vals = dict(ln1_w=k(p["ln1_w"]), ln1_b=k(p["ln1_b"]), qkv_w=qkv_w, qkv_b=qkv_b, o_w=k(p["o_w"]), o_b=k(p["o_b"]),
                        ln2_w=k(p["ln2_w"]), ln2_b=k(p["ln2_b"]), fc1_w=k(p["fc1_w"]), fc1_b=k(p["fc1_b"]),
                        fc2_w=k(p["fc2_w"]), fc2_b=k(p["fc2_b"]))
            for name, t in vals.items():
                setattr(arr[i], name, t.data_ptr())
            self._w["layers"].append(vals)
        self.keep_cls = bool(keep_cls)   # select_feature 'cls_patch' (clip_encoder.py:37): the CLS row stays in the output
        cfg = L.VitConfig(image_size, patch_size, H, heads, self.mlp, layers_run, ln_eps, L.dtype_code(dtype), int(self.keep_cls))
        w = L.VitWeights(self.patch_w.data_ptr(), self.class_emb.data_ptr(), self.pos_emb.data_ptr(),
                         self.pre_w.data_ptr(), self.pre_b.data_ptr(), arr)
        self._w.update(patch_w=self.patch_w, class_emb=self.class_emb, pos_emb=self.pos_emb, pre_ln_w=self.pre_w,
                       pre_ln_b=self.pre_b)
        self._h = C.c_void_p()
        with torch.cuda.device(dev):
            L.check(self.lib.fvs_vit_create(C.byref(self._h), C.byref(cfg), C.byref(w), L.cur_stream()), "fvs_vit_create")
        self.max_batch = 0
        self._ws = None
        self.reserve(max_batch)

    # The reference's serve CLI pickles the whole model into its memory-manager process (spawn start method,
    # cli_video_stream.py:210,253).  ctypes handles cannot travel; the prepared weights can (torch.multiprocessing shares CUDA
    # tensors by IPC handle, plain pickle copies them), and the engine is rebuilt from them on the other side.
    def __getstate__(self):
        return {"ctor": self._ctor, "weights": self._w}

    def __setstate__(self, st):
        self.__init__(st["weights"], **{**st["ctor"], "dtype": st["ctor"]["dtype"]})

    def reserve(self, max_batch: int):
        if max_batch > self.max_batch:
            n = self.lib.fvs_vit_workspace_bytes(self._h, max_batch)
            self._ws = torch.empty(n, dtype=torch.uint8, device=self.device)
            self.max_batch = max_batch

    def encode(self, pixels: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
        """pixels [B,3,S,S] -> [B, grid^2 (+1 with keep_cls), hidden]; processed in micro-batches of `max_batch` frames."""
        _chk_cuda(pixels, out)
        if pixels.dtype != self.dtype:
            pixels = pixels.to(self.dtype)
        pixels = _c(pixels)
        B = pixels.shape[0]
        assert tuple(pixels.shape[1:]) == (3, self.image, self.image), pixels.shape
        if out is None:
            out = torch.empty(B, self.tokens - (0 if self.keep_cls else 1), self.hidden, dtype=self.dtype, device=self.device)
        L.check(self.lib.fvs_vit_encode(self._h, L.ptr(pixels), L.ptr(out), B, L.ptr(self._ws), self._ws.numel(),
                                        L.cur_stream()), "fvs_vit_encode")
        return out

    __call__ = encode

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self.lib.fvs_vit_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass


# --------------------------------------------------------------------------------------------- consolidation
def spatial_pool(feat: torch.Tensor, target: int) -> torch.Tensor:
    """compress_spatial_features(compress_type='mean') arithmetic (vstream_arch.py:193-212) for [T, g*g, D] f16."""
    _chk_cuda(feat)
    feat = _c(feat)
    T, P, D = feat.shape
    g = round(math.sqrt(P))
    assert g * g == P, f"For ViT feature map, {g}*{g}={g**2} != {P}"
    if g == target:
        return feat
    k = g // target
    c = g // k
    if c * k != g:
        raise NotImplementedError(f"pooling {g}x{g} -> {target}x{target} with a remainder is not supported")
    out = torch.empty(T, c * c, D, dtype=feat.dtype, device=feat.device)
    L.check(L.load().fvs_spatial_pool(L.ptr(feat), L.ptr(out), T, g, c, D, L.dtype_code(feat.dtype), L.cur_stream()),
            "fvs_spatial_pool")
    return out


def spatial_pool3(feat: torch.Tensor, a: int = 8, b: int = 4):
    """One pass over [T, g*g, D]: level a, then b and 1 pooled from the rounded level a (vstream_arch.py:644,659-662)."""
    _chk_cuda(feat)
    feat = _c(feat)
    T, P, D = feat.shape
    g = round(math.sqrt(P))
    oa = torch.empty(T, a * a, D, dtype=feat.dtype, device=feat.device)
    ob = torch.empty(T, b * b, D, dtype=feat.dtype, device=feat.device)
    oc = torch.empty(T, 1, D, dtype=feat.dtype, device=feat.device)
    L.check(L.load().fvs_spatial_pool3(L.ptr(feat), L.ptr(oa), L.ptr(ob), L.ptr(oc), T, g, a, b, D,
                                       L.dtype_code(feat.dtype), L.cur_stream()), "fvs_spatial_pool3")
    return oa, ob, oc


_km_ws_cache: dict = {}


def weighted_kmeans(X: torch.Tensor, weights: Optional[torch.Tensor], init_idx: torch.Tensor, refill_idx: torch.Tensor,
                    K: int, max_iter: int = 10, tol: float = 1e-4):
    """Device-side Lloyd loop (no host synchronisation).  X [T,PD] f16; init_idx int32 [K]; refill_idx int32
    [max_iter*K].  Returns (C [K,PD], wsum [K], labels int32 [T], info int32 [4] = exit_step, refills, converged, 0)."""
    _chk_cuda(X, weights, init_idx, refill_idx)
    X = _c(X)
    T, PD = X.shape
    dev = X.device
    lib = L.load()
    need = lib.fvs_kmeans_workspace_bytes(T, K, PD)
    key = (dev.index, torch.cuda.current_stream().cuda_stream)
    ws = _km_ws_cache.get(key)
    if ws is None or ws.numel() < need:
        ws = torch.empty(max(need, 1 << 20), dtype=torch.uint8, device=dev)
        _km_ws_cache[key] = ws
    Cout = torch.empty(K, PD, dtype=X.dtype, device=dev)
    wsum = torch.empty(K, dtype=X.dtype, device=dev)
    labels = torch.empty(T, dtype=torch.int32, device=dev)
    info = torch.empty(4, dtype=torch.int32, device=dev)
    assert init_idx.dtype == torch.int32 and refill_idx.dtype == torch.int32
    assert refill_idx.numel() >= max_iter * K
    L.check(lib.fvs_weighted_kmeans(L.ptr(X), L.ptr(_c(weights)), L.ptr(init_idx), L.ptr(refill_idx), T, K, PD, max_iter,
                                    tol, L.ptr(Cout), L.ptr(wsum), L.ptr(labels), L.ptr(info), L.ptr(ws), ws.numel(),
                                    L.dtype_code(X.dtype), L.cur_stream()), "fvs_weighted_kmeans")
    return Cout, wsum, labels, info


def abstract_update(M, F, Wq, bq, Wk, bk, ratio=0.2, out=None):
    _chk_cuda(M, F, Wq, bq, Wk, bk)
    M, F = _c(M), _c(F)
    T1, D = M.shape
    T2 = F.shape[0]
    H = Wq.shape[0]
    if out is None:
        out = torch.empty_like(M)
    L.check(L.load().fvs_abstract_update(L.ptr(M), L.ptr(F), L.ptr(_c(Wq)), L.ptr(_c(bq)), L.ptr(_c(Wk)), L.ptr(_c(bk)),
                                         L.ptr(out), T1, T2, D, H, ratio, L.dtype_code(M.dtype), L.cur_stream()),
            "fvs_abstract_update")
    return out


def argsort_desc(w: torch.Tensor) -> torch.Tensor:
    """stable descending argsort of a 1-D weight vector.  Anything else is refused: the flattened order of a [n, n] matrix
    holds indices up to n² - 1, which key_retrieve would read as rows of the long memory."""
    if not isinstance(w, torch.Tensor):
        raise TypeError(f"argsort_desc: the weight must be a tensor, got {type(w).__name__}")
    if w.dim() != 1:
        raise ValueError(f"argsort_desc: the weight must be 1-D, got shape {tuple(w.shape)}")
    _chk_cuda(w)
    w = _c(w)
    out = torch.empty(w.numel(), dtype=torch.int64, device=w.device)
    L.check(L.load().fvs_argsort_desc(L.ptr(w), w.numel(), L.ptr(out), L.dtype_code(w.dtype), L.cur_stream()),
            "fvs_argsort_desc")
    return out


def key_retrieve(long_mem: torch.Tensor, order: torch.Tensor, key_len: int = 3) -> torch.Tensor:
    _chk_cuda(long_mem, order)
    long_mem = _c(long_mem)
    Lr, P, D = long_mem.shape
    kl = min(key_len, Lr)
    out = torch.empty(kl, dtype=torch.int64, device=long_mem.device)
    L.check(L.load().fvs_key_retrieve(L.ptr(long_mem), L.ptr(_c(order)), Lr, P, D, kl, L.ptr(out),
                                      L.dtype_code(long_mem.dtype), L.cur_stream()), "fvs_key_retrieve")
    return out


def gather_rows(src: torch.Tensor, idx: torch.Tensor, out: Optional[torch.Tensor] = None) -> torch.Tensor:
    _chk_cuda(src, idx, out)
    src = _c(src)
    n = idx.numel()
    row = src[0].numel()
    if out is None:
        out = torch.empty((n,) + tuple(src.shape[1:]), dtype=src.dtype, device=src.device)
    assert out.dtype == src.dtype and out.is_contiguous() and out.numel() == n * row
    L.check(L.load().fvs_gather_rows(L.ptr(src), L.ptr(_c(idx)), L.ptr(out), n, row, L.dtype_code(src.dtype),
                                     L.cur_stream()), "fvs_gather_rows")
    return out


# --------------------------------------------------------------------------------------------- streaming step on a bank
def star_config(cfg) -> "L.StarConfig":
    """the L.StarConfig of a dict of the reference's STAR knobs (an L.StarConfig passes through)"""
    if isinstance(cfg, L.StarConfig):
        return cfg
    return L.StarConfig(int(cfg["D"]), int(cfg["grid"]), int(cfg["cur_size"]), int(cfg["long_size"]), int(cfg["long_len"]),
                        int(cfg["tur_len"]), int(cfg["cur_len"]), int(cfg.get("key_len", 3)), int(cfg["ntm_dim"]),
                        float(cfg["ratio"]))


def min_device_frames(cfg, chunk_cap: int) -> int:
    """the smallest device_frames of a bank with this STAR config (dict or L.StarConfig) and chunk_cap: the long working
    set's rows of fvs_bank_rows, max(long_len, chunk_cap) + chunk_cap — a key frame is frames[i] for such a row i"""
    lw = C.c_int64()
    L.check(L.load().fvs_bank_rows(C.byref(star_config(cfg)), int(chunk_cap), C.byref(lw), None, None), "fvs_bank_rows")
    return lw.value


def device_window(cfg, chunk_cap: int, device_frames, who: str = "device_frames") -> Optional[int]:
    """device_frames validated for a bank of this config: None or an integer >= min_device_frames; ValueError otherwise"""
    v = HT.check_device_frames(device_frames, who)
    if v is not None and v < (m := min_device_frames(cfg, chunk_cap)):
        raise ValueError(f"{who} {v} < {m}: a LLaVA bank keeps at least its long working set's rows (max(long_len, "
                         f"chunk_cap) + chunk_cap) of frames in HBM, since every key frame is read from there")
    return v


class StreamBank:
    """One stream's persistent Flash memory on the GPU (fvs_bank + fvs_stream_step, include/fvs_b200.h): the state of
    embed_video_streaming (vstream_arch.py:611-697) — [cur, long, Turing, frame buffer] — lives in caller-owned device
    tensors that a step updates in place; the LLM's visual prefix [Turing | long | key | current] (vstream_arch.py:483) is
    `self.prefix()` — a view, never a concatenation.  All shapes of a step are host-known, so nothing here synchronises.

    cfg: dict with the reference's knobs (D, grid, cur_size, long_size, long_len, tur_len, cur_len, key_len, ntm_dim,
    ratio); ntm: (q_w, q_b, k_w, k_b) f16 CUDA tensors of NeuralTuringMachine.q_proj / k_proj.

    device_frames: None (default: the whole frame buffer in HBM, grown as needed) or N >= min_device_frames(): frames
    [0, N) stay in `frames`, which also holds a slot of chunk_cap rows for the clip's frames at or past N and never grows;
    after each step those frames are copied (asynchronously, on the step's stream) to pinned host chunks.  A step reads
    only key frames (below N) and the clip's own frames, so the bank's bits do not depend on the cap (DESIGN.md §3.14)."""

    CHUNK_BYTES = 1 << 25     # pinned host memory per chunk: 256 frames (4 minutes at 1 fps) of the default 8x8x1024 level

    def __init__(self, cfg: dict, ntm, *, chunk_cap: int = 32, frames_cap: int = 256, device="cuda",
                 device_frames: Optional[int] = None):
        self.lib = L.load()
        self.device = torch.device(device)
        if self.device.type != "cuda":
            raise L.FvsError("StreamBank needs a CUDA device (no CPU fallback)")
        self.cfg = star_config(cfg)
        self.D, self.pa, self.pb = self.cfg.D, self.cfg.cur_size ** 2, self.cfg.long_size ** 2
        self.chunk_cap = int(chunk_cap)
        lw, tw, pr = C.c_int64(), C.c_int64(), C.c_int64()
        L.check(self.lib.fvs_bank_rows(C.byref(self.cfg), self.chunk_cap, C.byref(lw), C.byref(tw), C.byref(pr)), "fvs_bank_rows")
        self.device_frames = device_window(self.cfg, self.chunk_cap, device_frames)
        f16 = torch.float16
        rows = max(int(frames_cap), 2 * self.chunk_cap) if self.device_frames is None else self.device_frames + self.chunk_cap
        with torch.cuda.device(self.device):
            self.prefix_buf = torch.zeros(pr.value, self.D, dtype=f16, device=self.device)
            self.long_work = torch.zeros(lw.value, self.pb, self.D, dtype=f16, device=self.device)
            self.tur_work = torch.zeros(tw.value, 1, self.D, dtype=f16, device=self.device)
            self.frames = torch.empty(rows, self.pa, self.D, dtype=f16, device=self.device)
            self.header = torch.zeros(8, dtype=torch.int64, device=self.device)
            self.ws = torch.empty(self.lib.fvs_stream_workspace_bytes(C.byref(self.cfg), self.chunk_cap), dtype=torch.uint8,
                                  device=self.device)
        self._ntm_keep = [t.detach().to(device=self.device, dtype=f16).contiguous() for t in ntm] if ntm is not None else None
        self.ntm = L.NtmWeights(*[t.data_ptr() for t in self._ntm_keep]) if ntm is not None else None
        self.bank = L.Bank(self.prefix_buf.data_ptr(), self.long_work.data_ptr(), self.tur_work.data_ptr(),
                           self.frames.data_ptr(), self.header.data_ptr(), self.frames.shape[0], self.chunk_cap, 0, 0, 0, 0, 0,
                           self.device_frames or 0)
        self.tier = HT.HostChunks()      # frames >= device_frames, laid out when the first one spills

    # ---- state as the reference sees it (views of the bank) ---------------------------------------------------------
    @property
    def steps(self) -> int:
        return int(self.bank.step)

    def prefix_rows(self) -> int:
        b = self.bank
        return b.n_tur + b.n_long * self.pb + b.n_cur * self.pa

    def prefix(self) -> torch.Tensor:
        """[Turing | long | key | current] flattened to [rows, D]: a VIEW of the bank (vstream_arch.py:483)"""
        return self.prefix_buf[:self.prefix_rows()]

    def state(self):
        """(cur [n_cur, a*a, D], long [n_long, b*b, D], Turing [n_tur, 1, D], frame buffer [n, a*a, D]) — views in the order
        of `video_embedding_memory` (vstream_arch.py:694).  Once frames have left HBM (device_frames), the frame buffer is
        the zero-row stand-in frames[:0], as the Manager-list publication sends it; frame_buffer() builds the whole one."""
        b = self.bank
        o1 = b.n_tur
        o2 = o1 + b.n_long * self.pb
        tur = self.prefix_buf[:o1].view(b.n_tur, 1, self.D)
        lng = self.prefix_buf[o1:o2].view(b.n_long, self.pb, self.D)
        cur = self.prefix_buf[o2:o2 + b.n_cur * self.pa].view(b.n_cur, self.pa, self.D)
        return cur, lng, tur, self.frames[:0] if self.n_host() else self.frames[:b.n_frames]

    @property
    def host_chunks(self) -> list:
        """the pinned chunks of the host tier (frames >= device_frames)"""
        return self.tier.chunks

    def n_host(self) -> int:
        """frames of the stream kept in the host chunks (those at or past device_frames)"""
        return 0 if self.device_frames is None else max(0, self.bank.n_frames - self.device_frames)

    def frame_buffer(self) -> torch.Tensor:
        """the whole frame buffer [n_frames, a*a, D] (img_feature_buffer): the device view frames[:n_frames] while every
        frame is in HBM, else built in pinned host memory — device rows D2H, host chunks H2H (synchronises the current
        stream, so the spills of the last steps have landed)"""
        if self.n_host() == 0:
            return self.frames[:self.bank.n_frames]
        with torch.cuda.device(self.device):
            return self.tier.to_host(self.frames[:self.device_frames])

    def reset(self):
        L.check(self.lib.fvs_bank_reset(C.byref(self.bank), L.cur_stream()), "fvs_bank_reset")
        self.tier = HT.HostChunks()

    # ---- host tier (device_frames) -------------------------------------------------------------------------------------
    def _host_tier(self) -> HT.HostChunks:
        """the host tier, laid out by CHUNK_BYTES as it is when the first frame spills"""
        if self.tier.dtype is None:
            self.tier.lay_out(self.frames.dtype, [(self.pa, self.D)], self.CHUNK_BYTES)
        return self.tier

    def _spill(self, n0: int, t: int) -> int:
        """after the step of frames [n0, n0 + t): copy those at or past device_frames from the slot to the host chunks,
        asynchronously on the current stream (ahead of the next step, which overwrites the slot).  The clip's frames are
        contiguous in `frames` from row min(n0, device_frames) (frame_row, csrc/stream_kernels.cu).  Returns the bytes."""
        N = self.device_frames
        k = t if N is None else max(0, min(t, N - n0))      # the clip's frames below N, which stay in HBM
        if k == t:
            return 0
        src = self.frames[min(n0, N) + k:min(n0, N) + t]
        self._host_tier().write(n0 + k - N, [src])
        return src.numel() * src.element_size()

    def _reserve_frames(self, t: int):
        if self.device_frames is not None:    # fixed at creation: frames [0, N) and one clip's slot
            return
        if self.bank.n_frames + t > self.frames.shape[0]:   # geometric growth of img_feature_buffer (device-resident)
            new = torch.empty(2 * (self.bank.n_frames + t), self.pa, self.D, dtype=self.frames.dtype, device=self.device)
            new[:self.bank.n_frames].copy_(self.frames[:self.bank.n_frames])
            self.frames = new
            self.bank.frames = new.data_ptr()
            self.bank.frames_cap = new.shape[0]

    # ---- checkpoint / restore (DESIGN.md §3.12) ------------------------------------------------------------------------
    def checkpoint(self, rng: Optional[dict] = None):
        """The stream's state as a checkpoint.StreamCheckpoint in pinned host memory: prefix, long / Turing working sets,
        frame buffer and counters.  Call it from the writer, between steps: on the current stream those arrays are a
        consistent state.  Returns once the copies have landed."""
        from . import checkpoint as CK
        b = self.bank
        counters = dict(n_tur=b.n_tur, n_long=b.n_long, n_cur=b.n_cur, n_frames=b.n_frames, step=b.step)
        with torch.cuda.device(self.device):
            spilled = self.n_host() > 0     # frame_buffer() is then a pinned host tensor made for this checkpoint alone
            frames = self.frame_buffer()
            ck = CK.llava(CK.star_config(self.cfg), counters, self.prefix(), self.long_work[:b.n_long],
                          self.tur_work[:b.n_tur], None if spilled else frames, rng=rng,
                          owned={"frames": frames} if spilled else None)
            torch.cuda.current_stream().synchronize()
        return ck

    def restore(self, ckpt):
        """Continue the stream of `ckpt` in this bank (any device, any chunk_cap whose capacities hold it, any
        device_frames): same STAR config or ValueError; the frame buffer grows as needed, or, with device_frames, frames
        [0, N) go to HBM and the rest to the host chunks.  One fvs_bank_restore: the working sets and frames by copy
        engine, the prefix and header under the seqlock, so readers that have this bank mapped never see a mix."""
        from . import checkpoint as CK
        CK.check_star(ckpt, self.cfg, "StreamBank.restore")
        n = ckpt.counters
        srcs = [ckpt.tensor(k) for k in ("prefix", "long", "tur", "frames")]
        for t in srcs:
            if t.numel() and not (t.is_cuda and t.device == self.device) and not (not t.is_cuda and t.is_pinned()):
                raise ValueError("StreamBank.restore: checkpoint tensors must be pinned host memory or on the bank's device")
        with torch.cuda.device(self.device):
            if n["n_frames"] > self.frames.shape[0]:
                self._reserve_frames(n["n_frames"] - self.bank.n_frames)
            L.check(self.lib.fvs_bank_restore(C.byref(self.cfg), C.byref(self.bank), n["n_tur"], n["n_long"], n["n_cur"],
                                              n["n_frames"], n["step"], *[t.data_ptr() if t.numel() else None for t in srcs],
                                              L.cur_stream()), "fvs_bank_restore")
            self.tier = HT.HostChunks()
            N = self.device_frames
            if N is not None and n["n_frames"] > N:           # frames >= N: to the host tier
                self._host_tier().write(0, [srcs[3][N:n["n_frames"]]])
            self.ws.zero_()       # the step's arrival counters start at zero (a fresh bank's workspace is uninitialised)
            torch.cuda.current_stream().synchronize()    # the sources may be freed as soon as this returns
        self._last_T = 0

    def __getstate__(self):     # see VitEncoder.__getstate__; the stream state itself is not transferred (a fresh bank)
        if self.steps > 0:
            raise L.FvsError("a StreamBank with a stream in progress cannot be pickled: reset_video_stream() first, or hand the "
                             "reader its tensors (flash_vstream_b200.serve.export_bank)")
        c = self.cfg
        return {"cfg": {n: getattr(c, n) for n, _ in c._fields_}, "ntm": self._ntm_keep, "chunk_cap": self.chunk_cap,
                "frames_cap": self.frames.shape[0], "device": str(self.device), "device_frames": self.device_frames}

    def __setstate__(self, st):
        self.__init__(st["cfg"], st["ntm"], chunk_cap=st["chunk_cap"], frames_cap=st["frames_cap"], device=st["device"],
                      device_frames=st.get("device_frames"))

    def needs_draws(self, t: int) -> bool:
        """does a step of t frames run the k-means (working set > long_len)?"""
        return self.bank.step > 0 and self.cfg.long_len > 0 and self.bank.n_long + t > self.cfg.long_len

    def working_rows(self, t: int) -> int:
        return (self.bank.n_long if self.bank.step > 0 else 0) + t

    # ---- one clip -----------------------------------------------------------------------------------------------------
    def step(self, inp: torch.Tensor, *, vit: Optional["VitEncoder"] = None, draws=None):
        """inp: pixels [t,3,S,S] (with `vit`) or finished ViT features [t, grid*grid, D] f16.  draws = (init_idx int32 [K],
        refill_idx int32 [10*K]) device tensors, needed when needs_draws(t).  The one-bank case of stream_step_many."""
        stream_step_many([self], [inp], vit=vit, draws=[draws])

    def info(self):
        """device views of the last step's diagnostics: labels int32 [T], info int32 [4], key_idx int64 [<=key_len],
        wsum f16 [long_len] (aliases of the workspace; clone before the next step)"""
        ptrs = [C.c_void_p() for _ in range(4)]
        L.check(self.lib.fvs_stream_step_info(C.byref(self.cfg), C.byref(self.bank), L.ptr(self.ws), *[C.byref(p) for p in ptrs]),
                "fvs_stream_step_info")
        base = self.ws.data_ptr()
        off = [p.value - base for p in ptrs]
        lab = self.ws[off[0]:off[0] + 4 * getattr(self, "_last_T", 0)].view(torch.int32)
        info = self.ws[off[1]:off[1] + 16].view(torch.int32)
        key = self.ws[off[2]:off[2] + 64].view(torch.int64)
        wsum = self.ws[off[3]:off[3] + 2 * max(self.cfg.long_len, 1)].view(torch.float16)
        return lab, info, key, wsum


def stream_step_many(banks, inputs, *, vit: Optional[VitEncoder] = None, draws=None, max_blocks: int = 0,
                     _packed: Optional[torch.Tensor] = None):
    """One step for many streams (fvs_stream_step_multi): banks[i] takes clip inputs[i] — pixels [t_i,3,S,S] (with `vit`)
    or finished ViT features [t_i, grid*grid, D] f16.  Bit-identical to banks[0].step(inputs[0], ...), then banks[1]...,
    with the same draws.  draws: None or a list with (init_idx, refill_idx) | None per bank.  max_blocks caps the blocks
    of one consolidation launch (0 = the device's co-residency limit).  If any bank's step is refused, no bank moves.
    _packed: the clips already back to back in one contiguous tensor (inputs[i] its consecutive slices, e.g. the views
    of a preprocessor's many()), which the step then reads in place of their concatenation."""
    banks, inputs = list(banks), list(inputs)
    if not banks or len(banks) != len(inputs):
        raise ValueError(f"{len(banks)} banks for {len(inputs)} clips")
    draws = list(draws) if draws is not None else [None] * len(banks)
    if len(draws) != len(banks):
        raise ValueError(f"{len(draws)} draws for {len(banks)} banks")
    if len({id(b) for b in banks}) != len(banks):
        raise ValueError("a bank appears twice in one step")
    _chk_cuda(*inputs)
    b0 = banks[0]
    for b in banks:
        if any(getattr(b.cfg, n) != getattr(b0.cfg, n) for n, _ in b0.cfg._fields_):
            raise ValueError("every bank of one step must have the same STAR config")
        if b.device != b0.device:
            raise ValueError("every bank of one step must live on the same device")
    jobs = (L.StreamJob * len(banks))()
    for i, (bank, inp, dr) in enumerate(zip(banks, inputs, draws)):      # host validation first: nothing moves on a refusal
        t = inp.shape[0]
        if t > bank.chunk_cap:
            raise ValueError(f"clip of {t} frames > chunk_cap {bank.chunk_cap}")
        init_idx, refill_idx = dr if dr is not None else (None, None)
        if bank.needs_draws(t):
            if init_idx is None or refill_idx is None:
                raise ValueError("this step runs the weighted k-means: pass draws=(init_idx, refill_idx)")
            assert init_idx.dtype == torch.int32 and refill_idx.dtype == torch.int32
            assert init_idx.numel() >= bank.cfg.long_len and refill_idx.numel() >= 10 * bank.cfg.long_len
        jobs[i].frames = t
        jobs[i].init_idx, jobs[i].refill_idx = L.ptr(init_idx), L.ptr(refill_idx)
    if vit is not None:
        inputs = [x.to(vit.dtype) if x.dtype != vit.dtype else x for x in inputs]
        for x in inputs:
            assert tuple(x.shape[1:]) == (3, vit.image, vit.image), x.shape
    else:
        for x in inputs:
            assert x.dtype == torch.float16 and x.shape[1] == b0.cfg.grid ** 2 and x.shape[2] == b0.D, x.shape
    if _packed is not None:
        if (not _packed.is_contiguous() or _packed.dtype != inputs[0].dtype or tuple(_packed.shape[1:]) != tuple(inputs[0].shape[1:])
                or _packed.shape[0] != sum(x.shape[0] for x in inputs)):
            raise ValueError(f"packed clips {_packed.dtype} {tuple(_packed.shape)} are not the {len(inputs)} clips back to back")
        row, off = _packed[0].numel() * _packed.element_size(), 0
        for x in inputs:
            if x.data_ptr() != _packed.data_ptr() + off * row:
                raise ValueError("packed clips: the clips are not consecutive slices of the packed tensor")
            off += x.shape[0]
        inp = _packed
    else:
        inp = _c(torch.cat(inputs, dim=0)) if len(inputs) > 1 else _c(inputs[0])
    for i, bank in enumerate(banks):
        t = inputs[i].shape[0]
        bank._reserve_frames(t)
        jobs[i].bank = C.pointer(bank.bank)
        jobs[i].ntm = C.pointer(bank.ntm) if bank.ntm is not None else None
        jobs[i].workspace, jobs[i].workspace_bytes = L.ptr(bank.ws), bank.ws.numel()
    if vit is not None:
        vit.reserve(min(inp.shape[0], max(vit.max_batch, 1)))
        kind, vh, vws, vwsn = L.INPUT_PIXELS, vit._h, L.ptr(vit._ws), vit._ws.numel()
    else:
        kind, vh, vws, vwsn = L.INPUT_FEATURES, None, None, 0
    last_T = [bank.working_rows(inputs[i].shape[0]) for i, bank in enumerate(banks)]
    first = [bank.bank.n_frames for bank in banks]
    L.check(b0.lib.fvs_stream_step_multi(C.byref(b0.cfg), jobs, len(banks), vh, L.ptr(inp), kind, vws, vwsn, int(max_blocks),
                                         L.cur_stream()), "fvs_stream_step_multi")
    for bank, T, n0, x in zip(banks, last_T, first, inputs):
        bank._last_T = T
        bank._spill(n0, x.shape[0])     # frames past device_frames: slot -> host chunks, behind the step on this stream


def bank_snapshot(prefix_buf: torch.Tensor, header: torch.Tensor, cur_size: int, long_size: int, out: Optional[torch.Tensor] = None,
                  status: Optional[torch.Tensor] = None):
    """Consistent copy of a bank prefix that another process / GPU may be updating (seqlock, see fvs_bank_snapshot).
    Returns (out [max_rows, D], status int64 [7] device = {seq0, seq1, n_tur, n_long, n_cur, n_frames, step})."""
    dev = out.device if out is not None else torch.device("cuda", torch.cuda.current_device())
    if out is None:
        out = torch.empty(prefix_buf.shape, dtype=prefix_buf.dtype, device=dev)
    if status is None:
        status = torch.zeros(8, dtype=torch.int64, device=dev)
    L.check(L.load().fvs_bank_snapshot(L.ptr(prefix_buf), L.ptr(header), L.ptr(out), out.shape[0], out.shape[1], cur_size,
                                       long_size, L.ptr(status), L.cur_stream()), "fvs_bank_snapshot")
    return out, status


# --------------------------------------------------------------------------------------------- alternate compressors
ALT_DROP, ALT_MERGE, ALT_KDROP, ALT_KMERGE, ALT_KMEANS = 0, 1, 2, 3, 4
_alt_ws_cache: dict = {}


def _alt_workspace(need: int, dev) -> torch.Tensor:
    key = (dev.index, torch.cuda.current_stream().cuda_stream)
    ws = _alt_ws_cache.get(key)
    if ws is None or ws.numel() < need:
        ws = torch.empty(max(need, 1 << 20), dtype=torch.uint8, device=dev)
        _alt_ws_cache[key] = ws
    return ws


def alt_sequential(method: int, X: torch.Tensor, T0: int, coins: Optional[torch.Tensor] = None,
                   sim_in: Optional[torch.Tensor] = None):
    """One launch of a sequential alternate compressor over X [T, PD] f16 (see fvs_alt_sequential).
    Returns (kept int32 [T0] | None, feat [T0, PD] | None, sim | None, pos int32 [T - T0])."""
    _chk_cuda(X, coins, sim_in)
    X = _c(X)
    T, PD = X.shape
    dev = X.device
    lib = L.load()
    ws = _alt_workspace(lib.fvs_alt_workspace_bytes(method, T, T0, PD), dev)
    kept = torch.empty(T0, dtype=torch.int32, device=dev)
    feat = torch.empty(T0, PD, dtype=X.dtype, device=dev) if method in (ALT_MERGE, ALT_KMERGE) else None
    if method == ALT_KDROP:
        sim = None
    elif method == ALT_KMERGE:
        sim = torch.empty(T0, T0, dtype=X.dtype, device=dev)
    else:
        sim = torch.empty(T0 - 1, dtype=X.dtype, device=dev)
    pos = torch.empty(T - T0, dtype=torch.int32, device=dev)
    L.check(lib.fvs_alt_sequential(method, L.ptr(X), T, T0, PD, L.ptr(_c(sim_in)), L.ptr(_c(coins)), L.ptr(kept), L.ptr(feat),
                                   L.ptr(sim), L.ptr(pos), L.ptr(ws), ws.numel(), L.dtype_code(X.dtype), L.cur_stream()),
            "fvs_alt_sequential")
    return kept, feat, sim, pos


def alt_kmeans(X: torch.Tensor, init_idx: torch.Tensor, refill_idx: torch.Tensor, K: int, max_iter: int = 10,
               tol: float = 1e-4):
    """kmeans_feature's device-side Lloyd loop.  Returns (C [K, PD], labels int32 [T], info int32 [4])."""
    _chk_cuda(X, init_idx, refill_idx)
    X = _c(X)
    T, PD = X.shape
    dev = X.device
    lib = L.load()
    ws = _alt_workspace(lib.fvs_alt_workspace_bytes(ALT_KMEANS, T, K, PD), dev)
    assert init_idx.dtype == torch.int32 and refill_idx.dtype == torch.int32 and refill_idx.numel() >= max_iter * K
    C = torch.empty(K, PD, dtype=X.dtype, device=dev)
    labels = torch.empty(T, dtype=torch.int32, device=dev)
    info = torch.empty(4, dtype=torch.int32, device=dev)
    L.check(lib.fvs_alt_kmeans(L.ptr(X), L.ptr(init_idx), L.ptr(refill_idx), T, K, PD, max_iter, tol, L.ptr(C), L.ptr(labels),
                               L.ptr(info), L.ptr(ws), ws.numel(), L.dtype_code(X.dtype), L.cur_stream()), "fvs_alt_kmeans")
    return C, labels, info
