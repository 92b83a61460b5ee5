"""The Qwen2-VL vision tower blocks on sm_90a: the `encode_patches` callable of VisualB200, i.e. what
FlashVStreamQwen2VisionTransformerPretrainedModel.forward_simple_not_merge runs after temporal_pool
(Flash-VStream-Qwen/models/vstream_qwen2vl_realtime.py:413-426: patch_embed, rot_pos_emb, cu_seqlens, the block loop).
One fvs_qwen_vit_encode call per clip; weights are taken from the reference module's own state dict."""
from __future__ import annotations

import ctypes as C
from typing import Optional

import torch

from .. import _lib as L
from ..ops import _c, _chk_cuda


class QwenVisionBlocksB200:
    """state-dict keys are the reference module's (transformers Qwen2-VL vision tower):
    patch_embed.proj.weight [E,3,2,14,14]; blocks.{i}.norm1/norm2.{weight,bias}; blocks.{i}.attn.qkv/proj.{weight,bias};
    blocks.{i}.mlp.fc1/fc2.{weight,bias}"""

    def __init__(self, state_dict: dict, *, depth: int, heads: int = 16, ln_eps: float = 1e-6, dtype=torch.bfloat16,
                 device="cuda", use_graphs: bool = False, graph_max_rows: int = 8192):
        self.lib = L.load()
        dev = torch.device(device)
        if dev.type != "cuda":
            raise L.FvsError("QwenVisionBlocksB200 needs a CUDA device (no CPU fallback)")
        if dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        self.dtype, self.device, self.depth, self.heads = dtype, dev, depth, heads
        self._ctor = dict(depth=depth, heads=heads, ln_eps=ln_eps, dtype=dtype, use_graphs=use_graphs,
                          graph_max_rows=graph_max_rows)
        # CUDA-graph replay of the whole encode for small clips (a few hundred launches of 5-40 us kernels each): one graph
        # per grid signature, static input / output buffers, bit-identical to the eager launches
        self.use_graphs, self.graph_max_rows, self._graphs = use_graphs, graph_max_rows, {}
        self._sd = {}                                         # the prepared device weights, under the state-dict keys

        def k(key, t):
            self._sd[key] = t.detach().to(device=dev, dtype=dtype).contiguous()
            return self._sd[key]
        pw = state_dict["patch_embed.proj.weight"]
        self.embed = pw.shape[0]
        self.patch_dim = pw[0].numel()
        self.patch_w = k("patch_embed.proj.weight", pw.reshape(self.embed, -1))
        self.mlp = state_dict["blocks.0.mlp.fc1.weight"].shape[0] if depth else 4 * self.embed
        arr = (L.VitLayerWeights * max(depth, 1))()
        names = dict(ln1_w="norm1.weight", ln1_b="norm1.bias", qkv_w="attn.qkv.weight", qkv_b="attn.qkv.bias",
                     o_w="attn.proj.weight", o_b="attn.proj.bias", ln2_w="norm2.weight", ln2_b="norm2.bias",
                     fc1_w="mlp.fc1.weight", fc1_b="mlp.fc1.bias", fc2_w="mlp.fc2.weight", fc2_b="mlp.fc2.bias")
        for i in range(depth):
            for field, key in names.items():
                setattr(arr[i], field, k(f"blocks.{i}.{key}", state_dict[f"blocks.{i}.{key}"]).data_ptr())
        head_dim = self.embed // heads
        dim = head_dim // 2                                   # VisionRotaryEmbedding(head_dim // 2)
        inv_freq = 1.0 / (10000.0 ** (torch.arange(0, dim, 2, dtype=torch.float) / dim))
        inv = (C.c_float * inv_freq.numel())(*inv_freq.tolist())
        cfg = L.QwenVitConfig(self.embed, heads, self.mlp, depth, self.patch_dim, ln_eps, L.dtype_code(dtype))
        self._h = C.c_void_p()
        with torch.cuda.device(dev):
            L.check(self.lib.fvs_qwen_vit_create(C.byref(self._h), C.byref(cfg), self.patch_w.data_ptr(), arr, inv,
                                                 L.cur_stream()), "fvs_qwen_vit_create")
            torch.cuda.current_stream().synchronize()          # the permuted weight copies are complete; originals of
        self._ws: Optional[torch.Tensor] = None               # qkv / proj are no longer referenced by the handle

    # The reference's CLI pickles the whole model into its memory-manager process (cli_server_2gpu.py:301-304).  A ctypes
    # handle cannot travel; the prepared weights can (torch.multiprocessing shares CUDA tensors by IPC handle, plain pickle
    # copies them), and the handle is rebuilt from them on the other side.
    def __getstate__(self):
        return {"ctor": self._ctor, "weights": self._sd, "device": str(self.device)}

    def __setstate__(self, st):
        self.__init__(st["weights"], device=st["device"], **st["ctor"])

    def to(self, device) -> "QwenVisionBlocksB200":
        """the same blocks on `device`: self when already there, else a new handle over copies of the weights"""
        dev = torch.device(device)
        if dev.type == "cuda" and dev.index is None:
            dev = torch.device("cuda", torch.cuda.current_device())
        if dev == self.device:
            return self
        return QwenVisionBlocksB200(self._sd, device=dev, **self._ctor)

    @classmethod
    def from_module(cls, visual, **kw):
        """from the reference's FlashVStreamQwen2VisionTransformerPretrainedModel instance"""
        sd = visual.state_dict()
        depth = len(visual.blocks)
        heads = visual.blocks[0].attn.num_heads
        p = next(visual.parameters())
        return cls(sd, depth=depth, heads=heads, dtype=kw.pop("dtype", p.dtype), **kw)

    def __call__(self, patch_rows: torch.Tensor, total_grid_thw) -> torch.Tensor:
        _chk_cuda(patch_rows)
        x = _c(patch_rows.to(self.dtype))
        grids = total_grid_thw.tolist() if isinstance(total_grid_thw, torch.Tensor) else [list(g) for g in total_grid_thw]
        rows = sum(t * h * w for t, h, w in grids)
        assert x.shape == (rows, self.patch_dim), f"patch rows {tuple(x.shape)} do not match grids {grids}"
        if self.use_graphs and rows <= self.graph_max_rows and not torch.cuda.is_current_stream_capturing():
            return self._replay(x, grids)
        return self._encode(x, grids, rows)

    def _replay(self, x: torch.Tensor, grids) -> torch.Tensor:
        key = tuple(tuple(int(v) for v in g) for g in grids)
        entry = self._graphs.get(key)
        if entry is None:
            static_in = torch.empty_like(x)
            static_in.copy_(x)
            side = torch.cuda.Stream(device=self.device)
            side.wait_stream(torch.cuda.current_stream())
            # the graph bakes in device pointers: it gets its own workspace, kept alive by the cache entry
            ws = torch.empty(self.lib.fvs_qwen_vit_workspace_bytes(self._h, x.shape[0]), dtype=torch.uint8, device=self.device)
            with torch.cuda.stream(side):
                self._encode(static_in, grids, x.shape[0], ws)      # warm-up: function attributes set outside the capture
                side.synchronize()
                graph = torch.cuda.CUDAGraph()
                with torch.cuda.graph(graph, stream=side):
                    static_out = self._encode(static_in, grids, x.shape[0], ws)
            torch.cuda.current_stream().wait_stream(side)
            entry = self._graphs[key] = (graph, static_in, static_out, ws)
        graph, static_in, static_out, _ = entry
        static_in.copy_(x)
        graph.replay()
        return static_out.clone()        # the static buffer is overwritten by the next replay

    def _encode(self, x: torch.Tensor, grids, rows: int, ws: Optional[torch.Tensor] = None) -> torch.Tensor:
        if ws is None:
            need = self.lib.fvs_qwen_vit_workspace_bytes(self._h, rows)
            if self._ws is None or self._ws.numel() < need:
                self._ws = torch.empty(need, dtype=torch.uint8, device=self.device)
            ws = self._ws
        out = torch.empty(rows, self.embed, dtype=self.dtype, device=self.device)
        flat = (C.c_int32 * (3 * len(grids)))(*[int(v) for g in grids for v in g])
        L.check(self.lib.fvs_qwen_vit_encode(self._h, L.ptr(x), L.ptr(out), flat, len(grids), L.ptr(ws), ws.numel(),
                                             L.cur_stream()), "fvs_qwen_vit_encode")
        return out

    def close(self):
        if getattr(self, "_h", None) is not None and self._h:
            self.lib.fvs_qwen_vit_destroy(self._h)
            self._h = None

    def __del__(self):
        try:
            self.close()
        except Exception:
            pass
