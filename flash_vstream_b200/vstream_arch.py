"""Drop-in mirror of the hot-path half of flash_vstream.model.vstream_arch (reference lines cited per method):
NeuralTuringMachine (:34-65) and the VStreamMetaForCausalLM methods encode_images (:159-161),
attention (:174-183), compress_spatial_features (:193-212), compress_temporal_features (:214-277) and
embed_video_streaming (:611-697), executing on libfvs_b200.so.  The LLM-side half of that file (prompt splicing,
:286-609) is out of scope (SURVEY.md §2).

Differences by design (DESIGN.md "state residency"): all per-stream state stays on the GPU — the reference's
`.cpu()` / Manager-list round trips (vstream_arch.py:650,672-676,693-695) are gone; `video_embedding_memory` is still
written as `[cur, long, Turing, buffer]` under the lock, but holds CUDA tensors (the unmodified reader at
vstream_arch.py:480-485 calls `.to(device)` on them, a no-op).

A stream on the fused path can be suspended and resumed (`save_video_stream` / `load_video_stream`, DESIGN.md §3.12), in
another process or on another GPU.  Its k-means draws come from the global generators (draws.GLOBAL), which a checkpoint
neither stores nor sets: a resumed stream continues from the resuming process's global generators, as the reference's would
after a restart.
"""
from __future__ import annotations

import math
from types import SimpleNamespace
from typing import List, Optional

import torch
import torch.nn as nn

from . import host_tier as HT
from . import ops
from .compress_functions import (attention_feature, drop_feature, k_drop_feature, k_merge_feature, kmeans_draws,
                                 kmeans_feature, merge_feature, weighted_kmeans_device, weighted_kmeans_feature)
from .draws import GLOBAL

KEY_LENGTH = 3  # hard-coded in the reference (vstream_arch.py:263, :683)


_ALTERNATES = (drop_feature, merge_feature, k_drop_feature, kmeans_feature, k_merge_feature)


def _refuse_alternate_weight(fn, T: int, T0: int, sample_type: str):
    """Raise where the reference's key retrieval raises on the weight an alternate compressor returns for T long rows
    (vstream_arch.py:258-266, :679-686).  The callers run this before the pooling of the call, its frame buffer append and
    any launch:
      * None -> TypeError from torch.argsort(None): kdrop and kmeans never return a weight, drop / merge / kmerge return
        None on their T <= T0 pass-through;
      * k_merge's [T0, T0] similarity matrix -> long_memory[argsort(weight)] is [T0, T0, P, D], and the distance to the
        long memory does not broadcast (T > T0 >= 2) -> RuntimeError.  Sorting that matrix flat instead would give indices
        up to T0² - 1, far past the T rows key retrieval reads.
    Draws: kdrop first draws its T - T0 coin flips, as the reference's k_drop_feature does before it returns; a refused
    kmeans draws nothing, while the reference draws its randperm and the refills of a Lloyd loop that would have to run."""
    if fn not in _ALTERNATES:
        return
    if fn is k_drop_feature and T > T0:
        GLOBAL.randints(0, 1, T - T0)
    if fn in (k_drop_feature, kmeans_feature) or T <= T0:
        raise TypeError(f"argsort(): video_sample_type = {sample_type} returns no weight for {T} long-memory rows "
                        f"and video_long_memory_length = {T0}, and the key retrieval sorts that weight")
    if fn is k_merge_feature:
        raise RuntimeError(f"video_sample_type = {sample_type} returns its [{T0}, {T0}] similarity matrix as the weight; "
                           f"the key centroids it selects do not broadcast against the {T} long-memory rows")


def _is_manager_proxy(obj) -> bool:
    try:
        from multiprocessing.managers import BaseProxy
    except Exception:   # pragma: no cover
        return False
    return isinstance(obj, BaseProxy)


class NeuralTuringMachine(nn.Module):
    """Parameter-compatible with the reference module (vstream_arch.py:34-45) so its checkpoints load unchanged;
    only q_proj / k_proj take part in the live path (get_weight, :47-52)."""

    def __init__(self, input_dim=1024, output_dim=1024, attention_dropout=0.1):
        super().__init__()
        self.input_dim, self.output_dim = input_dim, output_dim
        self.q_proj = nn.Linear(input_dim, output_dim)
        self.k_proj = nn.Linear(input_dim, output_dim)
        self.v_proj = nn.Linear(input_dim, output_dim)
        self.dropout = nn.Dropout(attention_dropout)
        self.out_proj = nn.Linear(output_dim, input_dim)
        self.out_dropout = nn.Dropout(attention_dropout)
        self.out_ln = nn.LayerNorm(input_dim, eps=1e-12)

    def forward(self, x, y):  # `attention2` (vstream_arch.py:185-191) is marked deprecated upstream
        raise NotImplementedError("NeuralTuringMachine.forward belongs to the deprecated attention2 path")


class VStreamMetaForCausalLM:
    """Mixin with the reference's method names.  The host class provides `self.config`, `self.get_model()` (an object
    with `.attention_model` and `.get_vision_tower()`), exactly like the reference's mixin (vstream_arch.py:143-157)."""

    use_video_streaming_mode = False
    video_embedding_memory = None
    video_embedding_mem_lock = None
    fvs_tie_order = "stable"  # "stable": our kernel (ties -> lower index); "torch": torch.argsort like the reference
    fvs_fused_stream = True   # streaming steps run as fvs_stream_step on a persistent bank (ops.StreamBank) when the config
    #                           allows it; False = the op-by-op path below (same arithmetic, bit-identical state)
    fvs_chunk_cap = 32        # frames per embed_video_streaming call the bank is sized for (grown on demand)
    fvs_bank_device_frames = None   # None: the bank's whole frame buffer in HBM; N: only frames [0, N) (N >= the long
    #                                 working set's rows), later ones in pinned host memory (ops.StreamBank device_frames)

    # ---------------------------------------------------------------------------------------------- encoder
    def get_vision_tower(self):
        return self.get_model().get_vision_tower()

    def encode_images(self, images):
        """vstream_arch.py:159-161"""
        return self.get_model().get_vision_tower()(images)

    def reshape_2x2_image_features(self, image_features):
        """vstream_arch.py:163-172 (`mm_use_4_vision_tokens`): every 2x2 block of neighbouring patches becomes one token
        of 4*D channels, [B, g*g, D] -> [B, (g/2)^2, 4*D], channel order (dy, dx, d).  Data layout only (no arithmetic)."""
        B, P, D = image_features.shape
        g = round(math.sqrt(P))
        assert g * g == P, f"For ViT feature map, {g}*{g}={g**2} != {P}"
        blocks = image_features.reshape(B, g // 2, 2, g // 2, 2, D).transpose(2, 3)      # [B, g/2, g/2, dy, dx, D]
        return blocks.reshape(B, (g // 2) ** 2, 4 * D)

    # ---------------------------------------------------------------------------------------------- abstract memory
    def attention(self, turing_memory, new_feature, update_ratio=0.2):
        """vstream_arch.py:174-183"""
        T1, D1 = turing_memory.shape
        T2, D2 = new_feature.shape
        assert D1 == D2, f"dimmension not match, {D1} != {D2}"
        m = self.get_model().attention_model
        dt = turing_memory.dtype
        ops.require_inference(turing_memory, new_feature, m.q_proj.weight, m.k_proj.weight, what="attention (fvs_abstract_update)")
        return ops.abstract_update(turing_memory, new_feature, m.q_proj.weight.to(dt), m.q_proj.bias.to(dt),
                                   m.k_proj.weight.to(dt), m.k_proj.bias.to(dt), update_ratio)

    # ---------------------------------------------------------------------------------------------- spatial pooling
    def compress_spatial_features(self, image_features, compress_size=1):
        """vstream_arch.py:193-212"""
        compress_type = getattr(self.config, "compress_type", None)
        patch_size = round(math.sqrt(image_features.shape[1]))
        assert patch_size * patch_size == image_features.shape[1], \
            f"For ViT feature map, {patch_size}*{patch_size}={patch_size**2} != {image_features.shape[1]}"
        if patch_size == compress_size:
            return image_features
        elif compress_type is not None:
            if 'mean' in self.config.compress_type:
                return ops.spatial_pool(image_features, compress_size)
            raise NotImplementedError(f"`compress_type` {self.config.compress_type} is not supported yet.")
        return image_features

    # ---------------------------------------------------------------------------------------------- helpers
    def _star_cfg(self):
        c = self.config
        return SimpleNamespace(
            compress_size=getattr(c, "compress_size", 1),
            long_len=getattr(c, "video_long_memory_length", 10), tur_len=getattr(c, "video_Turing_memory_length", 10),
            cur_len=getattr(c, "video_current_memory_length", 1),
            long_size=getattr(c, "compress_long_memory_size", 1), tur_size=getattr(c, "compress_Turing_memory_size", 1),
            ratio=getattr(c, "compress_Turing_update_ratio", 0.2), sample_type=c.video_sample_type)

    def _compress_fn(self, sample_type, streaming=False):
        table = {'drop': drop_feature, 'merge': merge_feature, 'kmeans': kmeans_feature,
                 'weighted_kmeans': weighted_kmeans_feature, 'kdrop': k_drop_feature, 'kmerge': k_merge_feature,
                 'attention': attention_feature}
        if streaming:  # vstream_arch.py:626-637
            table.update({'uni_kmerge': k_merge_feature, 'both_kmerge': k_merge_feature, 'split_kmerge': k_merge_feature})
        if sample_type not in table:
            raise NotImplementedError(f'max_length = {getattr(self.config, "video_max_frames", None)},'
                                      f'while video_sample_type = {sample_type} is not supported yet.')
        return table[sample_type]

    def _order(self, weight):
        if self.fvs_tie_order == "torch":
            return torch.argsort(weight, descending=True)      # the reference's own call (vstream_arch.py:261,681)
        return ops.argsort_desc(weight)

    def _compress_long(self, long_memory, s, draws=None, streaming=False):
        """compress_fn + key retrieval; returns (long_compressed, key_indices).  Sync-free for weighted_kmeans."""
        if s.sample_type == 'weighted_kmeans':
            init_idx, refill_idx = draws if draws is not None else (None, None)
            long_c, weight, _, _ = weighted_kmeans_device(long_memory, s.long_len, None, init_idx, refill_idx)
        else:   # the streaming table also knows the *_kmerge aliases (vstream_arch.py:626-637)
            fn = self._compress_fn(s.sample_type, streaming=streaming)
            _refuse_alternate_weight(fn, long_memory.shape[0], s.long_len, s.sample_type)   # the callers checked already
            long_c, weight, _ = fn(long_memory, s.long_len)
        order = self._order(weight)
        return long_c, ops.key_retrieve(long_memory, order, KEY_LENGTH), order, weight

    # ---------------------------------------------------------------------------------------------- offline
    def compress_temporal_features(self, image_features, draws=None):
        """vstream_arch.py:214-277: list of [T, P, D] -> list of [<=681, D] in the order [Turing | long | key | cur]."""
        s = self._star_cfg()
        self._compress_fn(s.sample_type)  # raises NotImplementedError for unknown types, like the reference
        new_image_features = []
        for img_feature in image_features:
            cur_start = min(s.cur_len, img_feature.shape[0])
            n_long = img_feature.shape[0] - cur_start
            if s.long_len != 0 and n_long > 0:     # before this video's pooling launches
                _refuse_alternate_weight(self._compress_fn(s.sample_type), n_long, s.long_len, s.sample_type)
            if cur_start == 0:
                cur_memory, long_memory, Turing_memory = img_feature[:0], img_feature, img_feature
            else:
                cur_memory = img_feature[-cur_start:]
                long_memory = img_feature[:-cur_start]
                Turing_memory = img_feature[:-cur_start]
            if s.long_size * s.long_size != long_memory.shape[1]:
                long_memory = self.compress_spatial_features(long_memory, s.long_size)
            if s.tur_size * s.tur_size != Turing_memory.shape[1]:
                Turing_memory = self.compress_spatial_features(Turing_memory, s.tur_size)
            if s.long_len == 0 or long_memory.shape[0] == 0:
                long_c = long_memory[:0]
            else:
                long_c, min_indices, _, _ = self._compress_long(long_memory, s, draws)
                key_memory = ops.gather_rows(img_feature, min_indices)
                cur_memory = torch.cat([key_memory, cur_memory], dim=0)
            if s.tur_len == 0 or Turing_memory.shape[0] == 0:
                tur_c = Turing_memory[:0]
            else:
                tur_c, _ = attention_feature(Turing_memory, s.tur_len, self.attention, update_ratio=s.ratio)
            new_image_features.append(torch.cat([tur_c.flatten(0, 1), long_c.flatten(0, 1), cur_memory.flatten(0, 1)], dim=0))
        return new_image_features

    def encode_video_memory(self, images=None, features=None, draws=None):
        """The offline branch of prepare_inputs_labels_for_multimodal (vstream_arch.py:311-329) up to the projector: a list
        of videos, given either as frames `images` ([T,3,H,W] each, encoded in one batch like :314-321) or as pre-extracted
        ViT `features` ([T,P,D] each — the `.safetensors` feature files of README.md:151-161, read by
        eval_video/model_msvd_qa_featuresloader.py:59-64) -> list of memory prefixes [<=681, D].  `cat_proj` (:331) follows."""
        assert (images is None) != (features is None), "give either frames or pre-extracted features"
        compress_size = getattr(self.config, "compress_size", 1)
        four = getattr(self.config, 'mm_use_4_vision_tokens', False)
        if images is not None:
            images = [image if len(image.shape) == 4 else image.unsqueeze(0) for image in images]
            feats = self.encode_images(torch.cat(list(images), dim=0))
            if four:
                feats = self.reshape_2x2_image_features(feats)
            feats = self.compress_spatial_features(feats, compress_size)
            per_video = list(torch.split(feats, [image.shape[0] for image in images], dim=0))
        else:
            per_video = [feat if len(feat.shape) == 3 else feat.unsqueeze(0) for feat in features]
            if four:
                per_video = [self.reshape_2x2_image_features(f) for f in per_video]
            per_video = [self.compress_spatial_features(f, compress_size) for f in per_video]
        return self.compress_temporal_features(per_video, draws=draws)

    # ---------------------------------------------------------------------------------------------- streaming
    def _append_buffer(self, feat):
        """device-resident img_feature_buffer with geometric growth (the reference grows a CPU tensor, :650,:676)"""
        n_new = feat.shape[0]
        st = self.__dict__.setdefault("_fvs_buf", {"cap": None, "n": 0})
        if st["cap"] is None or st["n"] + n_new > st["cap"].shape[0] or st["cap"].shape[1:] != feat.shape[1:]:
            old = st["cap"][:st["n"]] if st["cap"] is not None and st["cap"].shape[1:] == feat.shape[1:] else None
            new_cap = max(64, 2 * ((old.shape[0] if old is not None else 0) + n_new))
            cap = torch.empty((new_cap,) + tuple(feat.shape[1:]), dtype=feat.dtype, device=feat.device)
            if old is not None:
                cap[:old.shape[0]].copy_(old)
            else:
                st["n"] = 0
            st["cap"] = cap
        st["cap"][st["n"]:st["n"] + n_new].copy_(feat)
        st["n"] += n_new
        return st["cap"][:st["n"]]

    def reset_video_stream(self):
        self.__dict__.pop("_fvs_buf", None)
        bank = self.__dict__.get("_fvs_bank")
        if bank is not None:
            bank.reset()
        if self.video_embedding_memory is not None:
            self.video_embedding_memory[:] = []

    # ---- fused path: fvs_stream_step on a persistent bank ----------------------------------------------------------
    def _fused_reject(self, s, grid, D, dtype):
        """None when this STAR config can run as fvs_stream_step, else the knob that keeps it on the op-by-op path"""
        if not self.fvs_fused_stream:
            return "fvs_fused_stream"
        if self.fvs_tie_order != "stable" or "_order" in self.__dict__:   # a replayed / custom tie order: op-by-op only
            return "fvs_tie_order"
        if s.sample_type != 'weighted_kmeans':
            return "video_sample_type"
        a, b = s.compress_size, s.long_size
        ntm = self.get_model().attention_model
        checks = (("compress_type", 'mean' in (getattr(self.config, "compress_type", None) or '')),
                  ("compress_Turing_memory_size", s.tur_size == 1),
                  ("dtype", dtype == torch.float16),
                  ("compress_size", a > 0 and grid % a == 0 and grid != a and a * a <= 64),
                  ("compress_long_memory_size", b > 0 and a % b == 0 and a != b),
                  ("hidden size", D % 256 == 0 and (b * b * D) % 1024 == 0),
                  ("video_long_memory_length", 0 <= s.long_len <= 64),
                  ("video_Turing_memory_length", 0 < s.tur_len <= 64),
                  ("video_current_memory_length", s.cur_len >= 0),
                  ("attention_model", ntm.q_proj.weight.shape[0] <= 64 and ntm.q_proj.weight.shape[1] == D))
        return next((knob for knob, ok in checks if not ok), None)

    def _fused_cfg(self, s, grid, D, dtype):
        """dict for ops.StreamBank when this STAR config can run as fvs_stream_step, else None (op-by-op path)"""
        if self._fused_reject(s, grid, D, dtype) is not None:
            return None
        a, b = s.compress_size, s.long_size
        ntm = self.get_model().attention_model
        return dict(D=D, grid=grid, cur_size=a, long_size=b, long_len=s.long_len, tur_len=s.tur_len, cur_len=s.cur_len,
                    key_len=KEY_LENGTH, ntm_dim=ntm.q_proj.weight.shape[0], ratio=s.ratio)

    def _get_bank(self, cfg, t, device):
        bank = self.__dict__.get("_fvs_bank")
        key = tuple(sorted(cfg.items()))
        cap = HT.check_device_frames(self.fvs_bank_device_frames, "fvs_bank_device_frames")
        mid_stream = bank is not None and bank.steps > 0 and len(self.video_embedding_memory or []) > 0
        if mid_stream and cap != bank.device_frames:
            raise ValueError(f"fvs_bank_device_frames changed from {bank.device_frames} to {cap} in the middle of a stream: "
                             f"reset_video_stream() first, or save_video_stream() / load_video_stream() to move it")
        if bank is None or self.__dict__.get("_fvs_bank_key") != key or bank.device != device or t > bank.chunk_cap or \
                bank.device_frames != cap:
            if mid_stream:
                return None     # mid-stream change of shape: finish this stream op by op
            m = self.get_model().attention_model
            ntm = (m.q_proj.weight, m.q_proj.bias, m.k_proj.weight, m.k_proj.bias)
            chunk_cap = max(int(self.fvs_chunk_cap), t)
            bank = ops.StreamBank(cfg, ntm, chunk_cap=chunk_cap, device=device,
                                  device_frames=ops.device_window(cfg, chunk_cap, cap, "fvs_bank_device_frames"))
            self.__dict__["_fvs_bank"], self.__dict__["_fvs_bank_key"] = bank, key
        return bank

    def _stream_step_fused(self, bank, inp, vit, draws):
        mem = self.video_embedding_memory
        first = mem is None or len(mem) == 0
        if first:
            bank.reset()
        elif bank.steps == 0:
            return False            # the state in `video_embedding_memory` was not produced by this bank
        t = inp.shape[0]
        refills = None
        if draws is None and bank.needs_draws(t):
            *draws, refills = kmeans_draws(GLOBAL, bank.working_rows(t), bank.cfg.long_len, bank.device)
        bank.step(inp, vit=vit, draws=draws)
        if refills is not None:     # we drew the candidates ourselves: learn (asynchronously) how many the device consumed
            refills.consumed_from(bank.info()[1])
        self._publish(list(bank.state()))
        return True

    def _publish(self, new_state):
        """`self.video_embedding_memory[:] = [cur, long, Turing, buffer]` under the lock (vstream_arch.py:693-695); the
        tensors stay on the GPU (views of the bank on the fused path)"""
        lock = self.video_embedding_mem_lock
        if self.video_embedding_memory is None:
            self.video_embedding_memory = []
        mem = self.video_embedding_memory
        if _is_manager_proxy(mem):
            # the unmodified serve CLI hangs a Manager().list() here (cli_video_stream.py:237) and reads it from ANOTHER
            # process: every element is pickled through the Manager server, which cannot forward CUDA IPC handles — publish
            # host copies exactly like the reference does (:694).  The frame buffer (4th element) is never read by the
            # reader (vstream_arch.py:481 binds it to `_`) nor by this writer (the bank owns the frames), so an empty
            # stand-in travels instead of the whole O(n) buffer.  Device-resident readers: flash_vstream_b200.serve.
            cur, lng, tur, buf = new_state
            new_state = [cur.cpu(), lng.cpu(), tur.cpu(), buf[:0].cpu()]
        if lock is not None:
            with lock:
                mem[:] = new_state
        else:
            mem[:] = new_state

    def embed_video_streaming(self, images, draws=None):
        """vstream_arch.py:611-697.  images: [1, t, 3, H, W] (or a 1-element list of [t,3,H,W]).  Side effect:
        self.video_embedding_memory[:] = [cur, long, Turing, buffer].  Returns [] like the reference."""
        assert self.use_video_streaming_mode
        s = self._star_cfg()
        self._compress_fn(s.sample_type, streaming=True)
        if type(images) is list or images.ndim == 5:
            assert len(images) == 1
            images = [image if len(image.shape) == 4 else image.unsqueeze(0) for image in images]
            concat_images = images[0] if len(images) == 1 else torch.cat([image for image in images], dim=0)
        else:
            raise NotImplementedError('Should input video frames, not a single image')
        # fused: pixels -> ViT (pooled tail, the [t,576,D] feature map is never stored) -> one consolidation kernel
        tower = self.get_model().get_vision_tower()
        engine = getattr(tower, "engine", None)
        if engine is not None and concat_images.is_cuda and engine.dtype == torch.float16 and not engine.keep_cls:
            cfg = self._fused_cfg(s, engine.grid, engine.hidden, torch.float16)
            bank = self._get_bank(cfg, concat_images.shape[0], concat_images.device) if cfg is not None else None
            if bank is not None and self._stream_step_fused(bank, concat_images, engine, draws):
                return []
        self._refuse_stream(s, concat_images.shape[0])
        image_features = self.encode_images(concat_images)                           # [t, P, D]
        return self.consolidate_streaming(image_features, draws=draws)

    def _refuse_stream(self, s, t):
        """_refuse_alternate_weight for a streaming call of t frames, before its encoder, pooling and buffer append: its
        compression sees the published long rows plus t (the reference publishes only at the end of a call, :693-695,
        so a refused call leaves the stream as it was)"""
        fn = self._compress_fn(s.sample_type, streaming=True)
        mem = self.video_embedding_memory
        if fn in _ALTERNATES and s.long_len != 0 and mem is not None and len(mem) > 0:
            _refuse_alternate_weight(fn, mem[1].shape[0] + t, s.long_len, s.sample_type)

    def consolidate_streaming(self, image_features, draws=None):
        """Everything of embed_video_streaming after the encoder (vstream_arch.py:644-697)."""
        s = self._star_cfg()
        self._compress_fn(s.sample_type, streaming=True)   # unknown video_sample_type raises like the reference (:663-664)
        self._refuse_stream(s, image_features.shape[0])
        g = round(math.sqrt(image_features.shape[1]))
        if image_features.is_cuda and g * g == image_features.shape[1]:
            cfg = self._fused_cfg(s, g, image_features.shape[2], image_features.dtype)
            bank = self._get_bank(cfg, image_features.shape[0], image_features.device) if cfg is not None else None
            if bank is not None and self._stream_step_fused(bank, image_features, None, draws):
                return []
        if self.fvs_bank_device_frames is not None:   # the op-by-op path keeps its own, device-resident frame buffer
            knob = (self._fused_reject(s, g, image_features.shape[2], image_features.dtype) if image_features.is_cuda
                    else "device") or "fvs_chunk_cap"
            raise NotImplementedError(f"fvs_bank_device_frames bounds the frame buffer of the fused streaming step, and this "
                                      f"stream runs op by op ({knob}): unset fvs_bank_device_frames or change {knob}")
        fused = ('mean' in (getattr(self.config, "compress_type", None) or '') and s.tur_size == 1
                 and g % s.compress_size == 0 and s.compress_size % s.long_size == 0 and g != s.compress_size
                 and s.long_size != s.compress_size and s.compress_size ** 2 <= 64 and image_features.shape[2] % 64 == 0
                 and image_features.dtype == torch.float16)
        if fused:  # one pass over the ViT output: 8x8 (rounded), then 4x4 and 1x1 from the rounded 8x8
            image_feature, long_new, tur_new = ops.spatial_pool3(image_features, s.compress_size, s.long_size)
        else:
            image_feature = self.compress_spatial_features(image_features, s.compress_size).to(torch.float16)
            long_new = image_feature if s.long_size ** 2 == image_feature.shape[1] else \
                self.compress_spatial_features(image_feature, s.long_size)
            tur_new = image_feature if s.tur_size ** 2 == image_feature.shape[1] else \
                self.compress_spatial_features(image_feature, s.tur_size)
        cur_start = min(s.cur_len, image_feature.shape[0])
        cur_memory = image_feature[:0] if cur_start == 0 else image_feature[-cur_start:]
        if s.long_len == 0:
            # no long memory and no key retrieval from the first call on, as on the fused path and behind the guard of the
            # offline path (:256-257); the reference's streaming branch has none (a K = 0 k-means on its second call)
            long_new = long_new[:0]
        mem = self.video_embedding_memory
        first = mem is None or len(mem) == 0
        if first:
            self.__dict__.pop("_fvs_buf", None)
        elif "_fvs_buf" not in self.__dict__:      # continuing a stream the bank started: adopt its frame buffer
            self._append_buffer(mem[3].to(image_feature.device))
        buf = self._append_buffer(image_feature)
        long_c, tur_c = long_new, tur_new
        if not first:
            _, old_long, old_tur, _ = mem
            old_long, old_tur = old_long.to(image_feature.device), old_tur.to(image_feature.device)
            assert old_long.shape[1:] == long_new.shape[1:]
            long_memory = torch.cat((old_long, long_new), dim=0)
            if s.long_len == 0:
                long_c = long_memory
            else:
                long_c, min_indices, _, _ = self._compress_long(long_memory, s, draws, streaming=True)
                key_memory = ops.gather_rows(buf, min_indices)   # global buffer, working-set indices (quirk of :687-688)
                cur_memory = torch.cat([key_memory, cur_memory], dim=0)
            Turing_memory = torch.cat((old_tur, tur_new), dim=0)
            tur_c, _ = attention_feature(Turing_memory, s.tur_len, self.attention, update_ratio=s.ratio)
        self._publish([cur_memory, long_c, tur_c, buf])
        return []

    # ---- suspend / resume (DESIGN.md §3.12) -------------------------------------------------------------------------
    def _fused_knob(self):
        """the knob that keeps this model's stream off the fused path"""
        tower = self.get_model().get_vision_tower()
        engine = getattr(tower, "engine", None) if tower is not None else None
        D = self.get_model().attention_model.q_proj.weight.shape[1]
        return self._fused_reject(self._star_cfg(), engine.grid if engine is not None else 24, D, torch.float16) \
            or "fvs_chunk_cap"      # fused config, but a clip longer than the bank was streamed op by op

    def save_video_stream(self):
        """The stream in progress as a checkpoint.StreamCheckpoint (pinned host memory) that `load_video_stream` continues
        bit for bit, here or in another process or on another GPU.  Fused path only (the op-by-op path raises
        NotImplementedError naming the knob).  The draws of this model come from the global generators (draws.GLOBAL):
        they are settled first but neither stored nor set, so a resumed stream continues from the resuming process's global
        generators — as the reference's would after a restart."""
        bank = self.__dict__.get("_fvs_bank")
        mem = self.video_embedding_memory
        if mem is None or len(mem) == 0:
            raise ValueError("save_video_stream: no stream in progress")
        # the op-by-op path keeps its own frame buffer (_fvs_buf); on the fused path the bank is the stream (a Manager list
        # holds host copies of its state)
        fused = bank is not None and bank.steps > 0 and "_fvs_buf" not in self.__dict__ and \
            (_is_manager_proxy(mem) or mem[0].data_ptr() == bank.state()[0].data_ptr())
        if not fused:
            raise NotImplementedError(f"save_video_stream: this stream runs op by op ({self._fused_knob()}); "
                                      f"checkpoints cover the fused streaming step")
        GLOBAL.settle()
        return bank.checkpoint()

    def load_video_stream(self, ckpt):
        """Continue the stream of `ckpt` (from save_video_stream or StreamPool.checkpoint) in this model: the bank is
        restored and `video_embedding_memory` republished, so the unmodified reader and a Manager-list reader see the
        resumed memory.  A StreamPool checkpoint's own generators are not used: this model draws from the global ones."""
        from . import checkpoint as CK
        if ckpt.family != CK.LLAVA:
            raise ValueError(f"load_video_stream: a {ckpt.family!r} checkpoint is not a LLaVA stream's")
        c = ckpt.config
        cfg = self._fused_cfg(self._star_cfg(), int(c["grid"]), int(c["D"]), torch.float16)
        if cfg is None:
            raise NotImplementedError(f"load_video_stream: this model streams op by op "
                                      f"({self._fused_reject(self._star_cfg(), int(c['grid']), int(c['D']), torch.float16)}); "
                                      f"checkpoints cover the fused streaming step")
        CK.check_star(ckpt, cfg, "load_video_stream")       # before the current stream is dropped
        device = self.get_model().attention_model.q_proj.weight.device
        self.reset_video_stream()
        bank = self._get_bank(cfg, 1, device)
        bank.restore(ckpt)
        if bank.steps > 0:
            self._publish(list(bank.state()))

    def cat_proj(self, all_features):
        """vstream_arch.py:279-284: concatenate the per-video prefixes, project them together, split back"""
        feature_split_size = [x.shape[0] for x in all_features]
        feature_embed = torch.cat(all_features, dim=0)
        feature_proj = self.get_model().mm_projector(feature_embed)
        return torch.split(feature_proj, feature_split_size, dim=0)

    def memory_prefix(self):
        """[Turing | long | cur] flattened — what the reader builds at vstream_arch.py:480-485.  On the fused path the bank
        is laid out in exactly this order, so the prefix is a view (no copy); otherwise one concatenation."""
        bank = self.__dict__.get("_fvs_bank")
        mem = self.video_embedding_memory
        if bank is not None and bank.steps > 0 and mem is not None and len(mem) == 4 and \
                mem[0].data_ptr() == bank.state()[0].data_ptr():
            return bank.prefix()
        cur, lng, tur, _ = mem
        return torch.cat([tur.flatten(0, 1), lng.flatten(0, 1), cur.flatten(0, 1)], dim=0)


class _ModelHost:
    """what `get_model()` returns in the reference: an object with .attention_model and .get_vision_tower() (picklable)"""

    def __init__(self, attention_model, vision_tower):
        self.attention_model, self.vision_tower = attention_model, vision_tower

    def get_vision_tower(self):
        return self.vision_tower


class FlashVStreamB200(VStreamMetaForCausalLM):
    """Self-contained host for the mixin: ViT tower + abstract-memory module + STAR config, no HF / LLM needed.
    `config` accepts the reference's hot-path knobs (scripts/train_and_eval.sh:7-14 defaults)."""

    def __init__(self, vision_tower, attention_model: NeuralTuringMachine, **cfg):
        base = dict(compress_type="mean", compress_size=8, compress_long_memory_size=4, compress_Turing_memory_size=1,
                    compress_Turing_update_ratio=0.2, video_long_memory_length=25, video_Turing_memory_length=25,
                    video_current_memory_length=1, video_sample_type="weighted_kmeans", video_max_frames=50)
        base.update(cfg)
        self.config = SimpleNamespace(**base)
        self._model = _ModelHost(attention_model, vision_tower)
        self.use_video_streaming_mode = True
        self.video_embedding_memory = []
        from torch.multiprocessing import Lock      # what the reference hangs there (vstream_arch.py:24,150): shared with a
        self.video_embedding_mem_lock = Lock()      # spawned memory-manager process when the model is passed to it

    def get_model(self):
        return self._model
