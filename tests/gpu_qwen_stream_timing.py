"""End-to-end timing of the Qwen2-VL streaming step on one GPU (not a test):
    python tests/gpu_qwen_stream_timing.py > qwen_stream_timing.json
Every step = embed_new_video_clip on a clip of `t_clip` temporal patches (2 frames each) of a 336 x 336 stream with pixels
coming from pinned host memory: temporal_pool -> 32-layer sm_90a tower -> CSM k-means (61..62 -> 60 once the memory is
full) -> DAM retrieval of 30 frames over the growing bank -> PatchMerger of the 6480 memory tokens.  Wall clock per step is
taken with CUDA events around the whole call; the per-stage host timestamps are the reference's own 8 buckets (they are
host times with a synchronize inserted between stages ONLY in the breakdown pass)."""
import json
import os
import sys
import time

import numpy as np
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from flash_vstream_b200.qwen import vstream_qwen2vl_realtime as rt  # noqa: E402
from flash_vstream_b200.qwen.vision_tower import QwenVisionBlocksB200  # noqa: E402
from tests import qwen_rt_inputs as RI  # noqa: E402
from tests import qwen_vit_inputs as VI  # noqa: E402


def measure(depth=None, t_clip=None, steps=None, breakdown=True, prefill_patches=None):
    """returns the dict described in the module docstring (also called by bench.py's `rows.qwen_stream`, outside its timed region).
    prefill_patches: once the memory is full, append that many temporal patches of synthetic FEATURES to the three banks (full
    resolution, half resolution, merged) — the state of a stream that has been running for 2 x prefill_patches frames,
    without spending the minutes it takes to get there; the timed steps then retrieve from that bank."""
    prefill_patches = int(os.environ.get("QPREFILL", 0)) if prefill_patches is None else prefill_patches
    depth = int(os.environ.get("QVIT_DEPTH", 32)) if depth is None else depth
    t_clip = int(os.environ.get("QCLIP", 2)) if t_clip is None else t_clip
    steps = int(os.environ.get("QSTEPS", 60)) if steps is None else steps
    torch.set_grad_enabled(False)
    sd = VI.state_dict(dict(depth=depth, embed=1280, heads=16, seed=5), "bf16")
    tower = QwenVisionBlocksB200(sd, depth=depth, heads=16, dtype=torch.bfloat16, use_graphs=os.environ.get("QGRAPH", "0") == "1")
    merger = rt.PatchMerger.from_weights({k: v.cuda() for k, v in RI.merger_weights(1280, 3584, "bf16", 7).items()})
    host = rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(rt.FlashMemory(), merger, encode_patches=tower))
    g = torch.Generator().manual_seed(0)
    scenes = [torch.randn(576, 1176, generator=g) for _ in range(12)]
    clips = []
    for s in range(steps + 8):               # one pinned clip per step: a stream never shows the same frame twice (a repeated
        rows = torch.cat([scenes[(s * t_clip + i) // 5 % 12] + 0.3 * torch.randn(576, 1176, generator=g)   # frame duplicates
                          for i in range(t_clip)])                                                            # a CSM row)
        clips.append(rows.bfloat16().pin_memory())
    thw = torch.tensor([[t_clip, 24, 24]])
    torch.manual_seed(0)
    ms = []
    s_fill = 60 // t_clip + 1                # pre-fill once the CSM holds its 60 centroids (a long bank implies a full memory)
    for s in range(steps):
        a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        a.record()
        host.embed_new_video_clip(clips[s], thw, s * t_clip)
        b.record()
        torch.cuda.synchronize()
        ms.append(a.elapsed_time(b))
        if s == s_fill and prefill_patches:
            st = host.stream_state
            gd = torch.Generator(device="cuda").manual_seed(1)
            for c0 in range(0, prefill_patches, 256):
                n = min(256, prefill_patches - c0)
                st.bank_x.append(torch.randn(n, 576, 1280, device="cuda", generator=gd).bfloat16())
                st.bank_small.append(torch.randn(n, 144, 1280, device="cuda", generator=gd).bfloat16())
                st.bank_merged.append(torch.randn(n, 144, 3584, device="cuda", generator=gd).bfloat16())
            st.n_frames += prefill_patches
            with host.video_embedding_mem_lock:
                host.video_embedding_memory[:] = st.as_list()
            torch.cuda.synchronize()
    full = [m for i, m in enumerate(ms) if (i + 1) * t_clip > 60 + t_clip]      # steps with a full CSM (k-means runs)
    if prefill_patches:
        full = ms[s_fill + 1:]                                                   # ... and the long bank
    mem = host.video_embedding_memory
    out = {"depth": depth, "t_clip": t_clip, "steps": steps, "prefill_patches": prefill_patches, "tower_cuda_graph": tower.use_graphs, "bank_frames_end": int(mem[8][0]),
           "memory_tokens": int(mem[11].shape[0]),
           "ms_per_step_warmup_phase": float(np.median(ms[3:max(4, 60 // t_clip)])),
           "ms_per_step_full_memory": float(np.median(full)) if full else None,
           "temporal_patches_per_s_full_memory": t_clip / float(np.median(full)) * 1e3 if full else None,
           "frames_per_s_full_memory": 2 * t_clip / float(np.median(full)) * 1e3 if full else None,
           "steps_single_pass": host.stream_state.fast_steps, "steps_redone_for_duplicates": host.stream_state.redone_steps}
    if not breakdown:
        tower.close()
        return out
    # breakdown pass: synchronise at the reference's bucket boundaries (perturbs the total; for shares only)
    orig_fsm = host.visual.forward_simple_not_merge
    marks = {}

    def timed_fsm(*a, **k):
        torch.cuda.synchronize(); t0 = time.perf_counter()
        r = orig_fsm(*a, **k)
        torch.cuda.synchronize(); marks["tower"] = marks.get("tower", 0.0) + (time.perf_counter() - t0) * 1e3
        return r
    host.visual.forward_simple_not_merge = timed_fsm
    from flash_vstream_b200.qwen import compress_functions as CF
    orig_km, orig_se, orig_mg = CF.ordered_kmeans_enqueue_multi, host.visual.flash_memory.spatial_enhance, host.visual.merger.forward

    def wrap(fn, key):
        def f(*a, **k):
            torch.cuda.synchronize(); t0 = time.perf_counter()
            r = fn(*a, **k)
            torch.cuda.synchronize(); marks[key] = marks.get(key, 0.0) + (time.perf_counter() - t0) * 1e3
            return r
        return f
    CF.ordered_kmeans_enqueue_multi = wrap(orig_km, "temporal_compress")  # the k-means of the CSM (stream_state.py)
    host.visual.flash_memory.spatial_enhance = wrap(orig_se, "spatial_enhance")
    host.visual.merger.forward = wrap(orig_mg, "merger")
    acc = {}
    for s in range(steps, steps + 8):
        marks.clear()
        host.embed_new_video_clip(clips[s], thw, s * t_clip)
        for k, v in marks.items():
            acc.setdefault(k, []).append(v)
    CF.ordered_kmeans_enqueue_multi = orig_km
    out["breakdown_ms_synchronised"] = {k: float(np.median(v)) for k, v in acc.items()}   # merger = new frames + CSM rows
    return out


if __name__ == "__main__":
    print(json.dumps(measure()))
