"""Timing script (not a pytest file): the memory part of a QwenStreamPool round with the CSM half batched over the
streams (the default BATCH_MIN_JOBS: one job table per kernel, DESIGN.md §3.17) against a pool whose BATCH_MIN_JOBS is
above S, so each stream steps its memory in a one-item call, as it does alone; same tower, same clips.

Setup and windows of gpu_qwen_multistream_timing.py: 336 px, the 32-layer tower (seeded weights, bf16), the default
Flash Memory (CSM 60 frames, DAM 30), single-patch clips, memory full (64 warm-up rounds).  Both modes alternate window
by window; memory ms per round = round ms minus the tower calls' ms (CUDA events around every tower call).  At the end
of every row each batched stream is checked bit for bit against its per-stream twin.  Prints one JSON line; the card's
name, power limit and clocks are read with nvidia-smi in the same run."""
import argparse
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.gpu_qwen_multistream_timing import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="1,2,4,8,16,32")
    ap.add_argument("--seconds", type=float, default=2.0, help="timed seconds per row and mode (at least)")
    ap.add_argument("--depth", type=int, default=32)
    ap.add_argument("--out", default=None)
    a = ap.parse_args()
    import torch
    torch.set_grad_enabled(False)
    if not torch.cuda.is_available():
        raise SystemExit("gpu_qwen_mem_multi_timing.py needs a CUDA device")
    from flash_vstream_b200.qwen import QwenStreamPool
    from flash_vstream_b200.qwen import vstream_qwen2vl_realtime as rt
    from flash_vstream_b200.qwen.vision_tower import QwenVisionBlocksB200
    from tests import qwen_rt_inputs as RI
    from tests import qwen_vit_inputs as VI

    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    info_before = gpu_info()
    tower = QwenVisionBlocksB200(VI.state_dict(dict(depth=a.depth, embed=1280, heads=16, seed=5), "bf16"), depth=a.depth,
                                 heads=16, dtype=torch.bfloat16)
    merger = rt.PatchMerger.from_weights({k: v.cuda() for k, v in RI.merger_weights(1280, 3584, "bf16", 7).items()})
    host = rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(rt.FlashMemory(), merger, encode_patches=tower))
    g = torch.Generator().manual_seed(0)
    scenes = [torch.randn(576, 1176, generator=g) for _ in range(12)]
    src = torch.stack([scenes[i // 5 % 12] + 0.3 * torch.randn(576, 1176, generator=g) for i in range(256)]).bfloat16().to(dev)
    thw = torch.tensor([[1, 24, 24]])
    spans = []

    class Timed:
        def __init__(self, inner):
            self.inner = inner

        def __call__(self, *args):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            out = self.inner(*args)
            e1.record()
            spans.append((e0, e1))
            return out

    def make(S, batch):
        pool = QwenStreamPool(host)
        if not batch:
            pool.BATCH_MIN_JOBS = S + 1
        pool.tower = Timed(tower)
        sids = [pool.open(seed=100 + i) for i in range(S)]

        def round_fn(r):
            pool.step({s: (src[(r * 7 + i * 13) % 255].reshape(-1, 1176), thw) for i, s in enumerate(sids)})
        return pool, sids, round_fn

    rows, identical = [], True
    for S in [int(s) for s in a.streams.split(",")]:
        made = {"batched": make(S, True), "per_stream": make(S, False)}
        for k in range(64):                                       # fill the memory: the CSM k-means runs every step
            for m in made.values():
                m[2](k)
        tot = {m: [0.0, 0.0, 0] for m in made}
        r = 64
        torch.cuda.synchronize()
        while min(v[0] for v in tot.values()) < a.seconds * 1e3:
            for name, (_, _, fn) in made.items():
                spans.clear()
                e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                e0.record()
                for i in range(4):
                    fn(r + i)
                e1.record()
                e1.synchronize()
                tot[name][0] += e0.elapsed_time(e1)
                tot[name][1] += sum(x.elapsed_time(y) for x, y in spans)
                tot[name][2] += 4
            r += 4
        row = {"S": S, "batched_batch_min_jobs": made["batched"][0].BATCH_MIN_JOBS,
               "per_stream_batch_min_jobs": made["per_stream"][0].BATCH_MIN_JOBS}
        for name, (ms, tower_ms, n) in tot.items():
            row[f"{name}_ms_per_round"] = ms / n
            row[f"{name}_tower_ms_per_round"] = tower_ms / n
            row[f"{name}_memory_ms_per_round"] = (ms - tower_ms) / n
        row["memory_speedup"] = row["per_stream_memory_ms_per_round"] / row["batched_memory_ms_per_round"]
        (pa, sa, _), (pb, sb, _) = made["batched"], made["per_stream"]
        for x, y in zip(sa, sb):
            u, v = pa.state(x), pb.state(y)
            same = (u.n_frames == v.n_frames and u.steps == v.steps and u.fast_steps == v.fast_steps and
                    all(torch.equal(p, q) if torch.is_tensor(p) else p == q for p, q in zip(u.as_list(), v.as_list())))
            u.rng.settle()
            v.rng.settle()
            identical = identical and same and torch.equal(u.rng.cpu, v.rng.cpu) and u.rng.py.getstate() == v.rng.py.getstate()
        row["identical"] = identical
        row["frames_end"] = pa.state(sa[0]).n_frames
        row["sm_clock_after"] = (gpu_info() or {}).get("clocks.sm")
        rows.append(row)
        print(json.dumps({"partial": row}), file=sys.stderr, flush=True)
        del made, pa, pb
        torch.cuda.empty_cache()
    out = {"metric": "qwen_mem_multi_rounds", "tower": f"Qwen2-VL vision tower, {a.depth} layers (seeded weights, bf16), 336 px",
           "config": "FlashMemory defaults (CSM 60 frames, DAM 30, klarge_retrieve), single-patch clips, memory full",
           "gpu_before": info_before, "gpu_after": gpu_info(), "rows": rows, "batched_equals_per_stream_bits": identical,
           "time": time.strftime("%Y-%m-%d %H:%M:%S")}
    line = json.dumps(out)
    print(line, flush=True)
    if a.out:
        os.makedirs(os.path.dirname(os.path.abspath(a.out)), exist_ok=True)
        with open(a.out, "w") as f:
            f.write(line + "\n")
    if not identical:
        raise SystemExit("batched memory differs from the per-stream memory")


if __name__ == "__main__":
    main()
