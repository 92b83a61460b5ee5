"""Timing script (not a pytest file): QwenStreamPool rounds in three modes, alternated in one run: eager, lazy_full_res
(DESIGN.md §3.18) and lazy_full_res without a full-resolution bank (full_res_bank=False, §3.19), which re-encodes every
pick its previous DAM does not hold.

336 px (24 x 24 patches), the 32-layer tower (seeded weights, bf16), the default Flash Memory config (CSM 60 frames,
DAM 30), and the piecewise-stationary streams of gpu_qwen_lazy_timing.py (a scene plus noise, a new scene every 16 to
64 frames).  For S in --streams and t in (1, 8) temporal patches per clip, the three pools are warmed up until their
memory is full (past the CSM length), then timed over windows of --window rounds, the modes alternated, for at least
--seconds each, or until the streams would pass max(128, 4096 / S) frames (at least one window).  A row repeats such
passes, with fresh pools and streams, until each mode has at least --min-rounds timed rounds.  Per row and mode: round
ms (CUDA events around QwenStreamPool.step), tower ms (CUDA events around every tower call), full-resolution encodes per
stream and step and how many of them re-encode a frame encoded before, the peak HBM per stream (as in
gpu_qwen_lazy_timing.py) and the pinned host bytes per stream the pool holds at the end of that measurement.  At the
end of every pass each lazy and bank-less stream is checked bit for bit against its eager twin.  The card's name,
power limit and SM clock are read with nvidia-smi in the same run.

--baseline-tree DIR also times bench.py's qwen_stream row from DIR (another built checkout, e.g. the parent commit) and
from this tree, alternated, twice each.  Prints one JSON line."""
import argparse
import gc
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.gpu_qwen_lazy_timing import qwen_row  # noqa: E402
from tests.gpu_qwen_multistream_timing import gpu_info  # noqa: E402

MODES = {"eager": dict(lazy_full_res=False), "lazy": dict(lazy_full_res=True),
         "no_bank": dict(lazy_full_res=True, full_res_bank=False)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="1,4,16,32")
    ap.add_argument("--seconds", type=float, default=2.0, help="timed seconds per row and mode (at least)")
    ap.add_argument("--window", type=int, default=4, help="rounds per timed window")
    ap.add_argument("--min-rounds", type=int, default=12, help="timed rounds per row and mode (at least)")
    ap.add_argument("--depth", type=int, default=32)
    ap.add_argument("--baseline-tree", default=None)
    a = ap.parse_args()
    import torch
    torch.set_grad_enabled(False)
    if not torch.cuda.is_available():
        raise SystemExit("gpu_qwen_no_bank_timing.py needs a CUDA device")
    from flash_vstream_b200 import ops as O
    from flash_vstream_b200.qwen import QwenStreamPool
    from flash_vstream_b200.qwen import ops as Q
    from flash_vstream_b200.qwen import vstream_qwen2vl_realtime as rt
    from flash_vstream_b200.qwen.vision_tower import QwenVisionBlocksB200
    from tests import qwen_rt_inputs as RI
    from tests import qwen_vit_inputs as VI

    out = {"gpu_before": gpu_info()}
    print(json.dumps(out), file=sys.stderr, flush=True)
    dev = torch.device("cuda", 0)
    torch.cuda.set_device(dev)
    tower = QwenVisionBlocksB200(VI.state_dict(dict(depth=a.depth, embed=1280, heads=16, seed=5), "bf16"), depth=a.depth,
                                 heads=16, dtype=torch.bfloat16)
    merger = rt.PatchMerger.from_weights({k: v.cuda() for k, v in RI.merger_weights(1280, 3584, "bf16", 7).items()})
    host = rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(rt.FlashMemory(), merger, encode_patches=tower))
    h = w = 24
    T0 = host.visual.flash_memory.temporal_length

    class Timed:
        """the tower with CUDA events around each call"""

        def __init__(self, inner):
            self.inner, self.events = inner, []

        def __call__(self, *args):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            y = self.inner(*args)
            e1.record()
            self.events.append((e0, e1))
            return y

    class Stream:
        """a piecewise-stationary pixel stream: scene + noise, a new scene every 16..64 frames"""

        def __init__(self, seed):
            self.g = torch.Generator(device="cuda").manual_seed(seed)
            self.left, self.scene = 0, None

        def clip(self, t):
            rows = []
            for _ in range(t):
                if self.left <= 0:
                    self.scene = torch.randn(h * w, 1176, device="cuda", generator=self.g)
                    self.left = int(torch.randint(8, 33, (1,), generator=self.g, device="cuda"))   # patches = 2 frames
                self.left -= 1
                rows.append(self.scene + 0.2 * torch.randn(h * w, 1176, device="cuda", generator=self.g))
            return torch.cat(rows).bfloat16(), torch.tensor([[t, h, w]])

    def open_pool(mode, S, timed, seed0):
        pool = QwenStreamPool(host, **MODES[mode])
        pool.tower = timed
        sids = [pool.open(seed=seed0 + i) for i in range(S)]
        for sid in sids:
            pool.state(sid).tower = timed
        return pool, sids

    def counts(pool, sids, mode):
        """(full-resolution encodes, re-encodes) of the pool's streams so far"""
        st = [pool.state(x) for x in sids]
        if mode == "eager":
            return sum(x.n_frames for x in st), 0
        return sum(x.n_encoded for x in st), sum(x.re_encode_count() for x in st)

    def fresh():
        """drop the workspace caches of earlier pools: a measurement sees what its own pool allocates"""
        gc.collect()
        Q._ws_cache.clear()
        O._km_ws_cache.clear()
        torch.cuda.synchronize()
        torch.cuda.empty_cache()

    results = []
    for S in [int(s) for s in a.streams.split(",")]:
        for t in (1, 8):
            warm = (T0 + 2 * t) // t + 2                          # past the CSM length: the k-means runs every round
            cap = max(128, 4096 // S)
            acc = {mode: dict(ms=[], tower_ms=[], rounds=0, enc=0, again=0, frames=0) for mode in MODES}
            row = {"S": S, "t": t, "bit_exact": True, "passes": 0}
            while min(v["rounds"] for v in acc.values()) < a.min_rounds:
                p = row["passes"]
                modes = {}
                for mode in MODES:
                    timed = Timed(tower)
                    pool, sids = open_pool(mode, S, timed, 100 + 1000 * p)
                    modes[mode] = dict(pool=pool, sids=sids, timed=timed,
                                       src=[Stream(7 + 1000 * p + i) for i in range(S)], **acc[mode])

                def one_round(m):
                    m["pool"].step({sid: s.clip(t) for sid, s in zip(m["sids"], m["src"])})

                for _ in range(warm):
                    for m in modes.values():
                        one_round(m)
                c0 = {mode: counts(m["pool"], m["sids"], mode) for mode, m in modes.items()}
                torch.cuda.synchronize()
                spent, timed_here = 0.0, 0
                while spent < a.seconds * 1e3:
                    if timed_here and modes["eager"]["pool"].state(modes["eager"]["sids"][0]).n_frames + a.window * t > cap:
                        break
                    for m in modes.values():
                        m["timed"].events.clear()
                        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                        e0.record()
                        for _ in range(a.window):
                            one_round(m)
                        e1.record()
                        e1.synchronize()
                        m["ms"].append(e0.elapsed_time(e1))
                        m["tower_ms"].append(sum(x.elapsed_time(y) for x, y in m["timed"].events))
                        m["rounds"] += a.window
                    timed_here += a.window
                    spent = min(sum(m["ms"]) for m in modes.values())
                for mode, m in modes.items():
                    enc, again = counts(m["pool"], m["sids"], mode)
                    acc[mode]["ms"], acc[mode]["tower_ms"], acc[mode]["rounds"] = m["ms"], m["tower_ms"], m["rounds"]
                    acc[mode]["enc"] += enc - c0[mode][0]
                    acc[mode]["again"] += again - c0[mode][1]
                    acc[mode]["frames"] = m["pool"].state(m["sids"][0]).n_frames
                ep = modes["eager"]["pool"]
                for mode in ("lazy", "no_bank"):
                    mp = modes[mode]["pool"]
                    for x, y in zip(modes[mode]["sids"], modes["eager"]["sids"]):
                        for i, (u, v) in enumerate(zip(mp.state(x).as_list(), ep.state(y).as_list())):
                            if i != 7 and torch.is_tensor(u) and not (u.shape == v.shape and torch.equal(u.cpu(), v.cpu())):
                                row["bit_exact"] = False
                row["passes"] += 1
                del modes, ep, mp
                fresh()
            # peak HBM and pinned host bytes: each mode alone, from an empty allocator state to full memory and `window`
            # rounds past it
            for mode in MODES:
                base = torch.cuda.memory_allocated()
                pool, sids = open_pool(mode, S, tower, 5000)
                src = [Stream(5000 + i) for i in range(S)]
                torch.cuda.reset_peak_memory_stats()
                for _ in range(warm + a.window):
                    pool.step({sid: x.clip(t) for sid, x in zip(sids, src)})
                torch.cuda.synchronize()
                acc[mode]["peak"] = (torch.cuda.max_memory_allocated() - base) / S
                acc[mode]["pinned"] = sum(pool.state(x).pinned_bytes() for x in sids) / S
                acc[mode]["pinned_frames"] = pool.state(sids[0]).n_frames
                del pool, sids, src
                fresh()
            for mode, v in acc.items():
                steps = v["rounds"] * S
                row[mode] = {
                    "round_ms": round(sum(v["ms"]) / v["rounds"], 3), "tower_ms": round(sum(v["tower_ms"]) / v["rounds"], 3),
                    "full_res_encodes_per_stream_step": round(v["enc"] / steps, 3),
                    "re_encodes_per_stream_step": round(v["again"] / steps, 3),
                    "peak_hbm_mb_per_stream": round(v["peak"] / 2 ** 20, 1),
                    "pinned_mb_per_stream": round(v["pinned"] / 2 ** 20, 1), "pinned_at_frames": v["pinned_frames"],
                    "rounds": v["rounds"], "frames_per_stream_at_end": v["frames"]}
            row["no_bank_vs_lazy_round"] = round(row["lazy"]["round_ms"] / row["no_bank"]["round_ms"], 3)
            row["no_bank_vs_eager_round"] = round(row["eager"]["round_ms"] / row["no_bank"]["round_ms"], 3)
            results.append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
    out["rows"] = results
    tower.close()                                          # the baseline runs below need the HBM
    del host, tower, merger
    torch.cuda.empty_cache()
    if a.baseline_tree:
        rows = []
        for _ in range(2):
            rows.append({"baseline": qwen_row(a.baseline_tree), "this": qwen_row(ROOT)})
            print(json.dumps(rows[-1]), file=sys.stderr, flush=True)
        out["qwen_stream_row"] = rows
    out["gpu_after"] = gpu_info()
    print(json.dumps(out))


if __name__ == "__main__":
    main()
