"""Timing script (not a pytest file): QwenStreamPool rounds fed uint8 frames, with and without compact_pixels (DESIGN.md
§3.20), for lazy (§3.18) and bank-less (§3.19) pools, the four pools alternated in one run.

336 px frames (24 x 24 patches), the 32-layer tower (seeded weights, bf16), the default Flash Memory config, and
piecewise-stationary uint8 streams (a scene plus noise, a new scene every 16 to 64 frames).  For S in --streams and t in
(1, 8) temporal patches per clip, the pools are warmed up past the CSM length, then timed over windows of --window
rounds, alternated, until each has --min-rounds timed rounds.  Per row and pool: round ms (CUDA events around
QwenStreamPool.step, pre-processing included), tower ms (CUDA events around every tower call), pinned host bytes per
stream at the end, the pixel-store D2H bytes per round (the round's pixel rows or codes) and the re-encode H2D bytes
per round (the rows or codes the pixel gather reads).  Every compact stream is checked bit for bit against its twin.
The card's name, power limit and SM clock are read with nvidia-smi in the same run.

--baseline-tree DIR also times bench.py's qwen_stream row from DIR (another built checkout, e.g. the parent commit) and
from this tree, alternated, twice each.  Prints one JSON line."""
import argparse
import json
import os
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.gpu_qwen_lazy_timing import qwen_row  # noqa: E402
from tests.gpu_qwen_multistream_timing import gpu_info  # noqa: E402

MODES = {"lazy": dict(lazy_full_res=True), "lazy_compact": dict(lazy_full_res=True, compact_pixels=True),
         "no_bank": dict(lazy_full_res=True, full_res_bank=False),
         "no_bank_compact": dict(lazy_full_res=True, full_res_bank=False, compact_pixels=True)}


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="1,4,16")
    ap.add_argument("--window", type=int, default=4, help="rounds per timed window")
    ap.add_argument("--min-rounds", type=int, default=12, help="timed rounds per row and pool (at least)")
    ap.add_argument("--depth", type=int, default=32)
    ap.add_argument("--baseline-tree", default=None)
    a = ap.parse_args()
    import torch
    torch.set_grad_enabled(False)
    if not torch.cuda.is_available():
        raise SystemExit("gpu_qwen_compact_pixels_timing.py needs a CUDA device")
    from flash_vstream_b200 import preprocess as P
    from flash_vstream_b200.qwen import QwenStreamPool
    from flash_vstream_b200.qwen import vstream_qwen2vl_realtime as rt
    from flash_vstream_b200.qwen.vision_tower import QwenVisionBlocksB200
    from tests import qwen_rt_inputs as RI
    from tests import qwen_vit_inputs as VI

    out = {"gpu_before": gpu_info()}
    print(json.dumps(out), file=sys.stderr, flush=True)
    torch.cuda.set_device(0)
    tower = QwenVisionBlocksB200(VI.state_dict(dict(depth=a.depth, embed=1280, heads=16, seed=5), "bf16"), depth=a.depth,
                                 heads=16, dtype=torch.bfloat16)
    merger = rt.PatchMerger.from_weights({k: v.cuda() for k, v in RI.merger_weights(1280, 3584, "bf16", 7).items()})
    host = rt.FlashVStreamQwen2VLRealtimeB200(rt.VisualB200(rt.FlashMemory(), merger, encode_patches=tower))
    proc = P.Qwen2VLFramePreprocessor()
    side, hw = 336, 24 * 24
    T0 = host.visual.flash_memory.temporal_length

    class Timed:
        def __init__(self):
            self.events = []

        def __call__(self, *args):
            e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
            e0.record()
            y = tower(*args)
            e1.record()
            self.events.append((e0, e1))
            return y

    class Stream:
        """piecewise-stationary uint8 frames: scene + noise, a new scene every 16..64 frames"""

        def __init__(self, seed):
            self.g = torch.Generator(device="cuda").manual_seed(seed)
            self.left, self.scene = 0, None

        def clip(self, t):
            out = []
            for _ in range(2 * t):
                if self.left <= 0:
                    self.scene = torch.randint(0, 256, (side, side, 3), device="cuda", generator=self.g).float()
                    self.left = int(torch.randint(16, 65, (1,), generator=self.g, device="cuda"))
                self.left -= 1
                noise = 12 * torch.randn(side, side, 3, device="cuda", generator=self.g)
                out.append((self.scene + noise).clamp(0, 255).to(torch.uint8))
            return torch.stack(out)

    results = []
    for S in [int(s) for s in a.streams.split(",")]:
        for t in (1, 8):
            pools = {}
            for mode, kw in MODES.items():
                timed = Timed()
                pool = QwenStreamPool(host, preprocess=proc, **kw)
                pool.tower = timed
                sids = [pool.open(seed=100 + i) for i in range(S)]
                for sid in sids:
                    pool.state(sid).tower = timed
                pools[mode] = dict(pool=pool, sids=sids, timed=timed, src=[Stream(7 + i) for i in range(S)], ms=[],
                                   tower_ms=[], rounds=0)

            def one_round(m):
                m["pool"].step({sid: s.clip(t) for sid, s in zip(m["sids"], m["src"])})

            for _ in range((T0 + 2 * t) // t + 2):
                for m in pools.values():
                    one_round(m)
            enc0 = {mode: sum(m["pool"].state(x).n_encoded for x in m["sids"]) for mode, m in pools.items()}
            torch.cuda.synchronize()
            while min(m["rounds"] for m in pools.values()) < a.min_rounds:
                for m in pools.values():
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
            row = {"S": S, "t": t, "bit_exact": True}
            for mode, m in pools.items():
                pool, sids = m["pool"], m["sids"]
                elem = 1 if "compact" in mode else 2
                enc = sum(pool.state(x).n_encoded for x in sids) - enc0[mode]
                row[mode] = {"round_ms": round(sum(m["ms"]) / m["rounds"], 3),
                             "tower_ms": round(sum(m["tower_ms"]) / m["rounds"], 3),
                             "pinned_mb_per_stream": round(sum(pool.state(x).pinned_bytes() for x in sids) / S / 2 ** 20, 2),
                             "pixel_d2h_mb_per_round": round(S * t * hw * 1176 * elem / 2 ** 20, 2),
                             "re_encode_h2d_mb_per_round": round(enc / m["rounds"] * hw * 1176 * elem / 2 ** 20, 2),
                             "frames_per_stream_at_end": pool.state(sids[0]).n_frames, "rounds": m["rounds"]}
            for base in ("lazy", "no_bank"):
                bp, cp = pools[base], pools[base + "_compact"]
                for x, y in zip(cp["sids"], bp["sids"]):
                    for i, (u, v) in enumerate(zip(cp["pool"].state(x).as_list(), bp["pool"].state(y).as_list())):
                        if torch.is_tensor(u) and not (u.shape == v.shape and torch.equal(u.cpu(), v.cpu())):
                            row["bit_exact"] = False
                row[base + "_compact_speedup"] = round(row[base]["round_ms"] / row[base + "_compact"]["round_ms"], 3)
            results.append(row)
            print(json.dumps(row), file=sys.stderr, flush=True)
            del pools
            torch.cuda.synchronize()
            torch.cuda.empty_cache()
    out["rows"] = results
    tower.close()
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
