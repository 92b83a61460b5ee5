"""Timing script (not a pytest file): many Qwen2-VL streams on one GPU, batched (QwenStreamPool.step: one tower call, one
PatchMerger call and one host wait per round) against the same streams stepped one after the other (per stream: the
host's tower pass, forward_simple_not_merge, then QwenStreamState.step with its own host wait).

336 px (24 x 24 patches, 576 + 144 tower rows per temporal patch), the 32-layer tower (seeded weights, bf16), the
default Flash Memory config (CSM 60 frames, DAM 30), pixels in HBM.  For S in --streams, three rows:
  - t1_filling: single-patch clips (the reference CLI's steady state) while the memory fills (T <= 60);
  - t1_full:    single-patch clips once the CSM k-means runs every step;
  - t8_full:    8-patch clips, memory full.
Each row runs warm-up rounds and then at least --seconds of CUDA-event-timed rounds, batched and sequential alternated
per window.  Reported per round: ms, tower ms (CUDA events around the tower calls), memory ms (round minus tower) and the
host waits (event synchronisations) of one round.  The card's name and power limit are read with nvidia-smi in the same
run.  At the end every batched stream is checked bit for bit against its sequential twin.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return dict(zip(q.split(","), [v.strip() for v in out[0].split(",")])) if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--streams", default="1,2,4,8,16,32")
    ap.add_argument("--seconds", type=float, default=3.0, help="timed seconds per row and mode (at least)")
    ap.add_argument("--depth", type=int, default=32)
    a = ap.parse_args()
    import torch
    torch.set_grad_enabled(False)
    if not torch.cuda.is_available():
        raise SystemExit("gpu_qwen_multistream_timing.py needs a CUDA device")
    from flash_vstream_b200.draws import DrawSource
    from flash_vstream_b200.qwen import QwenStreamPool, QwenStreamState
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
    visual = host.visual
    g = torch.Generator().manual_seed(0)
    scenes = [torch.randn(576, 1176, generator=g) for _ in range(12)]
    src = torch.stack([scenes[i // 5 % 12] + 0.3 * torch.randn(576, 1176, generator=g) for i in range(256)]).bfloat16().to(dev)
    thw = {t: torch.tensor([[t, 24, 24]]) for t in (1, 8)}

    def clip(r, i, t):
        k = (r * 7 + i * 13) % (src.shape[0] - t)
        return src[k: k + t].reshape(-1, 1176), thw[t]

    # tower time inside a round: CUDA events around every tower call (both modes call the same QwenVisionBlocksB200)
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

    waits = [0]
    sync0 = torch.cuda.Event.synchronize

    def counting_sync(self):
        waits[0] += 1
        return sync0(self)

    def batched(S, seed0):
        pool = QwenStreamPool(host)
        pool.tower = Timed(tower)
        sids = [pool.open(seed=seed0 + i) for i in range(S)]

        def round_fn(r, t):
            pool.step({s: clip(r, i, t) for i, s in enumerate(sids)})
        return [pool.state(s) for s in sids], round_fn

    def sequential(S, seed0):
        states = []
        for i in range(S):
            st = QwenStreamState(visual.flash_memory, merger)
            st.rng = DrawSource(seed0 + i, dev)
            states.append(st)
        timed_visual = rt.VisualB200(visual.flash_memory, merger, encode_patches=Timed(tower))

        def round_fn(r, t):
            for i, st in enumerate(states):
                pix, grid = clip(r, i, t)
                feats, _, _ = timed_visual.forward_simple_not_merge(pix, grid)
                n = t * 576
                st.step(feats[:n], feats[n: n + n // 4], t, (24, 24), (12, 12), st.n_frames)
        return states, round_fn

    def measure(fns, t, rounds_from, seconds, renew=None):
        """alternate the modes window by window; -> {mode: (ms, tower ms, waits) per round}.  renew(mode) -> a fresh
        round function, or None to keep the current one (between windows, outside the timed region)"""
        tot = {m: [0.0, 0.0, 0] for m in fns}
        r = dict(rounds_from)
        torch.cuda.Event.synchronize = counting_sync
        try:
            for m, fn in fns.items():                       # host waits of one round
                waits[0] = 0
                fn(r[m], t)
                r[m] += 1
                tot[m].append(waits[0])
            torch.cuda.synchronize()
            while min(v[0] for v in tot.values()) < seconds * 1e3:
                for m in list(fns):
                    fresh = renew(m) if renew is not None else None
                    if fresh is not None:
                        fns[m], r[m] = fresh, 0
                    fn = fns[m]
                    spans.clear()
                    e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                    e0.record()
                    for _ in range(4):
                        fn(r[m], t)
                        r[m] += 1
                    e1.record()
                    sync0(e1)
                    tot[m][0] += e0.elapsed_time(e1)
                    tot[m][1] += sum(x.elapsed_time(y) for x, y in spans)
                    tot[m][2] += 4
        finally:
            torch.cuda.Event.synchronize = sync0
        return {m: (v[0] / v[2], v[1] / v[2], v[3]) for m, v in tot.items()}, r

    rows, identical = [], True
    for S in [int(s) for s in a.streams.split(",")]:
        row = {"S": S}
        for name, t, warm_to in (("t1_filling", 1, 4), ("t1_full", 1, 64), ("t8_full", 8, 12)):
            made = {"batched": batched(S, 100), "sequential": sequential(S, 100)}
            fns = {m: v[1] for m, v in made.items()}
            for k in range(warm_to):                        # warm up (and, for the full rows, fill the memory)
                for m, fn in fns.items():
                    fn(k, t)
            r = {m: warm_to for m in fns}
            renew = None
            if name == "t1_filling":                        # fresh streams before the CSM would run its k-means
                def renew(m, made=made):
                    if made[m][0][0].n_frames + 5 <= 60:
                        return None
                    made[m] = (batched if m == "batched" else sequential)(S, 100)
                    return made[m][1]
            res, r = measure(fns, t, r, a.seconds, renew)
            for m, (ms, tower_ms, w) in res.items():
                row[f"{name}_{m}_ms_per_round"] = ms
                row[f"{name}_{m}_tower_ms_per_round"] = tower_ms
                row[f"{name}_{m}_memory_ms_per_round"] = ms - tower_ms
                row[f"{name}_{m}_host_waits_per_round"] = w
            row[f"{name}_speedup"] = res["sequential"][0] / res["batched"][0]
            b, s = made["batched"][0], made["sequential"][0]
            for x, y in zip(b, s):
                same = (x.n_frames == y.n_frames and x.steps == y.steps and x.fast_steps == y.fast_steps and
                        x.redone_steps == y.redone_steps and
                        all(torch.equal(u, v) if torch.is_tensor(u) else u == v for u, v in zip(x.as_list(), y.as_list())))
                x.rng.settle()
                y.rng.settle()
                same = same and torch.equal(x.rng.cpu, y.rng.cpu) and x.rng.py.getstate() == y.rng.py.getstate()
                identical = identical and same
            row[f"{name}_frames_end"] = b[0].n_frames
            del made, fns, renew, b, s, x, y            # the banks of 2 S streams: free them before the next row
            torch.cuda.empty_cache()
        row["sm_clock_after"] = (gpu_info() or {}).get("clocks.sm")
        rows.append(row)
        print(json.dumps({"partial": row}), file=sys.stderr, flush=True)

    out = {"metric": "qwen_multistream_rounds", "tower": f"Qwen2-VL vision tower, {a.depth} layers (seeded weights, bf16), 336 px",
           "config": "FlashMemory defaults (CSM 60 frames, DAM 30, klarge_retrieve)", "gpu_before": info_before,
           "gpu_after": gpu_info(), "rows": rows, "batched_equals_sequential_bits": identical,
           "time": time.strftime("%Y-%m-%d %H:%M:%S")}
    print(json.dumps(out), flush=True)
    if not identical:
        raise SystemExit("batched streams differ from the sequential ones")


if __name__ == "__main__":
    main()
