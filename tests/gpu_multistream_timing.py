"""Timing script (not a pytest file): many single-frame streams on one GPU, batched (StreamPool.step, one
fvs_stream_step_multi per round) against the same streams stepped one after the other (StreamBank.step per stream: a
one-bank call, so one consolidation launch per stream).

ViT-L/14 at 336 px (random weights, 23 layers run, f16) and the default 681-token STAR config; every step takes one frame
from device-resident pixels, with pre-drawn k-means draws as bench.py uses, so the timed region has no host RNG work.
For S in --streams it reports, per round of S frames:
  - aggregate frames/s into memory, batched and sequential (pixels in, banks updated);
  - consolidation ms per round (finished ViT features in: pool3 + the consolidation launches), batched and sequential;
  - kernel launches per round;
and, once, a single stream fed 32-frame clips (the clip rate the batched step approaches).  Every row runs warm-up steps
and then at least --seconds of CUDA-event-timed rounds.  The card's name, power limit and SM clocks are read (read-only)
with nvidia-smi in the same run.  At the largest S the batched banks are checked bit for bit against the sequential ones.
Prints one JSON line."""
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
    ap.add_argument("--seconds", type=float, default=3.0, help="timed seconds per row (at least)")
    ap.add_argument("--warm", type=int, default=30, help="warm-up rounds per row (fills the banks past the 25-slot warm-up)")
    ap.add_argument("--check-rounds", type=int, default=30)
    a = ap.parse_args()
    import torch
    torch.set_grad_enabled(False)
    from flash_vstream_b200 import StreamPool, ops
    from flash_vstream_b200.clip_encoder import CLIPVisionTower
    from flash_vstream_b200.vstream_arch import FlashVStreamB200, NeuralTuringMachine
    from oracle import fvs_oracle as O
    from tests import golden_inputs as GI

    if not torch.cuda.is_available():
        raise SystemExit("gpu_multistream_timing.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    lib = ops.L.load()
    S_list = [int(s) for s in a.streams.split(",")]
    tower = CLIPVisionTower.from_weights(O.random_vit_weights(O.VitConfig(), 0), select_layer=-2, max_batch=32, device=dev)
    ntm = NeuralTuringMachine(1024, 32)
    GI.load_ntm(ntm, 0)
    model = FlashVStreamB200(tower, ntm.half().to(dev))
    engine = tower.engine
    g = torch.Generator().manual_seed(1)
    pix = torch.randn(64, 3, 336, 336, generator=g).half().to(dev)
    feats = tower(pix)                                                    # [64, 576, 1024] finished features
    draws = [tuple(torch.from_numpy(d).to(dev) for d in GI.kmeans_draws(26, 25, 300 + i)) for i in range(16)]
    mw = model.get_model().attention_model
    ntm_w = (mw.q_proj.weight, mw.q_proj.bias, mw.k_proj.weight, mw.k_proj.bias)

    def frame(r, i, src):
        k = (r * 7 + i * 13) % src.shape[0]
        return src[k:k + 1]

    def draw(bank, r, i):
        return draws[(r + 3 * i) % len(draws)] if bank.needs_draws(1) else None

    def timed(round_fn, warm, seconds):
        """(ms per round, launches per round): warm-up, then CUDA-event-timed rounds until `seconds` have passed"""
        for r in range(warm):
            round_fn(r)
        torch.cuda.synchronize()
        n0 = lib.fvs_launch_count()
        round_fn(warm)
        launches = lib.fvs_launch_count() - n0
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n, total_ms, r = 0, 0.0, warm + 1
        while total_ms < seconds * 1e3:
            chunk = max(1, n)            # double the number of rounds per timed window
            e0.record()
            for _ in range(chunk):
                round_fn(r)
                r += 1
            e1.record()
            e1.synchronize()
            total_ms += e0.elapsed_time(e1)
            n += chunk
        return total_ms / n, launches

    def batched(S, src):
        pool = StreamPool(model, chunk_cap=1)
        sids = [pool.open() for _ in range(S)]

        def round_fn(r):
            pool.step({s: frame(r, i, src) for i, s in enumerate(sids)},
                      draws={s: draw(pool.bank(s), r, i) for i, s in enumerate(sids) if pool.bank(s).needs_draws(1)})
        return pool, round_fn

    def sequential(S, src):
        banks = [ops.StreamBank(model._fused_cfg(model._star_cfg(), 24, 1024, torch.float16), ntm_w, chunk_cap=1, device=dev)
                 for _ in range(S)]
        vit = engine if src is pix else None

        def round_fn(r):
            for i, b in enumerate(banks):
                b.step(frame(r, i, src), vit=vit, draws=draw(b, r, i))
        return banks, round_fn

    rows = []
    info_before = gpu_info()
    for S in S_list:
        row = {"S": S}
        for name, make in (("batched", batched), ("sequential", sequential)):
            _, fn = make(S, pix)
            ms, launches = timed(fn, a.warm, a.seconds)
            row[f"{name}_frames_per_s"] = S * 1e3 / ms
            row[f"{name}_ms_per_round"] = ms
            row[f"{name}_launches_per_round"] = launches
            _, fn = make(S, feats)
            ms, launches = timed(fn, a.warm, a.seconds)
            row[f"{name}_consolidation_ms_per_round"] = ms
            row[f"{name}_consolidation_launches_per_round"] = launches
            torch.cuda.empty_cache()
        row["speedup"] = row["batched_frames_per_s"] / row["sequential_frames_per_s"]
        row["sm_clock_after"] = (gpu_info() or {}).get("clocks.sm")
        rows.append(row)
        print(json.dumps({"partial": row}), file=sys.stderr, flush=True)

    # one stream fed 32-frame clips: the rate of the reference's clip-per-call regime
    clip_bank = ops.StreamBank(model._fused_cfg(model._star_cfg(), 24, 1024, torch.float16), ntm_w, chunk_cap=32, device=dev,
                               frames_cap=4096)
    clip_draws = [tuple(torch.from_numpy(d).to(dev) for d in GI.kmeans_draws(57, 25, 700 + i)) for i in range(8)]
    pix2 = torch.cat([pix, pix])

    def clip_round(r):
        if clip_bank.bank.n_frames + 32 > 4096:
            clip_bank.reset()
        k = (r * 32) % 64
        clip_bank.step(pix2[k:k + 32], vit=engine, draws=clip_draws[r % 8] if clip_bank.needs_draws(32) else None)
    ms32, l32 = timed(clip_round, 4, a.seconds)

    # bit-identity of the largest batch against the same streams stepped one by one
    S = max(S_list)
    pool, fb = batched(S, pix)
    banks, fs = sequential(S, pix)
    for r in range(a.check_rounds):
        fb(r)
        fs(r)
    torch.cuda.synchronize()
    same = all(torch.equal(pool.prefix(s), b.prefix()) and torch.equal(pool.bank(s).header, b.header) and
               torch.equal(pool.bank(s).long_work, b.long_work) and torch.equal(pool.bank(s).tur_work, b.tur_work) and
               pool.bank(s).bank.n_frames == b.bank.n_frames
               for s, b in zip(sorted(pool._streams), banks))

    out = {"metric": "multistream_single_frame_steps", "tower": "ViT-L/14-336 (random weights, 23 layers run, f16)",
           "config": "681-token default (long 25, Turing 25, current 1, key 3)", "gpu_before": info_before,
           "gpu_after": gpu_info(), "rows": rows,
           "clip32_frames_per_s": 32 * 1e3 / ms32, "clip32_ms_per_step": ms32, "clip32_launches_per_step": l32,
           f"batched_equals_sequential_S{S}_bits": same, "check_rounds": a.check_rounds, "time": time.strftime("%Y-%m-%d %H:%M:%S")}
    print(json.dumps(out), flush=True)
    if not same:
        raise SystemExit("batched banks differ from the sequential ones")


if __name__ == "__main__":
    main()
