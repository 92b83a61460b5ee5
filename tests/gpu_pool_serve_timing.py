"""Timing script (not a pytest file): many single-frame camera streams fed decoded uint8 frames, pre-processed in one call
per round (StreamPool(preprocess=CLIPFramePreprocessor), one fvs_preprocess_multi launch pair per 32 streams) against
a loop of per-stream pre-processing calls followed by StreamPool.step on the pixels.

ViT-L/14 at 336 px (random weights, 23 layers run, f16) and the default 681-token STAR config; frames are uint8
[1, H, W, 3] in pinned host memory, one per stream per round, at 720p and 1080p.  For S in --streams and each size it
reports, per round:
  - pre-processing ms (CUDA events around the pre-processing alone: one many() call, or S single-clip calls), and the
    pre-processing launches;
  - aggregate frames/s into memory over whole rounds (frames in, banks updated), both modes, alternated row by row;
and checks that the two modes' banks are bit-identical after the same rounds.  The card's name and power limit are read
(read-only) with nvidia-smi in the same run.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys

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
    ap.add_argument("--streams", default="1,4,16,32")
    ap.add_argument("--sizes", default="720x1280,1080x1920")
    ap.add_argument("--warm", type=int, default=30, help="warm-up rounds per mode (past the 25-slot warm-up)")
    ap.add_argument("--rounds", type=int, default=40, help="timed rounds per mode")
    ap.add_argument("--reps", type=int, default=50, help="timed pre-processing calls per mode")
    a = ap.parse_args()
    import torch
    torch.set_grad_enabled(False)
    from transformers.models.clip.image_processing_pil_clip import CLIPImageProcessorPil

    from flash_vstream_b200 import StreamPool, ops
    from flash_vstream_b200.clip_encoder import CLIPVisionTower
    from flash_vstream_b200.preprocess import CLIPFramePreprocessor
    from flash_vstream_b200.vstream_arch import FlashVStreamB200, NeuralTuringMachine
    from oracle import fvs_oracle as O
    from tests import golden_inputs as GI

    if not torch.cuda.is_available():
        raise SystemExit("gpu_pool_serve_timing.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    lib = ops.L.load()
    tower = CLIPVisionTower.from_weights(O.random_vit_weights(O.VitConfig(), 0), select_layer=-2, max_batch=32, device=dev)
    ntm = NeuralTuringMachine(1024, 32)
    GI.load_ntm(ntm, 0)
    model = FlashVStreamB200(tower, ntm.half().to(dev))
    pre = CLIPFramePreprocessor(CLIPImageProcessorPil(size={"shortest_edge": 336}, crop_size={"height": 336, "width": 336}))

    def events(fn, n):
        s, e = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        torch.cuda.synchronize()
        s.record()
        for _ in range(n):
            fn()
        e.record()
        e.synchronize()
        return s.elapsed_time(e) / n

    rows = []
    for size in a.sizes.split(","):
        H, W = (int(v) for v in size.split("x"))
        for S in (int(s) for s in a.streams.split(",")):
            g = torch.Generator().manual_seed(S * 7 + H)
            n_frames = a.warm + a.rounds
            frames = [[torch.randint(0, 256, (1, H, W, 3), dtype=torch.uint8, generator=g).pin_memory() for _ in range(S)]
                      for _ in range(min(n_frames, 4))]                  # 4 distinct rounds of frames, cycled
            pools = {"many": StreamPool(model, preprocess=pre), "loop": StreamPool(model)}
            sids = {m: [p.open(seed=100 + i) for i in range(S)] for m, p in pools.items()}

            def round_many(k):
                pools["many"].step(dict(zip(sids["many"], frames[k % len(frames)])))

            def round_loop(k):
                pools["loop"].step({sid: pre(f).unsqueeze(0) for sid, f in zip(sids["loop"], frames[k % len(frames)])})
            fns = {"many": round_many, "loop": round_loop}
            for k in range(a.warm):
                for m in ("many", "loop"):
                    fns[m](k)
            fps = {m: 0.0 for m in fns}
            for m in ("many", "loop", "many", "loop"):                 # alternated, half the rounds each time
                k0 = a.warm + (a.rounds // 2 if fps[m] else 0)
                it = iter(range(k0, k0 + a.rounds // 2))
                ms = events(lambda: fns[m](next(it)), a.rounds // 2)
                fps[m] += S * 1000.0 / ms / 2
            same = all(torch.equal(pools["many"].prefix(x).view(torch.int16), pools["loop"].prefix(y).view(torch.int16))
                       and torch.equal(pools["many"].bank(x).header, pools["loop"].bank(y).header)
                       for x, y in zip(sids["many"], sids["loop"]))
            f0 = frames[0]
            prep = {}
            for m, fn in (("many", lambda: pre.many(f0)), ("loop", lambda: [pre(f) for f in f0])) * 2:
                fn()
                n0 = lib.fvs_launch_count()
                fn()
                launches = lib.fvs_launch_count() - n0
                prep[m] = (min(prep.get(m, (1e9,))[0], events(fn, a.reps)), launches)
            row = {"size": size, "streams": S, "preprocess_ms": {m: round(v[0], 4) for m, v in prep.items()},
                   "preprocess_launches": {m: v[1] for m, v in prep.items()},
                   "frames_per_s": {m: round(v, 1) for m, v in fps.items()}, "banks_bit_identical": same}
            print(json.dumps({"partial": row}), file=sys.stderr, flush=True)
            rows.append(row)
    print(json.dumps({"gpu": gpu_info(), "rows": rows}), flush=True)


if __name__ == "__main__":
    main()
