"""Timing script (not a pytest file): the ViT-L/14-336 encoder alone (23 layers run, f16, random weights) on one
micro-batch of nf frames per call, pixels in HBM, the pooled STAR tail (fvs_vit_encode_pool3, 8x8 / 4x4 / 1x1), the
layer stack replayed from its CUDA graph.  For each nf in --frames it runs warm-up calls and then at least --seconds of
CUDA-event-timed calls, and reports ms per micro-batch, frames/s, kernel launches per call and a SHA-256 of the pooled
outputs (equal digests across two builds mean equal bits).  The card's name, power limit and SM clocks are read
(read-only) with nvidia-smi in the same run.  Prints one JSON line.

Used to set kSplitMin in csrc/vit_engine.cu: run it from two builds in one session, alternating, and compare rows."""
import argparse
import hashlib
import json
import os
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

from tests.gpu_multistream_timing import gpu_info  # noqa: E402


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--frames", default="2,4,8,16,32", help="frames per micro-batch, one row each")
    ap.add_argument("--seconds", type=float, default=2.0, help="timed seconds per row (at least)")
    ap.add_argument("--warm", type=int, default=5, help="untimed calls per row (the first runs eagerly, the second captures)")
    a = ap.parse_args()
    import torch
    torch.set_grad_enabled(False)
    from flash_vstream_b200 import ops
    from oracle import fvs_oracle as O

    if not torch.cuda.is_available():
        raise SystemExit("gpu_vit_overlap_timing.py needs a CUDA device")
    dev = torch.device("cuda", 0)
    L = ops.L
    cfg = O.VitConfig()
    frames = [int(f) for f in a.frames.split(",")]
    eng = ops.VitEncoder(O.random_vit_weights(cfg, 0), layers_run=23, dtype=torch.float16, device=dev,
                         max_batch=max(frames))
    lib = eng.lib
    g = torch.Generator().manual_seed(1)
    pix = (torch.randn(max(frames), 3, 336, 336, generator=g) * 0.5).half().to(dev)

    rows = []
    info_before = gpu_info()
    for nf in frames:
        outs = [torch.empty(nf, n, cfg.hidden, dtype=torch.float16, device=dev) for n in (64, 16, 1)]

        def call():
            L.check(lib.fvs_vit_encode_pool3(eng._h, L.ptr(pix), *[L.ptr(o) for o in outs], nf, 8, 4, L.ptr(eng._ws),
                                             eng._ws.numel(), L.cur_stream()), "fvs_vit_encode_pool3")
        for _ in range(a.warm):
            call()
        torch.cuda.synchronize()
        n0 = lib.fvs_launch_count()
        call()
        launches = lib.fvs_launch_count() - n0
        e0, e1 = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
        n, total_ms = 0, 0.0
        while total_ms < a.seconds * 1e3:
            chunk = max(1, n)            # double the number of calls per timed window
            e0.record()
            for _ in range(chunk):
                call()
            e1.record()
            e1.synchronize()
            total_ms += e0.elapsed_time(e1)
            n += chunk
        h = hashlib.sha256()
        for o in outs:
            h.update(o.cpu().numpy().tobytes())
        ms = total_ms / n
        row = {"frames": nf, "ms_per_microbatch": ms, "frames_per_s": nf * 1e3 / ms, "calls_timed": n,
               "launches_per_call": launches, "outputs_sha256": h.hexdigest()[:16],
               "sm_clock_after": (gpu_info() or {}).get("clocks.sm")}
        rows.append(row)
        print(json.dumps({"partial": row}), file=sys.stderr, flush=True)

    print(json.dumps({"metric": "vit_encoder_microbatch", "tower": "ViT-L/14-336 (random weights, 23 layers run, f16)",
                      "tail": "pool3 (8x8, 4x4, 1x1)", "gpu_before": info_before, "gpu_after": gpu_info(), "rows": rows,
                      "time": time.strftime("%Y-%m-%d %H:%M:%S")}), flush=True)


if __name__ == "__main__":
    main()
