"""A/B device timing of fvs_attention / fvs_attention80 across builds of libfvs_b200.so.  Not a test; run on the GPU:

    python tests/gpu_attention_timing.py --out DIR [--repeats 2] LIB [LIB ...]

Each build runs in its own subprocess (FVS_LIB_PATH=LIB), and the builds alternate LIB1, LIB2, ..., LIB1, LIB2, ... for
`--repeats` rounds, so a drift of the card's clock shows up as spread instead of as a difference between builds.  Every
worker times both entry points at both dtypes on three shapes: the ViT-L/14-336 layer (32 frames x 577 tokens x 16 heads)
and the Qwen2-VL full (576 tokens) and half (144 tokens) grids of an 8-patch clip.  Timing: CUDA events around
back-to-back launches, >= 1 s per row after 3 warm-up launches; TFLOP/s counted as bench.py counts attention
(4 * frames * heads * tokens^2 * head_dim).  The first round's outputs are written under DIR/outputs/<build index>/ and
compared with torch.equal across builds (then removed unless --keep-outputs; their sha256 stays in the summary).
Prints the card's name, power limit and maximum SM clock (nvidia-smi queries), one JSON line per worker and a summary."""
import argparse
import hashlib
import json
import os
import shutil
import statistics
import subprocess
import sys

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

SHAPES = [  # (name, frames, tokens, heads)
    ("vit_l", 32, 577, 16),
    ("qwen_full", 8, 576, 16),
    ("qwen_half", 8, 144, 16),
]


def worker(out_dir, save, min_s):
    sys.path.insert(0, ROOT)
    import torch
    from flash_vstream_b200 import _lib, ops
    torch.cuda.set_device(0)
    rows = {}
    for name, frames, tokens, heads in SHAPES:
        for hd in (64, 80):
            for dtype in (torch.float16, torch.bfloat16):
                key = f"{name}_hd{hd}_{'bf16' if dtype == torch.bfloat16 else 'f16'}"
                g = torch.Generator().manual_seed(frames * 1000 + tokens + hd)
                qkv = torch.randn(frames * tokens, 3 * heads * hd, generator=g).to(dtype).cuda()
                out = torch.empty(frames * tokens, heads * hd, dtype=dtype, device="cuda")
                fn = ops.attention if hd == 64 else ops.attention80

                def launch():
                    fn(qkv, frames, tokens, heads, out=out)
                for _ in range(3):
                    launch()
                torch.cuda.synchronize()
                a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
                a.record()
                for _ in range(10):
                    launch()
                b.record()
                torch.cuda.synchronize()
                n = max(10, int(min_s * 1e3 / (a.elapsed_time(b) / 10)) + 1)
                a.record()
                for _ in range(n):
                    launch()
                b.record()
                torch.cuda.synchronize()
                ms = a.elapsed_time(b)
                us = ms * 1e3 / n
                flop = 4.0 * frames * heads * tokens * tokens * hd
                rows[key] = {"us_per_launch": us, "tflops": flop / (us * 1e-6) / 1e12, "launches": n, "seconds": ms / 1e3,
                             "sha256": hashlib.sha256(out.cpu().view(torch.int16).numpy().tobytes()).hexdigest()}
                if save:
                    torch.save(out.cpu(), os.path.join(out_dir, key + ".pt"))
    print(json.dumps({"lib": str(_lib.lib_path()), "device": torch.cuda.get_device_name(0), "rows": rows}), flush=True)


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("libs", nargs="*", help="paths of libfvs_b200.so builds to compare")
    ap.add_argument("--out", required=True, help="output directory")
    ap.add_argument("--repeats", type=int, default=2, help="rounds over all builds (>= 2)")
    ap.add_argument("--min-s", type=float, default=1.0, help="seconds of launches per timed row")
    ap.add_argument("--keep-outputs", action="store_true")
    ap.add_argument("--worker", action="store_true", help=argparse.SUPPRESS)
    ap.add_argument("--save", action="store_true", help=argparse.SUPPRESS)
    a = ap.parse_args()
    if a.worker:
        worker(a.out, a.save, a.min_s)
        return
    if not a.libs:
        ap.error("give at least one library path")
    if a.repeats < 2:
        ap.error("--repeats must be at least 2")
    os.makedirs(a.out, exist_ok=True)
    smi = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit,clocks.max.sm", "--format=csv"],
                         capture_output=True, text=True)
    print(smi.stdout.strip() or smi.stderr.strip(), flush=True)
    libs = [os.path.abspath(p) for p in a.libs]
    results = {i: [] for i in range(len(libs))}
    for r in range(a.repeats):
        for i, lib in enumerate(libs):
            odir = os.path.join(a.out, "outputs", str(i))
            os.makedirs(odir, exist_ok=True)
            cmd = [sys.executable, os.path.abspath(__file__), "--worker", "--out", odir, "--min-s", str(a.min_s)]
            if r == 0:
                cmd.append("--save")
            p = subprocess.run(cmd, env=dict(os.environ, FVS_LIB_PATH=lib), capture_output=True, text=True)
            if p.returncode != 0:
                sys.stderr.write(p.stdout + p.stderr)
                raise SystemExit(f"worker for {lib} failed with exit code {p.returncode}")
            line = json.loads(p.stdout.strip().splitlines()[-1])
            print(json.dumps({"round": r, "build": i, **line}), flush=True)
            results[i].append(line)
    import torch
    keys = list(results[0][0]["rows"])
    summary = {"nvidia_smi": smi.stdout.strip(), "device": results[0][0]["device"], "libs": libs, "rows": {}}
    for k in keys:
        row = {}
        for i in range(len(libs)):
            us = [res["rows"][k]["us_per_launch"] for res in results[i]]
            tf = [res["rows"][k]["tflops"] for res in results[i]]
            row[f"build{i}"] = {"us_median": statistics.median(us), "us_min": min(us), "us_max": max(us),
                                "tflops_median": statistics.median(tf), "sha256": results[i][0]["rows"][k]["sha256"]}
        base = torch.load(os.path.join(a.out, "outputs", "0", k + ".pt"))
        row["equal_to_build0"] = [torch.equal(base, torch.load(os.path.join(a.out, "outputs", str(i), k + ".pt")))
                                  for i in range(len(libs))]
        row["speedup_vs_build0"] = [row["build0"]["us_median"] / row[f"build{i}"]["us_median"] for i in range(len(libs))]
        summary["rows"][k] = row
    if not a.keep_outputs:
        shutil.rmtree(os.path.join(a.out, "outputs"))
    with open(os.path.join(a.out, "attention_timing.json"), "w") as f:
        json.dump(summary, f, indent=1)
    print(json.dumps(summary), flush=True)


if __name__ == "__main__":
    main()
