"""Timing script (not a pytest file): frame pre-processing on the GPU (fvs_preprocess) against the reference's CPU path.

For 480p, 720p and 1080p uint8 RGB frames in 32-frame clips it reports:
  - GPU pre-processing time per frame, CLIP layout (336 shortest edge + 336 center crop, f16) and Qwen2-VL layout
    (default min/max pixels, additional_pool_size 2, fp32 patches): CUDA events over at least --seconds of launches on
    device-resident frames, with caller-owned output and workspace;
  - the host-to-device copy of the pinned uint8 frames, per frame, timed the same way, apart from the kernels;
  - the reference's CPU path on this host: the PIL-backed CLIP image processor of transformers (Pillow bicubic, numpy
    rescale / normalize, what cli_video_stream.py:186 runs per clip), frames/s over at least --seconds;
and, at --e2e-res, frames/s into memory of the ViT-L/14-336 streaming path (random weights, 23 layers, f16; 32-frame
steps) fed (a) f16 pixels already in HBM and (b) pinned uint8 host frames through CLIPFramePreprocessor.  The card's
name, power limit and SM clocks are read (read-only) with nvidia-smi in the same run.  Prints one JSON line."""
import argparse
import json
import os
import subprocess
import sys
import time

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
sys.path.insert(0, ROOT)

RES = {"480p": (480, 640), "720p": (720, 1280), "1080p": (1080, 1920)}


def gpu_info():
    q = "name,power.limit,clocks.sm,clocks.max.sm"
    try:
        out = subprocess.run(["nvidia-smi", f"--query-gpu={q}", "--format=csv,noheader"], capture_output=True, text=True,
                             timeout=30).stdout.strip().splitlines()
        return dict(zip(q.split(","), [v.strip() for v in out[0].split(",")])) if out else None
    except (OSError, subprocess.SubprocessError):
        return None


def ev_time(torch, fn, seconds, warm=5):
    """mean ms per call of fn over >= `seconds` of back-to-back calls, CUDA events around the whole window"""
    for _ in range(warm):
        fn()
    torch.cuda.synchronize()
    t0 = time.perf_counter()
    fn()
    torch.cuda.synchronize()
    n = max(10, int(seconds / max(time.perf_counter() - t0, 1e-6)))
    a, b = torch.cuda.Event(enable_timing=True), torch.cuda.Event(enable_timing=True)
    a.record()
    for _ in range(n):
        fn()
    b.record()
    b.synchronize()
    return a.elapsed_time(b) / n, n


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=2.0)
    ap.add_argument("--clip", type=int, default=32, help="frames per call / step")
    ap.add_argument("--e2e-res", default="720p,1080p")
    a = ap.parse_args()
    import numpy as np
    import torch
    torch.set_grad_enabled(False)
    if not torch.cuda.is_available():
        raise SystemExit("gpu_preprocess_timing.py needs a CUDA device")
    from transformers.models.clip.image_processing_pil_clip import CLIPImageProcessorPil
    from flash_vstream_b200 import CLIPFramePreprocessor, Qwen2VLFramePreprocessor

    dev = torch.device("cuda", 0)
    T = a.clip
    hf = CLIPImageProcessorPil(size={"shortest_edge": 336}, crop_size={"height": 336, "width": 336})
    clip = CLIPFramePreprocessor(hf)
    qwen = Qwen2VLFramePreprocessor(additional_pool_size=2)
    rows = {}
    host_frames = {}
    for name, (H, W) in RES.items():
        f = torch.from_numpy(np.random.default_rng(H).integers(0, 256, (T, H, W, 3), dtype=np.uint8)).pin_memory()
        host_frames[name] = f
        fd = f.to(dev)
        out_c = torch.empty(clip.output_shape(T, H, W), dtype=torch.float16, device=dev)
        ws_c = torch.empty(clip.workspace_bytes(T, H, W, dev), dtype=torch.uint8, device=dev)
        out_q = torch.empty(qwen.output_shape(T, H, W), dtype=torch.float32, device=dev)
        ws_q = torch.empty(qwen.workspace_bytes(T, H, W, dev), dtype=torch.uint8, device=dev)
        ms_c, n_c = ev_time(torch, lambda: clip(fd, out=out_c, workspace=ws_c), a.seconds)
        ms_q, n_q = ev_time(torch, lambda: qwen(fd, out=out_q, workspace=ws_q), a.seconds)
        stage = torch.empty_like(fd)
        ms_h2d, _ = ev_time(torch, lambda: stage.copy_(f, non_blocking=True), a.seconds)
        clip_np = list(f.numpy())
        t0, n_cpu = time.perf_counter(), 0
        while True:
            hf.preprocess(clip_np, return_tensors="pt")["pixel_values"].half()
            n_cpu += 1
            if time.perf_counter() - t0 >= a.seconds:
                break
        cpu_fps = n_cpu * T / (time.perf_counter() - t0)
        rows[name] = dict(
            clip_us_per_frame=round(ms_c * 1e3 / T, 2), clip_launches=n_c,
            qwen_us_per_frame=round(ms_q * 1e3 / T, 2), qwen_launches=n_q, qwen_resized=list(qwen.resized(H, W)),
            h2d_us_per_frame=round(ms_h2d * 1e3 / T, 2), h2d_GBps=round(f.numel() / (ms_h2d * 1e-3) / 1e9, 1),
            cpu_reference_fps=round(cpu_fps, 1), cpu_threads=torch.get_num_threads())
        print(f"[{name}] {rows[name]}", file=sys.stderr, flush=True)
        del fd, out_c, ws_c, out_q, ws_q, stage

    # end to end: the streaming path fed pixels in HBM vs pinned uint8 frames through the GPU pre-processing
    from flash_vstream_b200.clip_encoder import CLIPVisionTower
    from flash_vstream_b200.vstream_arch import FlashVStreamB200, NeuralTuringMachine
    from oracle import fvs_oracle as O
    from tests import golden_inputs as GI
    tower = CLIPVisionTower.from_weights(O.random_vit_weights(O.VitConfig(), 0), select_layer=-2, max_batch=32, device=dev)
    ntm = NeuralTuringMachine(1024, 32)
    GI.load_ntm(ntm, 0)
    e2e = {}
    for name in a.e2e_res.split(","):
        f = host_frames[name]
        pix = clip(f).clone()

        def run(step, seconds=a.seconds):
            model = FlashVStreamB200(tower, ntm.half().to(dev))
            ms, n = ev_time(torch, lambda: step(model), seconds, warm=30)     # past the 25-slot warm-up
            return round(T / (ms * 1e-3), 1)
        e2e[name] = dict(
            pixels_in_hbm_fps=run(lambda m: m.embed_video_streaming(pix.unsqueeze(0))),
            pinned_uint8_fps=run(lambda m: m.embed_video_streaming(clip(f).unsqueeze(0))))
        print(f"[e2e {name}] {e2e[name]}", file=sys.stderr, flush=True)
    print(json.dumps(dict(gpu=gpu_info(), clip_frames=T, seconds=a.seconds, preprocess=rows, e2e=e2e)))


if __name__ == "__main__":
    main()
