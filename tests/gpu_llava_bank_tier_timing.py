"""Timing of the LLaVA bank's device window (DESIGN.md §3.14, §4): StreamPool single-frame steps at S = 1, 8, 32 streams,
and one stream of 32-frame clips pre-filled to 10 000 frames by restore — each uncapped and capped at the minimum window,
side by side in one process, in alternating blocks.  Reports per-round median / max step time (host clock around the
step and a device synchronise), the D2H bytes of the spills per round and the device bytes per stream, with the card's
name and power limit.  Prints one JSON line (and writes it to --out when given).

    python tests/gpu_llava_bank_tier_timing.py [--seconds 3] [--out FILE]
"""
import argparse
import json
import os
import statistics
import subprocess
import sys
import time

import torch

sys.path.insert(0, os.path.dirname(os.path.dirname(os.path.abspath(__file__))))

from flash_vstream_b200 import checkpoint as CK  # noqa: E402
from flash_vstream_b200 import ops  # noqa: E402
from flash_vstream_b200.multistream import StreamPool  # noqa: E402
from flash_vstream_b200.vstream_arch import FlashVStreamB200, NeuralTuringMachine  # noqa: E402

D = 1024


def card():
    try:
        q = subprocess.run(["nvidia-smi", "--query-gpu=name,power.limit", "--format=csv,noheader"], capture_output=True,
                           text=True, timeout=30).stdout.strip().splitlines()[0]
    except Exception as e:     # noqa: BLE001
        q = f"unknown ({e})"
    return q


def bank_bytes(bank):
    return sum(t.numel() * t.element_size() for t in (bank.prefix_buf, bank.long_work, bank.tur_work, bank.frames,
                                                      bank.header, bank.ws))


def model():
    torch.manual_seed(0)
    ntm = NeuralTuringMachine(D, 32).half().cuda()
    return FlashVStreamB200(None, ntm)


def spill_bytes(bank, n0, t):
    N = bank.device_frames
    return 0 if N is None else max(0, n0 + t - max(n0, N)) * bank.pa * D * 2


def time_rows(arms, seconds, block, before_block=None):
    """arms: {name: step() -> D2H bytes}; alternate blocks of `block` rounds until every arm has `seconds` of steps;
    before_block: {name: fn()} run untimed before each of that arm's blocks"""
    times = {k: [] for k in arms}
    d2h = {k: [] for k in arms}
    while min(sum(v) for v in times.values()) < seconds:
        for k, step in arms.items():
            if before_block:
                before_block[k]()
            for _ in range(block):
                torch.cuda.synchronize()
                t0 = time.perf_counter()
                b = step()
                torch.cuda.synchronize()
                times[k].append(time.perf_counter() - t0)
                d2h[k].append(b)
    return {k: {"rounds": len(v), "median_ms": 1e3 * statistics.median(v), "max_ms": 1e3 * max(v),
                "d2h_bytes_per_round": statistics.mean(d2h[k])} for k, v in times.items()}


def pool_rows(S, seconds):
    g = torch.Generator(device="cuda").manual_seed(S)
    feats = torch.randn(64, 576, D, generator=g, device="cuda").half()
    ref = StreamPool(model())
    pools = {"uncapped": ref, "capped": StreamPool(model(), device_frames=ops.min_device_frames(ref.cfg, 1))}
    sids = {k: [p.open(seed=i) for i in range(S)] for k, p in pools.items()}
    ctr = {"i": 0}

    def arm(k):
        p = pools[k]

        def step():
            i = ctr["i"] = ctr["i"] + 1
            banks = [p.bank(s) for s in sids[k]]
            n0 = [b.bank.n_frames for b in banks]
            p.step({s: feats[(i + j) % 64:(i + j) % 64 + 1] for j, s in enumerate(sids[k])})
            return sum(spill_bytes(b, n, 1) for b, n in zip(banks, n0))
        return step

    arms = {k: arm(k) for k in pools}
    for _ in range(40):                    # warm-up past the 25-slot memory and the 26-frame window
        for a in arms.values():
            a()
    rows = time_rows(arms, seconds, 25)
    for k, p in pools.items():
        b = p.bank(sids[k][0])
        rows[k].update(streams=S, frames_per_stream=b.bank.n_frames, device_bytes_per_stream=bank_bytes(b),
                       host_bytes_per_stream=len(b.host_chunks) * b.CHUNK_BYTES)
    return rows


def clip_rows(seconds, prefill=10_000, t=32):
    m = model()
    cfg = m._fused_cfg(m._star_cfg(), 24, D, torch.float16)
    ntm = m.get_model().attention_model
    w = (ntm.q_proj.weight, ntm.q_proj.bias, ntm.k_proj.weight, ntm.k_proj.bias)
    g = torch.Generator(device="cuda").manual_seed(1)
    feats = torch.randn(4 * t, 576, D, generator=g, device="cuda").half()
    seed = ops.StreamBank(cfg, w, chunk_cap=t)
    for i in range(4):
        seed.step(feats[i * t:(i + 1) * t], draws=_draws(seed, t, i))
    ck = seed.checkpoint()
    frames = torch.empty(prefill, 64, D, dtype=torch.float16, pin_memory=True)
    frames[:4 * t].copy_(ck.tensor("frames"))
    frames[4 * t:].copy_(torch.randn(prefill - 4 * t, 64, D, generator=g, device="cuda").half().cpu())
    big = CK.StreamCheckpoint(CK.LLAVA, ck.config, {**ck.counters, "n_frames": prefill},
                              {**ck.tensors, "frames": frames})
    banks = {"uncapped": ops.StreamBank(cfg, w, chunk_cap=t),
             "capped": ops.StreamBank(cfg, w, chunk_cap=t, device_frames=ops.min_device_frames(cfg, t))}
    t0 = time.perf_counter()
    for b in banks.values():
        b.restore(big)
    restore_s = time.perf_counter() - t0
    ctr = {"i": 0}

    def arm(b):
        def step():
            i = ctr["i"] = ctr["i"] + 1
            n0 = b.bank.n_frames
            b.step(feats[(i % 4) * t:(i % 4 + 1) * t], draws=_draws(b, t, i))
            return spill_bytes(b, n0, t)
        return step

    def refill(b):       # back to the pre-filled stream every block: the row stays at 10 000 - 16 400 frames
        return lambda: b.restore(big) if b.bank.n_frames >= prefill + 150 * t else None

    arms = {k: arm(b) for k, b in banks.items()}
    for _ in range(5):
        for a in arms.values():
            a()
    rows = time_rows(arms, seconds, 50, {k: refill(b) for k, b in banks.items()})
    for k, b in banks.items():
        rows[k].update(streams=1, clip=t, frames_per_stream=f"{prefill}-{prefill + 200 * t}", device_bytes_per_stream=bank_bytes(b),
                       host_bytes_per_stream=len(b.host_chunks) * b.CHUNK_BYTES)
    rows["restore_both_s"] = restore_s
    return rows


def _draws(bank, t, i):
    if not bank.needs_draws(t):
        return None
    gen = torch.Generator().manual_seed(1000 + i)
    T, K = bank.working_rows(t), bank.cfg.long_len
    init = torch.randperm(T, generator=gen)[:K].to(torch.int32)
    refill = torch.randint(0, T, (10 * K,), generator=gen).to(torch.int32)
    return init.cuda(), refill.cuda()


def main():
    ap = argparse.ArgumentParser()
    ap.add_argument("--seconds", type=float, default=3.0)
    ap.add_argument("--out", default=None, help="also write the JSON result to this file")
    a = ap.parse_args()
    torch.set_grad_enabled(False)
    out = {"card": card(), "rows": {}}
    for S in (1, 8, 32):
        out["rows"][f"pool_S{S}"] = pool_rows(S, a.seconds)
        print(S, json.dumps(out["rows"][f"pool_S{S}"]), flush=True)
    out["rows"]["clip32_10k"] = clip_rows(a.seconds)
    print(json.dumps(out["rows"]["clip32_10k"]), flush=True)
    out["card_after"] = card()
    if a.out:
        with open(a.out, "w") as f:
            json.dump(out, f, indent=1)
    print(json.dumps(out))


if __name__ == "__main__":
    main()
