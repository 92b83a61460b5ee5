"""Generate tests/golden/alt_shapes.npz by EXECUTING THE REFERENCE's alternate compressors
(flash_vstream.model.compress_functions.{drop,merge,kmeans,k_drop,k_merge}_feature) on CPU f16 tensors, on the moderate
cases of tests/alt_shapes_inputs.py (GOLDEN: the clip and duplicates profiles, T0 = 2 and the k-means cases up to T = 200,
at PD <= 16384).

    PYTHONDONTWRITEBYTECODE=1 python tests/golden/make_golden_alt_shapes.py [path of the Flash-VStream-LLaVA checkout]

The draws are the case's explicit ones: random.randint returns the coin flips (drop variants) or the refill candidates
(kmeans), torch.randperm a permutation that starts with the case's init_idx; the count consumed is checked / stored.
Every k-means case has T > 25, so torch.cdist takes its matmul form, the one the kernels implement.
Stored per case: the per-step member lists, the final similarities, a strided element subset of the features (every
61st element of every row, which visits every lane and slice position), the refills a k-means consumed, and the input
checksum.  Every case of the table stores its input checksum, so the GPU tests can tell a drifted input from a wrong
kernel.

It also records what the reference's key retrieval (vstream_arch.py:259-267) does with each compressor's weight on small
long memories: the exception it raises, or the key indices."""
from __future__ import annotations

import os
import random
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.dirname(os.path.dirname(HERE)))
sys.path.insert(0, sys.argv[1] if len(sys.argv) > 1 else "/root/reference/Flash-VStream-LLaVA")
sys.dont_write_bytecode = True

from flash_vstream.model import compress_functions as ref_cf  # noqa: E402

from tests import alt_shapes_inputs as AS  # noqa: E402
from tests.golden.make_golden_alternates import flat_steps  # noqa: E402

STRIDE = 61
GLUE_FNS = ("drop_feature", "merge_feature", "k_drop_feature", "k_merge_feature")

def run_case(name):
    """(feat, sim, steps, refills consumed) of the reference on case `name`"""
    c = AS.CASES[name]
    x = AS.features(name)
    kmeans = c["fn"] == "kmeans_feature"
    if kmeans:
        init, refill = AS.kmeans_draws(name)
        draws = refill.tolist()
        rest = [i for i in range(c["T"]) if i not in set(init.tolist())]
        perm = torch.tensor(init.tolist() + rest, dtype=torch.int64)
    else:
        draws = list(AS.coins(name))
    n_draws = len(draws)
    real_ri, real_rp = random.randint, torch.randperm

    def ri(a, b):
        assert (a, b) == ((0, c["T"] - 1) if kmeans else (0, 1))
        return draws.pop(0)

    def rp(n, *a, **k):
        assert kmeans and n == c["T"]
        return perm.clone()
    random.randint, torch.randperm = ri, rp
    try:
        sim_in = AS.sim_in(name)
        feat, sim, steps = getattr(ref_cf, c["fn"])(x.clone(), c["T0"], sim_in)
    finally:
        random.randint, torch.randperm = real_ri, real_rp
    assert kmeans or not draws, "the reference consumed fewer coins than the case holds"
    return feat, sim, steps, n_draws - len(draws)


def key_retrieval(long_memory, weight):
    """the reference's retrieval of vstream_arch.py:261-267 on a compressor's weight"""
    order = torch.argsort(weight, descending=True)
    key = long_memory[order]
    key = key[:3] if key.shape[0] > 3 else key
    dists = ((long_memory.unsqueeze(1) - key.unsqueeze(0)) ** 2).sum(dim=3).sum(dim=2).sqrt()
    return torch.argmin(dists, dim=0)


def main():
    out = {}
    for name in AS.CASES:
        out[name + "_chk"] = AS.checksum(AS.features(name))
    for name in AS.GOLDEN:
        feat, sim, steps, used = run_case(name)
        c = AS.CASES[name]
        out[name + "_refills"] = np.array(used if c["fn"] == "kmeans_feature" else 0, np.int32)
        out[name + "_feat"] = feat.reshape(c["T0"], -1)[:, ::STRIDE].contiguous().numpy().view(np.int16)
        out[name + "_sim"] = sim.numpy().view(np.int16) if sim is not None else np.zeros(0, np.int16)
        out[name + "_n_rows"], out[name + "_n_mem"], out[name + "_mem"] = flat_steps(steps)
        print(name, tuple(feat.shape), "steps", len(steps), "last", steps[-1][:4])
    for fn in GLUE_FNS:
        for T, T0 in AS.GLUE_SHAPES:
            key = f"glue_{fn}_{T}_{T0}"
            x = AS.glue_features(T, T0)
            random.seed(T)
            try:
                _, weight, _ = getattr(ref_cf, fn)(x.clone(), T0)
                idx = key_retrieval(x, weight)
                out[key + "_exc"] = np.array("ok")
                out[key + "_idx"] = idx.numpy().astype(np.int64)
            except Exception as e:      # noqa: BLE001 - the exception type is what is recorded
                out[key + "_exc"] = np.array(type(e).__name__)
            print(key, out[key + "_exc"])
    np.savez_compressed(os.path.join(HERE, "alt_shapes.npz"), **out)
    print("alt_shapes.npz", len(out), os.path.getsize(os.path.join(HERE, "alt_shapes.npz")))


if __name__ == "__main__":
    main()
