"""CPU: the Qwen2-VL Flash Memory kernels in the built library.  Every single-stream call runs as the one-job table
(kJobs = 1), so only the job-table kernels and the per-tier range sweep exist, and the one-job instantiations use no
local memory or stack and keep the register counts the single calls need: the Lloyd update at most 80 (3 blocks of 256
per SM) and the f16 bank sweeps at most 100 (Euclidean) and 98 (cosine).  Read from `cuobjdump -res-usage` (no GPU
needed)."""
import os
import re
import subprocess
from pathlib import Path

import pytest

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"
KUPDATE = 8              # MemStage of qwen_kernels.cu
KL_SWEEP_EUCLIDEAN, KL_SWEEP_COSINE = 0, 2   # KlStage of qwen_kernels.cu


def qwen_memory_kernels():
    """{mangled name: (registers, stack bytes, local bytes)} of the kernels of qwen_kernels.cu and qwen_bank.cu"""
    from flash_vstream_b200 import _build
    _build.build()
    out = subprocess.run([CUOBJDUMP, "-res-usage", str(_build.LIB_PATH)], capture_output=True, text=True).stdout
    res, fn = {}, None
    for line in out.splitlines():
        m = re.search(r"Function (\S+):", line)
        if m:
            fn = m.group(1)
            continue
        m = re.search(r"REG:(\d+) STACK:(\d+) SHARED:\d+ LOCAL:(\d+)", line)
        if m and fn and (fn.startswith("_ZN3fvs4qwen") or "dam_gather" in fn):
            res[fn] = tuple(int(v) for v in m.groups())
        fn = None
    return res


def kind(name):
    """(kernel, template arguments) from a mangled name, e.g. ('mem_multi_kernel', (1, 8))"""
    base = re.search(r"\d+([a-z][a-z_]*_kernel)", name).group(1)
    args = tuple(int(v) for v in re.findall(r"L[ib](\d+)E", name))
    return base, args


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_single_calls_are_one_job_tables():
    ks = qwen_memory_kernels()
    by = {}
    for name, r in ks.items():
        base, args = kind(name)
        by.setdefault(base, {})[args] = r
    assert sorted(by) == ["am_rope_kernel", "dam_gather_multi_kernel", "klarge_multi_kernel", "klarge_partial_kernel",
                          "mem_multi_kernel", "temporal_pool_kernel"], sorted(by)
    jobs = {a[0] for base in ("mem_multi_kernel", "klarge_multi_kernel", "dam_gather_multi_kernel") for a in by[base]}
    assert jobs == {1, 16}, jobs
    assert len(by["klarge_partial_kernel"]) == 6                 # (f16 | bf16) x the three sweep modes, range form only
    one = {(base, a): r for base in ("mem_multi_kernel", "klarge_multi_kernel", "dam_gather_multi_kernel")
           for a, r in by[base].items() if a[0] == 1}
    assert len(one) == 14 + 2 * 9 + 1
    for (base, a), (reg, stack, local) in one.items():
        assert stack == 0 and local == 0, f"{base}{a}: stack {stack} B, local {local} B"
    assert one[("mem_multi_kernel", (1, KUPDATE))][0] <= 80
    assert one[("klarge_multi_kernel", (1, 0, KL_SWEEP_EUCLIDEAN))][0] <= 100
    assert one[("klarge_multi_kernel", (1, 0, KL_SWEEP_COSINE))][0] <= 98


def test_bank_kernels_are_one_per_operation():
    """qwen_bank.cu has one kernel per operation: the DAM gather (every stream kind, and the pixel gather of tower-dtype
    rows), the pick plan (with or without a bank), the bank scatter, the code decode and the code gather"""
    src = (Path(__file__).resolve().parents[1] / "flash_vstream_b200" / "csrc" / "qwen_bank.cu").read_text()
    kernels = re.findall(r"__global__\s+void\s+(?:__launch_bounds__\([^)]*\)\s+)?(\w+)", src)
    assert sorted(kernels) == ["bank_scatter_kernel", "dam_gather_multi_kernel", "pick_plan_kernel",
                               "pixel_codes_gather_kernel", "pixel_decode_kernel"], kernels
