"""CPU: the compiled attention kernels keep the softmax of S_{j+1} between the two wgmma waits of a KV step, i.e. the
exponentials run while O += P_j V_j is still on the tensor cores.  ptxas is free to move WARPGROUP.DEPBAR within a basic
block; if a compiler or source change pulls the wait for P V above the softmax again, every exponential lands after it and
the warpgroup alternates between tensor cores and SFU.  Read from the SASS of the built library (no GPU needed)."""
import os
import re
import subprocess

import pytest

CUOBJDUMP = "/usr/local/cuda/bin/cuobjdump"


def attention_windows():
    """{instantiation: [MUFU.EX2 count between each `DEPBAR.LE gsb0, 0x1` and the next `DEPBAR.LE gsb0, 0x0`]}"""
    from flash_vstream_b200 import _build
    _build.build()
    sass = subprocess.run([CUOBJDUMP, "-sass", str(_build.LIB_PATH)], capture_output=True, text=True).stdout
    out, fn, win = {}, None, None
    for line in sass.splitlines():
        m = re.search(r"Function : (\S+)", line)
        if m:
            k = re.search(r"attention_kernelILb([01])ELb([01])E", m.group(1))
            fn = (("bf16" if k.group(1) == "1" else "f16") + ("_hd80" if k.group(2) == "1" else "_hd64")) if k else None
            if fn:
                out[fn] = []
            win = None
            continue
        if fn is None:
            continue
        if "WARPGROUP.DEPBAR.LE gsb0, 0x1" in line:
            win = 0
        elif "WARPGROUP.DEPBAR.LE gsb0, 0x0" in line and win is not None:
            out[fn].append(win)
            win = None
        elif "MUFU.EX2" in line and win is not None:
            win += 1
    return out


@pytest.mark.skipif(not os.path.exists(CUOBJDUMP), reason="cuobjdump not available")
def test_softmax_exponentials_overlap_the_pv_wgmma():
    wins = attention_windows()
    assert sorted(wins) == ["bf16_hd64", "bf16_hd80", "f16_hd64", "f16_hd80"]
    for name, counts in wins.items():
        # one window for the full-width step (32 + 2 exponentials per thread), one for the narrow last tile (8 + 2)
        assert len(counts) == 2, (name, counts)
        assert all(c >= 10 for c in counts), f"{name}: exponentials outside the P V wgmma window {counts}"
        assert max(counts) >= 34, f"{name}: full-width step does not overlap its exponentials {counts}"
