"""The resource budget of the attention forward (both instantiations of attn_flash_fwd_kernel), read from the built
library like tests/test_attention_bwd_regs_cpu.py. Its 288-thread block (two MMA warpgroups and a producer warp) is
allocated as 12 warps, so 168 registers per thread is the most that lets a launch succeed; each warpgroup keeps its
output accumulator, a score fragment and (with relative positions) a 64 x 128 position-score fragment in registers, and
anything that did not fit would go to local memory on every key block."""
import re
import shutil
import subprocess

import pytest


def test_attn_flash_fwd_fits_its_launch_bounds_without_local_memory():
    from speecht5_b200.build import LIB
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True).stdout
    elf = subprocess.run(["cuobjdump", "-elf", LIB], capture_output=True, text=True).stdout
    threads = {}
    for sec in re.split(r"\n(?=\.nv\.info\.)", elf):
        m = re.match(r"\.nv\.info\.(\S+)", sec)
        t = re.search(r"EIATTR_MAX_THREADS\s*\n\s*Format:\s*\S+\s*\n\s*Value:\s*(0x[0-9a-f]+) (0x[0-9a-f]+) (0x[0-9a-f]+)",
                      sec)
        if m and t and "attn_flash_fwd_kernel" in m.group(1):
            threads[m.group(1)] = int(t.group(1), 16) * int(t.group(2), 16) * int(t.group(3), 16)
    assert len(threads) == 2 and set(threads.values()) == {288}, f"attn_flash_fwd_kernel launch bounds: {threads}"
    found = [m for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) \S+ LOCAL:(\d+)", res)
             if "attn_flash_fwd_kernel" in m.group(1)]
    assert len(found) == 2, [m.group(1) for m in found]  # <false> and <true> (relative positions)
    for f in found:
        regs, stack, local = (int(f.group(i)) for i in (2, 3, 4))
        assert regs <= 168, f"{f.group(1)}: {regs} registers"
        assert stack == 0 and local == 0, f"{f.group(1)} spills: STACK {stack}, LOCAL {local}"
