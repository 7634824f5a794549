"""The resource budget of the fused attention backward (attn_fused_bwd_kernel), read from the built library like
tests/test_frontend_regs_cpu.py. Its 288-thread block (two MMA warpgroups and a producer warp) is allocated as 12 warps,
so 168 registers per thread is the most that lets a launch succeed; the kernel keeps dK, dV and a score-sized fragment
of each warpgroup in registers, and anything that did not fit would go to local memory on every step."""
import re
import shutil
import subprocess

import pytest


def test_attn_fused_bwd_fits_its_launch_bounds_without_local_memory():
    from speecht5_b200.build import LIB
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True).stdout
    elf = subprocess.run(["cuobjdump", "-elf", LIB], capture_output=True, text=True).stdout
    threads = None
    for sec in re.split(r"\n(?=\.nv\.info\.)", elf):
        m = re.match(r"\.nv\.info\.(\S+)", sec)
        t = re.search(r"EIATTR_MAX_THREADS\s*\n\s*Format:\s*\S+\s*\n\s*Value:\s*(0x[0-9a-f]+) (0x[0-9a-f]+) (0x[0-9a-f]+)",
                      sec)
        if m and t and "attn_fused_bwd_kernel" in m.group(1):
            threads = int(t.group(1), 16) * int(t.group(2), 16) * int(t.group(3), 16)
    assert threads == 288, f"attn_fused_bwd_kernel launch bounds: {threads} threads"
    found = [m for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) \S+ LOCAL:(\d+)", res)
             if "attn_fused_bwd_kernel" in m.group(1)]
    assert len(found) == 1, [m.group(1) for m in found]
    regs, stack, local = (int(found[0].group(i)) for i in (2, 3, 4))
    assert regs <= 168, f"attn_fused_bwd_kernel: {regs} registers"
    assert stack == 0 and local == 0, f"attn_fused_bwd_kernel spills: STACK {stack}, LOCAL {local}"
