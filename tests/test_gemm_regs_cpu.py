"""The wgmma GEMM's resource budget, read from the built library: the block size comes from the kernel's launch bounds
(EIATTR_MAX_THREADS, the same constant gemm_launch launches with), so a change of the warp layout is checked at its
real size. Registers x threads must fit the 64 K register file of an SM (otherwise every launch fails with 'too many
resources requested', which no CPU check would notice), and no instantiation may spill to local memory."""
import re
import shutil
import subprocess

import pytest


def test_gemm_registers_fit_the_real_block_size():
    from speecht5_b200.build import LIB
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True).stdout
    elf = subprocess.run(["cuobjdump", "-elf", LIB], capture_output=True, text=True).stdout
    threads = {}
    for sec in re.split(r"\n(?=\.nv\.info\.)", elf):
        m = re.match(r"\.nv\.info\.(\S*gemm_bf16_wgmma\S*)", sec)
        t = re.search(r"EIATTR_MAX_THREADS\s*\n\s*Format:\s*\S+\s*\n\s*Value:\s*(0x[0-9a-f]+) (0x[0-9a-f]+) (0x[0-9a-f]+)",
                      sec)
        if m and t:
            threads[m.group(1)] = int(t.group(1), 16) * int(t.group(2), 16) * int(t.group(3), 16)
    seen = 0
    for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) \S+ LOCAL:(\d+)", res):
        name, regs, stack, local = m.group(1), int(m.group(2)), int(m.group(3)), int(m.group(4))
        if "gemm_bf16_wgmma" not in name:
            continue
        assert name in threads, f"{name}: no launch bounds"
        nthr = threads[name]
        assert nthr * (-(-regs // 8) * 8) <= 65536, (name, regs, nthr)
        assert stack == 0 and local == 0, f"{name} spills: STACK {stack}, LOCAL {local}"
        seen += 1
    assert seen == 8  # BN in {64, 128} x operand majors
