"""The resource budget of the waveform front-end (conv0_*) and decode-attention (attn_decode_*) kernels, read from the
built library like tests/test_gemm_regs_cpu.py. The block size comes from each kernel's launch bounds
(EIATTR_MAX_THREADS): the GroupNorm-mode launcher runs one thread per channel, up to 512 per block, and a kernel
without launch bounds lets the compiler use more registers than such a block can hold -- every launch then fails with
'too many resources requested', which no CPU check would notice. Registers x threads must fit the 64 K register file
of an SM, and no kernel may spill to local memory."""
import re
import shutil
import subprocess

import pytest


def test_frontend_and_decode_registers_fit_their_launch_bounds():
    from speecht5_b200.build import LIB
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    res = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True).stdout
    elf = subprocess.run(["cuobjdump", "-elf", LIB], capture_output=True, text=True).stdout
    ours = re.compile(r"conv0_|attn_decode_")
    threads = {}
    for sec in re.split(r"\n(?=\.nv\.info\.)", elf):
        m = re.match(r"\.nv\.info\.(\S+)", sec)
        t = re.search(r"EIATTR_MAX_THREADS\s*\n\s*Format:\s*\S+\s*\n\s*Value:\s*(0x[0-9a-f]+) (0x[0-9a-f]+) (0x[0-9a-f]+)",
                      sec)
        if m and t and ours.search(m.group(1)):
            threads[m.group(1)] = int(t.group(1), 16) * int(t.group(2), 16) * int(t.group(3), 16)
    seen = set()
    for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+) STACK:(\d+) \S+ LOCAL:(\d+)", res):
        name, regs, stack, local = m.group(1), int(m.group(2)), int(m.group(3)), int(m.group(4))
        if not ours.search(name):
            continue
        assert name in threads, f"{name}: no launch bounds"
        nthr = threads[name]
        assert nthr * (-(-regs // 8) * 8) <= 65536, (name, regs, nthr)
        assert stack == 0 and local == 0, f"{name} spills: STACK {stack}, LOCAL {local}"
        seen.add(name)
    # GroupNorm mode: stats, finalize, apply x2, bwd_sums x2, bwd_finalize, bwd_w x2, reduce_w; LayerNorm mode: fwd x2,
    # bwd x 2 dtypes x 2 KH; decode: split x2, combine
    assert sum("conv0_" in n for n in seen) == 10 + 6, sorted(seen)
    assert sum("attn_decode_" in n for n in seen) == 3, sorted(seen)
