"""CPU: the C-ABI library loads and exports every symbol include/speecht5_b200.h declares; host-side plumbing."""
import ctypes
import os
import re

import pytest
import torch

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.fixture(scope="module")
def lib():
    from speecht5_b200.build import build
    build()
    from speecht5_b200 import _lib
    return _lib.load()


def test_header_symbols_are_exported(lib):
    hdr = open(os.path.join(ROOT, "include", "speecht5_b200.h")).read()
    declared = set(re.findall(r"\b(st5_[a-z0-9_]+)\s*\(", hdr))
    declared -= {"st5_gemm_args", "st5_attn_args"}
    assert len(declared) >= 19
    from speecht5_b200._lib import EXPORTS
    assert declared == set(EXPORTS), declared ^ set(EXPORTS)
    for name in declared:
        assert getattr(lib, name) is not None
    # every prototype in the ctypes table has as many parameters as the declaration in the header
    from speecht5_b200._lib import _PROTOS
    flat = re.sub(r"/\*.*?\*/", " ", hdr, flags=re.S)
    for name in declared:
        m = re.search(r"\b" + name + r"\s*\(([^;{]*?)\)\s*;", flat, flags=re.S)
        assert m, name
        params = m.group(1).strip()
        n = 0 if params in ("", "void") else params.count(",") + 1
        assert n == len(_PROTOS[name][1]), (name, n, len(_PROTOS[name][1]))


def test_version_and_error_text(lib):
    assert lib.st5_version() >= 100
    assert isinstance(lib.st5_last_error(), bytes)


def test_struct_layout_matches_header(tmp_path):
    """The ctypes mirrors in speecht5_b200/_lib.py must have exactly the layout a C compiler gives the structs of
    include/speecht5_b200.h: gcc compiles the header and prints sizeof / offsetof of every field."""
    import shutil
    import subprocess
    from speecht5_b200._lib import AttnArgs, GemmArgs
    if shutil.which("gcc") is None:
        pytest.skip("gcc not available")
    structs = {"st5_gemm_args": GemmArgs, "st5_attn_args": AttnArgs}
    lines = ['#include <stdio.h>', '#include <stddef.h>', '#include "speecht5_b200.h"', "int main(void) {"]
    for cname, cls in structs.items():
        lines.append(f'  printf("{cname} size %zu\\n", sizeof({cname}));')
        for fname, _ in cls._fields_:
            lines.append(f'  printf("{cname} {fname} %zu\\n", offsetof({cname}, {fname}));')
    lines += ["  return 0;", "}"]
    src = tmp_path / "layout.c"
    src.write_text("\n".join(lines))
    exe = tmp_path / "layout"
    subprocess.run(["gcc", "-std=c99", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    out = subprocess.run([str(exe)], check=True, capture_output=True, text=True).stdout.split("\n")
    seen = 0
    for line in out:
        if not line.strip():
            continue
        cname, field, val = line.split()
        cls = structs[cname]
        if field == "size":
            assert ctypes.sizeof(cls) == int(val), (cname, ctypes.sizeof(cls), val)
        else:
            assert getattr(cls, field).offset == int(val), (cname, field, getattr(cls, field).offset, val)
        seen += 1
    assert seen == 2 + len(GemmArgs._fields_) + len(AttnArgs._fields_)


def test_product_path_refuses_cpu_tensors():
    from speecht5_b200 import kernels as K
    a = torch.zeros(8, 8, dtype=torch.bfloat16)
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        K.gemm(a, a, torch.zeros(8, 8), M=8, N=8, K=8)


def test_missing_library_fails_loudly(monkeypatch, tmp_path):
    from speecht5_b200 import _lib
    monkeypatch.setattr(_lib, "_lib", None)
    monkeypatch.setattr(_lib, "LIB_PATH", str(tmp_path / "nope.so"))
    with pytest.raises(RuntimeError, match="no CPU fallback"):
        _lib.load()


def test_argument_errors_are_reported_without_touching_a_device(lib):
    """Error behaviour of the C ABI: negative return code + st5_last_error() text, decided before any CUDA call (so it
    holds on a box without a GPU); st5_device_ok() itself fails loudly here instead of pretending."""
    from speecht5_b200 import _lib
    g = _lib.GemmArgs()
    g.M, g.N, g.K, g.nb1, g.nb2 = 8, 8, 0, 1, 1
    assert lib.st5_gemm_bf16(ctypes.byref(g), None) == -2 and b"st5_gemm_bf16" in lib.st5_last_error()
    g.K, g.accumulate, g.c_fp32 = 8, 1, 0  # accumulation needs an fp32 output
    assert lib.st5_gemm_bf16(ctypes.byref(g), None) == -3
    a = _lib.AttnArgs()
    a.B, a.H, a.Tq, a.Tk, a.dtype = 1, 1, 4, 4, 0  # fp32 activations: the fused kernels are bf16 only
    assert lib.st5_attn_fused_fwd(ctypes.byref(a), None, None, None, None, None) == -2 and b"bf16" in lib.st5_last_error()
    a.dtype, a.Tk = 1, 400
    assert lib.st5_attn_fused_fwd(ctypes.byref(a), None, None, None, None, None) == -2
    if not torch.cuda.is_available():
        assert lib.st5_device_ok() != 0
    with pytest.raises(RuntimeError, match="st5_gemm_bf16"):
        _lib.check(-2, "st5_gemm_bf16")


def test_register_budget_of_the_wide_kernels(lib):
    """A launch fails with 'too many resources requested' when registers x allocated warps exceed the 64 K file. Warps
    are allocated four at a time, so a 9-warp block (288 threads: both attention kernels) pays for 12 and the 12-warp
    GEMM block for 12: 168 registers per thread is the ceiling. (A build over the ceiling passes every CPU check and
    fails every launch on the GPU; ptxas does not know the block size unless __launch_bounds__ says so.)"""
    import shutil
    import subprocess
    from speecht5_b200.build import LIB
    if shutil.which("cuobjdump") is None:
        pytest.skip("cuobjdump not available")
    out = subprocess.run(["cuobjdump", "-res-usage", LIB], capture_output=True, text=True).stdout
    threads = {"gemm_bf16_wgmma": (384, 1), "attn_fused_bwd_kernel": (288, 1), "attn_flash_fwd_kernelILb1": (288, 1),
               "attn_flash_fwd_kernelILb0": (288, 1)}  # (threads per block, blocks that must fit one SM)
    seen = 0
    for m in re.finditer(r"Function (\S+):\s*\n\s*REG:(\d+)", out):
        name, regs = m.group(1), int(m.group(2))
        for key, (nthr, ctas) in threads.items():
            if key in name:
                warps = -(-(nthr // 32) // 4) * 4
                assert ctas * warps * 32 * (-(-regs // 8) * 8) <= 65536, (name, regs, nthr, ctas)
                seen += 1
    assert seen >= 10
