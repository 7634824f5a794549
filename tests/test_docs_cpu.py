"""Documentation integrity: reference citations (file:line) in sources, header and docs resolve against the reference
tree (oracle/ref_loader.py: ST5_REFERENCE_ROOT; the check skips where that tree is not available)."""
import os
import subprocess
import sys

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


@pytest.mark.skipif(not os.path.isdir(os.environ.get("ST5_REFERENCE_ROOT", "/root/reference")),
                    reason="reference tree not available: the citations are checked against its source files")
def test_reference_citations_resolve():
    r = subprocess.run([sys.executable, os.path.join(ROOT, "tools", "check_citations.py")], capture_output=True,
                       text=True, timeout=300)
    assert r.returncode == 0, r.stdout[-2000:]


def test_header_entry_points_all_cite_the_reference():
    """include/speecht5_b200.h: every exported entry point carries a doc comment that names what it replaces."""
    import re
    text = open(os.path.join(ROOT, "include", "speecht5_b200.h")).read()
    protos = list(re.finditer(r"\n(?:ST5_API\s+)?(?:int|void|const char\s*\*|size_t)\s+(st5_\w+)\s*\(", text))
    assert len(protos) > 20
    missing = []
    for m in protos:
        if m.group(1) in ("st5_version", "st5_last_error", "st5_device_ok", "st5_cast_bf16", "st5_ln_bwd_blocks"):
            continue  # library plumbing without a reference counterpart
        block = text[max(0, m.start() - 2500): m.start()]  # the section comment above the prototype group
        if not re.search(r"\.py:\d+", block):
            missing.append(m.group(1))
    assert not missing, missing


def test_integration_md_binding_matches_the_shipped_ctypes_struct():
    """The ctypes stub INTEGRATION.md shows a maintainer is the struct the package itself binds (same field names, order
    and C types), and its example call compiles."""
    import ctypes
    import re
    text = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    block = text[text.index("class st5_gemm_args(ctypes.Structure)"): text.index("lib.st5_gemm_bf16.argtypes")]
    ns = {"ctypes": ctypes}
    exec(block, ns)  # the documentation snippet itself
    doc_fields = [(n, t) for n, t in ns["st5_gemm_args"]._fields_]
    from speecht5_b200._lib import GemmArgs
    assert [(n, t) for n, t in GemmArgs._fields_] == doc_fields
    assert ctypes.sizeof(GemmArgs) == ctypes.sizeof(ns["st5_gemm_args"])
    assert re.search(r"act=2\b", text) and "ST5_ACT_GELU" in open(os.path.join(ROOT, "include", "speecht5_b200.h")).read()


def test_no_gpu_test_is_gated_behind_an_environment_variable():
    """No GPU test hides behind an ST5_TEST_* opt-in variable: a GPU test either runs or does not exist."""
    import glob
    import re
    for path in glob.glob(os.path.join(ROOT, "tests", "*_gpu.py")):
        src = open(path).read()
        assert not re.findall(r"ST5_TEST_[A-Z0-9]+", src), path
        assert "skipif(os.environ" not in src, path

