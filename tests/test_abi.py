"""CPU-side checks of the drop-in boundary: the C-ABI library loads, exports every symbol that
include/lance_b200.h declares, and fails loudly (no CPU fallback) without a GPU."""
import os
import re

import numpy as np
import pytest

import lance_b200 as lb
from lance_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))


def _declared_symbols():
    src = open(os.path.join(ROOT, "include", "lance_b200.h")).read()
    src = re.sub(r"/\*.*?\*/", "", src, flags=re.S)
    return sorted(set(re.findall(r"\b(lb2_[a-z0-9_]+)\s*\(", src)))


def test_library_exports_every_declared_symbol():
    L = _lib.lib()
    declared = _declared_symbols()
    assert len(declared) >= 35
    for s in declared:
        assert hasattr(L, s), f"{s} declared in include/lance_b200.h but not exported"
    assert sorted(_lib.EXPORTS) == declared


def test_version_and_error_buffer():
    assert b"sm_90a" in _lib.lib().lb2_version()


def test_product_never_imports_oracle():
    # the oracle is test infrastructure; the product package must not reference it
    for dirpath, _, files in os.walk(os.path.join(ROOT, "lance_b200")):
        for f in files:
            if f.endswith((".py", ".cu", ".cuh", ".h")):
                txt = open(os.path.join(dirpath, f)).read()
                assert "oracle" not in txt.replace("the oracle", "").replace("oracle/", "").replace("-problem oracle", "") \
                    or f in ("_lib.py",), f


def test_every_environment_knob_is_in_the_integration_table():
    """each LB2_* variable the library reads is listed in INTEGRATION.md's table of environment knobs"""
    names = set()
    csrc = os.path.join(ROOT, "lance_b200", "csrc")
    for f in os.listdir(csrc):
        if f.endswith((".cu", ".cuh")):
            names |= set(re.findall(r'getenv\(\s*"(LB2_[A-Z0-9_]+)"', open(os.path.join(csrc, f)).read()))
    assert "LB2_CHUNK_ROWS" in names and "LB2_MAX_RESIDENT_MB" in names
    doc = open(os.path.join(ROOT, "INTEGRATION.md")).read()
    table = doc.split("### Environment knobs", 1)[1].split("\n\n", 2)[1]
    assert table.startswith("| Variable |")
    documented = set(re.findall(r"`(LB2_[A-Z0-9_]+)", table))
    assert sorted(names - documented) == []


@pytest.mark.skipif(lb.device_count() > 0, reason="only meaningful on a box without a GPU")
def test_no_gpu_fails_loudly():
    with pytest.raises(lb.LanceB200Error) as e:
        lb.compute_partitions(np.zeros((4, 8), np.float32), np.zeros((10, 8), np.float32))
    assert e.value.status == _lib.NO_DEVICE
    with pytest.raises(lb.LanceB200Error):
        lb.IvfPqIndex.build(np.zeros((300, 16), np.float32), params=lb.IvfBuildParams(num_partitions=4, num_sub_vectors=2))


def test_header_is_plain_c11_and_cxx17(tmp_path):
    """the boundary is a C ABI: include/lance_b200.h must compile as C and as C++ with no CUDA / torch headers"""
    import shutil
    import subprocess
    root = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
    for cc, std, ext in (("gcc", "-std=c11", "c"), ("g++", "-std=c++17", "cc")):
        if shutil.which(cc) is None:
            continue
        src = tmp_path / f"use_header.{ext}"
        src.write_text('#include "lance_b200.h"\nint main(void) { return lb2_device_count == 0; }\n')
        out = subprocess.run([cc, std, "-Wall", "-Wextra", "-pedantic", "-fsyntax-only", "-I", os.path.join(root, "include"), str(src)],
                             capture_output=True, text=True)
        assert out.returncode == 0, out.stderr
