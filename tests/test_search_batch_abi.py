"""CPU-side checks of lb2_index_search_batch: the ctypes structs match the header's layout (a C snippet compiled
against include/lance_b200.h), and search_batch refuses bad shapes before it calls the library."""
import ctypes as C
import os
import shutil
import subprocess

import numpy as np
import pytest

import lance_b200 as lb
from lance_b200 import _lib

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

FIELDS = {"lb2_query_filter": (_lib.QueryFilter, ["allow_bitmap", "has_max_len", "max_len", "mask_ids", "num_mask_ids"]),
          "lb2_query_params": (_lib.QueryParams, ["k", "nprobes", "minimum_nprobes", "maximum_nprobes", "refine_factor",
                                                  "filter", "ef", "has_lower_bound", "has_upper_bound", "lower_bound",
                                                  "upper_bound"])}


@pytest.mark.skipif(shutil.which("cc") is None, reason="needs a C compiler")
def test_struct_layout_matches_header(tmp_path):
    lines = ["#include <stdio.h>", "#include <stddef.h>", '#include "lance_b200.h"', "int main(void) {"]
    for name, (_, fields) in FIELDS.items():
        lines.append(f'  printf("{name} %zu\\n", sizeof({name}));')
        lines += [f'  printf("{name}.{f} %zu\\n", offsetof({name}, {f}));' for f in fields]
    lines += ["  return 0;", "}"]
    src, exe = tmp_path / "layout.c", tmp_path / "layout"
    src.write_text("\n".join(lines) + "\n")
    subprocess.run(["cc", "-I", os.path.join(ROOT, "include"), str(src), "-o", str(exe)], check=True)
    got = dict(line.split() for line in subprocess.run([str(exe)], check=True, capture_output=True,
                                                       text=True).stdout.splitlines())
    for name, (cls, fields) in FIELDS.items():
        assert int(got[name]) == C.sizeof(cls), name
        assert [f for f, _ in cls._fields_] == fields
        for f in fields:
            assert int(got[f"{name}.{f}"]) == getattr(cls, f).offset, (name, f)


class _NoLibrary(lb.IvfPqIndex):
    """an index whose handle must never reach the library"""

    def __init__(self):
        super().__init__(None)


@pytest.mark.parametrize("kw", [
    dict(k=np.array([5, 5, 5])),                                   # k of the wrong length
    dict(k=np.array([5, 0, 5, 5])),                                # k = 0
    dict(nprobes=np.array([1, 2])),                                # nprobes of the wrong length
    dict(nprobes=-1),                                              # nprobes < 0
    dict(nprobes=0, minimum_nprobes=0),                            # minimum_nprobes = 0 for the probe rule
    dict(nprobes=None, maximum_nprobes=np.array([1, 2])),          # maximum_nprobes of the wrong length
    dict(refine_factor=2),                                         # refine without vectors
    dict(refine_factor=-1),
    dict(filter_of=0),                                             # no filters
    dict(filters=[np.zeros(1, np.uint64)], filter_of=np.array([0, 1, -1, 0])),
    dict(lower_bound=np.zeros(3, np.float32)),
    dict(ef=-1),
    dict(out=(np.empty((4, 3), np.uint64), np.empty((4, 3), np.float32))),   # rows shorter than the largest k
    dict(out=(np.empty((3, 5), np.uint64), np.empty((3, 5), np.float32))),   # wrong number of rows
])
def test_arguments_are_checked_before_the_library(kw):
    args = dict(k=5, nprobes=3)
    args.update(kw)
    with pytest.raises(ValueError):
        _NoLibrary().search_batch(np.zeros((4, 8), np.float32), **args)
