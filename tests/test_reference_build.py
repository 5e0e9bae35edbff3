"""oracle/_ref/libbsref.so, built from a reference checkout by oracle/ref/Makefile: it loads and exports every entry
oracle/ref_kernels.py binds, and no line of the reference sources it compiles is kept in the repository."""
import os
import subprocess

import pytest

from oracle import ref_kernels as rk

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
REF = os.environ.get("BLOCKSPARSE_REFERENCE") or "/root/reference"
SOURCES = ["ew_op_gpu.cu", "embedding_op_gpu.cu", "layer_norm_nc_op_gpu.cu", "layer_norm_cn_op_gpu.cu",
           "transformer_op_gpu.cu", "optimize_op_gpu.cu", "bst_softmax_op_gpu.cu", "blocksparse_l2_norm_op_gpu.cu",
           "ew_op_gpu.h", "gpu_types.h"]


def test_library_exports_every_bound_entry():
    if not rk.available():
        pytest.skip("oracle/_ref/libbsref.so not built (no reference checkout)")
    lib = rk.load()
    for name in rk.SIGNATURES:
        assert hasattr(lib, name), name


def test_no_reference_line_in_oracle():
    if not os.path.isfile(os.path.join(REF, "src", "ew_op_gpu.h")):
        pytest.skip("no reference checkout")
    lines = set()
    for f in SOURCES:
        with open(os.path.join(REF, "src", f), errors="replace") as fh:
            for line in fh:
                s = "".join(line.split())
                if len(s) >= 10:
                    lines.add(s)
    tracked = subprocess.run(["git", "ls-files", "oracle"], cwd=ROOT, capture_output=True, text=True)
    if tracked.returncode != 0:
        pytest.skip("not a git checkout")
    for path in tracked.stdout.split():
        with open(os.path.join(ROOT, path), errors="replace") as fh:
            for n, line in enumerate(fh, 1):
                s = "".join(line.split())
                assert s not in lines, "%s:%d repeats a line of the reference sources" % (path, n)
