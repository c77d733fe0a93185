"""Compiler report of the random-walk kernels (csrc/random_walk.cu) for sm_90a, without a GPU: every kernel
instantiation is listed, with no stack frame and no spills.  Skipped where nvcc is missing."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "pytorch_geometric_b200", "csrc", "random_walk.cu")


@pytest.fixture(scope="module")
def report(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    from pytorch_geometric_b200 import _build
    out = tmp_path_factory.mktemp("ptxas") / "random_walk.cubin"
    cmd = [nvcc, *_build.ARCH_FLAGS, "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-DB200MP_BUILD",
           "-I", _build.INCLUDE, "-Xptxas", "-v", "-cubin", SRC, "-o", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout + r.stderr


def _kernels(text):
    lines = text.splitlines()
    return {m.group(1): lines[i + 1] for i, line in enumerate(lines[:-1])
            if (m := re.search(r"Function properties for (\S*walk_\w*kernel\S*)", line))}


def test_every_instantiation_is_reported(report):
    names = _kernels(report)
    # the walk: index dtype x (uniform, node2vec); the row-order check: index dtype
    counts = {"walk_kernel": 2 * 2, "walk_rows_unsorted_kernel": 2}
    for kern, n in counts.items():
        assert sum(f"{len(kern)}{kern}" in k for k in names) == n, kern
    for inst in ("walk_kernelIiLb0E", "walk_kernelIiLb1E", "walk_kernelIlLb0E", "walk_kernelIlLb1E"):
        assert any(inst in k for k in names), inst


def test_no_stack_frame_and_no_spills(report):
    bad = {k: v.strip() for k, v in _kernels(report).items()
           if not re.search(r"\b0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", v)}
    assert not bad, bad
