"""Compiler report of the clustering kernels (csrc/cluster.cu) for sm_90a, without a GPU: every kernel instantiation
is listed, with no stack frame and no spills.  Skipped where nvcc is missing."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "pytorch_geometric_b200", "csrc", "cluster.cu")


@pytest.fixture(scope="module")
def report(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    from pytorch_geometric_b200 import _build
    out = tmp_path_factory.mktemp("ptxas") / "cluster.cubin"
    cmd = [nvcc, *_build.ARCH_FLAGS, "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-DB200MP_BUILD",
           "-I", _build.INCLUDE, "-Xptxas", "-v", "-cubin", SRC, "-o", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout + r.stderr


def _kernels(text):
    lines = text.splitlines()
    return {m.group(1): lines[i + 1] for i, line in enumerate(lines[:-1])
            if (m := re.search(r"Function properties for (\S*cluster_\w*kernel\S*)", line))}


def test_every_instantiation_is_reported(report):
    names = _kernels(report)
    # graclus: index dtype x weight (none, fp32, bf16, fp64); grid: value dtype (fp32, fp64)
    counts = {"cluster_graclus_kernel": 2 * 4, "cluster_grid_kernel": 2, "cluster_minmax_kernel": 2,
              "cluster_minmax_fold_kernel": 2}
    for kern, n in counts.items():
        assert sum(f"{len(kern)}{kern}" in k for k in names) == n, kern
    for w in ("GcNoWeight", "IifE", "IlfE", "bfloat16", "IidE", "IldE"):
        assert any(w in k for k in names if "graclus" in k), w


def test_no_stack_frame_and_no_spills(report):
    bad = {k: v.strip() for k, v in _kernels(report).items()
           if not re.search(r"\b0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", v)}
    assert not bad, bad
