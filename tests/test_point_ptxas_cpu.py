"""Compiler report of the point-cloud kernels (csrc/point.cu) for sm_90a, without a GPU: every kernel instantiation is
listed, with no stack frame and no spills.  Skipped where nvcc is missing."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "pytorch_geometric_b200", "csrc", "point.cu")


@pytest.fixture(scope="module")
def report(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    from pytorch_geometric_b200 import _build
    out = tmp_path_factory.mktemp("ptxas") / "point.cubin"
    cmd = [nvcc, *_build.ARCH_FLAGS, "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-DB200MP_BUILD",
           "-I", _build.INCLUDE, "-Xptxas", "-v", "-cubin", SRC, "-o", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout + r.stderr


def _kernels(text):
    lines = text.splitlines()
    return {m.group(1): lines[i + 1] for i, line in enumerate(lines[:-1])
            if (m := re.search(r"Function properties for (\S*point_\w*kernel\S*)", line))}


def test_every_instantiation_is_reported(report):
    names = _kernels(report)
    # the sweep: value dtype x selector (three register lists, the shared-memory list, radius count and fill) x staged
    counts = {"point_sweep_kernel": 2 * 6 * 2, "point_fps_kernel": 2, "point_fps_count_kernel": 1,
              "point_scan_kernel": 1, "point_compact_kernel": 1}
    for kern, n in counts.items():
        assert sum(f"{len(kern)}{kern}" in k for k in names) == n, kern
    for sel in ("PtRegTopKILi8E", "PtRegTopKILi16E", "PtRegTopKILi32E", "PtSmemTopK", "PtRadiusILb0E", "PtRadiusILb1E"):
        assert sum(sel in k for k in names) == 4, sel


def test_no_stack_frame_and_no_spills(report):
    bad = {k: v.strip() for k, v in _kernels(report).items()
           if not re.search(r"\b0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", v)}
    assert not bad, bad
