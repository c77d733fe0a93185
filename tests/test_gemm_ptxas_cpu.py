"""Compiler report of the 3xTF32 GEMM (csrc/gemm_tf32x3.cu) for sm_90a, without a GPU.

The consumer warpgroups hold two m64 accumulators and one A fragment set per half inside their setmaxnreg budget;
a spill would put local-memory traffic on the MMA path.  ptxas also must not serialize the wgmma instructions
(warnings C7518 / C7519, which a wait on an in-flight group or a register dependence it cannot prove safe brings
back).  Only the normal build is held to this; the -DB200MP_GEMM_TRACE build of benchmarks/gemm_stalls.py is not.  Skipped where nvcc is missing."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))
SRC = os.path.join(ROOT, "pytorch_geometric_b200", "csrc", "gemm_tf32x3.cu")


def _nvcc():
    cand = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    return cand if os.path.exists(cand) else None


@pytest.fixture(scope="module")
def report(tmp_path_factory):
    nvcc = _nvcc()
    if nvcc is None:
        pytest.skip("nvcc not available")
    from pytorch_geometric_b200 import _build
    out = tmp_path_factory.mktemp("ptxas") / "gemm_tf32x3.cubin"
    cmd = [nvcc, *_build.ARCH_FLAGS, "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-DB200MP_BUILD",
           "-I", _build.INCLUDE, "-Xptxas", "-v", "-cubin", SRC, "-o", str(out)]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout + r.stderr


def _kernels(text):
    """{mangled name: properties line} of every gemm_tf32x3_kernel instantiation."""
    props = {}
    lines = text.splitlines()
    for i, line in enumerate(lines):
        m = re.search(r"Function properties for (\S*gemm_tf32x3_kernel\S*)", line)
        if m and i + 1 < len(lines):
            props[m.group(1)] = lines[i + 1]
    return props


def test_every_instantiation_is_reported(report):
    # 12 forms: BN in {64, 128} x (A, B) layouts / pre-split, plus the two grouped layouts
    assert len(_kernels(report)) == 12


def test_no_spills(report):
    bad = {k: v.strip() for k, v in _kernels(report).items()
           if not re.search(r"\b0 bytes spill stores, 0 bytes spill loads", v)}
    assert not bad, bad


def test_no_wgmma_serialization(report):
    assert not re.search(r"C751[89]", report), [l for l in report.splitlines() if re.search(r"C751[89]", l)]
