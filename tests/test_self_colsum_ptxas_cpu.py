"""Compiler report of the self-loop column-sum sweep (csr_reduce_kernel with SELF_COLSUM, csrc/csr_reduce.cuh) for
sm_90a, without a GPU: every lane-group shape fits the 64-register cap of its launch (128-thread CTAs, 8 resident per
SM), and the fp32 shapes keep the grid-stride loop's state and the edge loop's broadcast values in registers -- no
spill reloads in front of the gathers.  Skipped where nvcc is missing."""
import os
import re
import shutil
import subprocess

import pytest

ROOT = os.path.dirname(os.path.dirname(os.path.abspath(__file__)))

# one call per (value, index) dtype pair instantiates the sweep for every lane-group shape
TU = """
#include "csr_reduce.cuh"
using namespace b200mp;
template <typename T, typename I>
void instantiate() {
    LongRowPlan plan{};
    int64_t parts = 0;
    csr_sum_self_colsum<T, I>(nullptr, nullptr, nullptr, nullptr, nullptr, 0, 0, plan, nullptr, 1, parts, nullptr);
}
void all() {
    instantiate<float, int32_t>();
    instantiate<float, int64_t>();
    instantiate<__nv_bfloat16, int32_t>();
    instantiate<__nv_bfloat16, int64_t>();
}
"""


@pytest.fixture(scope="module")
def report(tmp_path_factory):
    nvcc = shutil.which("nvcc") or "/usr/local/cuda/bin/nvcc"
    if not os.path.exists(nvcc):
        pytest.skip("nvcc not available")
    from pytorch_geometric_b200 import _build
    d = tmp_path_factory.mktemp("ptxas")
    src = d / "self_colsum.cu"
    src.write_text(TU)
    cmd = [nvcc, *_build.ARCH_FLAGS, "-O3", "-std=c++17", "--expt-relaxed-constexpr", "-DB200MP_BUILD",
           "-I", _build.INCLUDE, "-I", _build.CSRC, "-Xptxas", "-v", "-cubin", str(src), "-o", str(d / "self_colsum.cubin")]
    r = subprocess.run(cmd, capture_output=True, text=True)
    assert r.returncode == 0, r.stdout + r.stderr
    return r.stdout + r.stderr


def _sweeps(text):
    """{mangled name: (registers, properties line)} of every SELF_COLSUM csr_reduce_kernel instantiation (template flag
    Lb1 last)."""
    lines = text.splitlines()
    out = {}
    for i, line in enumerate(lines[:-2]):
        m = re.search(r"Function properties for (\S*csr_reduce_kernel\S*Lb1EEEv\S*)", line)
        if m:
            out[m.group(1)] = (int(re.search(r"Used (\d+) registers", lines[i + 2]).group(1)), lines[i + 1].strip())
    return out


def test_every_lane_group_shape_is_instantiated(report):
    # G = 1, 2, 4, 8, 16 with one vector per lane, G = 32 with 1, 2 or 4: 8 shapes x 2 value x 2 index dtypes
    assert len(_sweeps(report)) == 32


def test_registers_allow_eight_ctas_per_sm(report):
    # 65536 registers / (128 threads x 8 CTAs) = 64
    bad = {k: r for k, (r, _) in _sweeps(report).items() if r > 64}
    assert not bad, bad


def test_fp32_sweeps_do_not_spill(report):
    bad = {k: p for k, (_, p) in _sweeps(report).items() if "bfloat16" not in k
           and not re.search(r"\b0 bytes stack frame, 0 bytes spill stores, 0 bytes spill loads", p)}
    assert not bad, bad
