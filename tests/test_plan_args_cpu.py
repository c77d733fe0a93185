"""Every C-ABI entry point that takes a long-row plan rejects a malformed one with B200MP_ERR_INVALID_ARG before it
launches anything: include/b200mp.h requires n_long_rows >= 0 and n_chunks >= 0, and with long rows the row list, the
chunk offsets, a positive chunk and (where the sweep writes them) the fp32 partials.  The softmax- and power-mean-
aggregation entry points also refuse power mean's clamp bounds out of order, and a parameter gradient whose rows do
not fit in shared memory, before they launch anything."""
import re

import numpy as np
import pytest
import torch

import pytorch_geometric_b200 as pgb
from pytorch_geometric_b200 import _build

# The calls below pass host addresses where the library expects device buffers.  Without a device a plan that slips
# through its check fails at the launch (B200MP_ERR_CUDA); on a GPU it would launch a kernel on those addresses.
pytestmark = pytest.mark.skipif(torch.cuda.is_available(), reason="passes host buffers as device pointers")

INVALID_ARG = -1
UNSUPPORTED = -2

# entry point -> its plans, each as the names of its (n_long_rows, n_chunks, partials) arguments; partials is None for
# the sweeps that only split rows and write no partials
PLANS = {
    "spmm_csr": [("n_long_rows", "n_chunks", "partials")],
    "segment_csr": [("n_long_rows", "n_chunks", "partials")],
    "multi_aggr_csr": [("n_long_rows", "n_chunks", "partials")],
    "edge_relu_csr": [("n_long_rows", "n_chunks", "partials")],
    "edge_relu_backward_x": [("n_long_rows", "n_chunks", "partials")],
    "edge_relu_backward_edge": [("n_long_rows", "n_chunks", None)],
    "gated_csr": [("n_long_rows", "n_chunks", "partials")],
    "gated_backward_dst": [("n_long_rows", "n_chunks", "partials")],
    "gated_backward_src": [("n_long_rows", "n_chunks", "partials")],
    "cg_csr": [("n_long_rows", "n_chunks", "partials")],
    "cg_backward_dst": [("n_long_rows", "n_chunks", "partials")],
    "cg_backward_src": [("n_long_rows", "n_chunks", "partials")],
    "softmax_aggr_csr": [("n_long_rows", "n_chunks", "partials")],
    "softmax_aggr_backward_dst": [("n_long_rows", "n_chunks", None)],
    "softmax_aggr_backward_src": [("n_long_rows", "n_chunks", "partials")],
    "power_mean_csr": [("n_long_rows", "n_chunks", "partials")],
    "power_mean_backward_dst": [("n_long_rows", "n_chunks", None)],
    "power_mean_backward_src": [("n_long_rows", "n_chunks", "partials")],
    "pna_edge_stats": [("n_long_rows", "n_chunks", "partials")],
    "attn_csr_forward": [("n_long_rows", "n_chunks", "part_acc")],
    "attn_csr_backward": [("n_long_rows", "n_chunks", "partials"), ("n_long_rows_t", "n_chunks_t", "partials_t")],
    "gat_fused_csr": [("n_long_rows", "n_chunks", "part_acc")],
    "gat_fused_csr_backward": [("n_long_rows", "n_chunks", "partials")],
}

# Valid scalar arguments by name: 4 rows of 8 fp32 features, 8 edges, int64 indices, no long rows.  One head of 8
# channels with dot-product scores (mode 2) and an edge-feature row, so that every attention operand is in use; softmax
# and power-mean aggregation with relu(x + e) + eps messages, a scalar t or p and clamp bounds.
SCALARS = {
    "n_rows": 4, "n_cols": 4, "n_src": 4, "n_dst": 4, "n_edges": 8, "feat": 8, "width": 8, "ld": 8, "ld_u": 16,
    "ld_v": 16, "v_ld": 8, "heads": 1, "chan": 8, "v_stride": 0, "k_stride": 0, "q_stride": 0, "n_local_cols": 0,
    "peer_rows": 0, "chunk": 4, "n_long_rows": 0, "n_chunks": 0, "n_long_rows_t": 0, "n_chunks_t": 0,
    "reduce": 0, "flags": 0, "count_self_zero": 0, "message": 1, "t_mode": 1, "semi_grad": 0, "mode": 2,
    "p_mode": 1, "clamp_min": 1e-4, "clamp_max": 100.0,
    "idx_dtype": 1, "val_dtype": 0, "slope": 0.2, "scale": 1.0, "eps": 1e-7, "dropout_p": 0.0, "dropout_seed": 0,
}
# Pointers whose presence selects another mode with its own preconditions (halo rows, peer table, fused ReLU backward,
# tie mask), and the stream, stay NULL; every other pointer gets the address of a real 16-byte-aligned buffer.
NULL = {"stream", "x_halo", "peer_ptrs", "relu_mask", "hit_mask"}

MALFORMED = {
    "negative_long_rows": lambda nl, nc, part: {nl: -1},
    "negative_chunks": lambda nl, nc, part: {nl: 1, nc: -1},
    "zero_chunk": lambda nl, nc, part: {nl: 1, nc: 1, "chunk": 0},
    "no_chunk_offsets": lambda nl, nc, part: {nl: 1, nc: 1, nl.replace("n_long_rows", "chunk_ptr"): None},
    "no_partials": lambda nl, nc, part: {nl: 1, nc: 1, part: None},
}

_RAW = np.zeros(1 << 16, dtype=np.uint8)
BUF = _RAW.ctypes.data + (-_RAW.ctypes.data) % 16

with open(f"{_build.INCLUDE}/b200mp.h") as _f:
    _HEADER = re.sub(r"/\*.*?\*/", "", _f.read(), flags=re.S)
# entry point -> [(parameter name, is a pointer)] from its prototype
PROTOS = {m.group(1): [(re.findall(r"\w+", p)[-1], "*" in p) for p in m.group(2).split(",")]
          for m in re.finditer(r"\bb200mp_(\w+)\s*\(([^)]*)\)\s*;", _HEADER)}


def _call(name, **override):
    args = []
    for pname, is_ptr in PROTOS[name]:
        if pname in override:
            args.append(override[pname])
        elif is_ptr:
            args.append(None if pname in NULL else BUF)
        else:
            args.append(SCALARS[pname])
    return getattr(pgb.lib(), "b200mp_" + name)(*args)


VALID = [pytest.param(name, i, id=f"{name}-plan{i}") for name, plans in PLANS.items() for i in range(len(plans))]
BAD = [pytest.param(name, i, case, id=f"{name}-plan{i}-{case}") for name, plans in PLANS.items()
       for i, (_, _, part) in enumerate(plans) for case in MALFORMED if part or case != "no_partials"]


def test_every_plan_taking_entry_point_is_listed():
    takes_plan = {name for name, params in PROTOS.items() if {("long_rows", True), ("n_chunks", False)} <= set(params)}
    assert takes_plan == set(PLANS)


@pytest.mark.parametrize("long_rows", [False, True], ids=["no_long_rows", "long_rows"])
@pytest.mark.parametrize("name,plan", VALID)
def test_valid_plan_passes_the_checks(name, plan, long_rows):
    # the control for the cases below: the same call with a well-formed plan gets past argument checking
    nl, nc, _ = PLANS[name][plan]
    override = {nl: 1, nc: 1} if long_rows else {}
    assert _call(name, **override) != INVALID_ARG, pgb.lib().b200mp_last_error()


@pytest.mark.parametrize("name,plan,case", BAD)
def test_malformed_plan_is_rejected(name, plan, case):
    override = MALFORMED[case](*PLANS[name][plan])
    assert _call(name, **override) == INVALID_ARG, pgb.lib().b200mp_last_error()


@pytest.mark.parametrize("clamp", [dict(clamp_min=0.0), dict(clamp_min=-1.0), dict(clamp_min=2.0, clamp_max=1.0)],
                         ids=["zero_min", "negative_min", "max_below_min"])
@pytest.mark.parametrize("name", ["power_mean_csr", "power_mean_backward_dst", "power_mean_backward_src"])
def test_power_mean_rejects_a_bad_clamp(name, clamp):
    assert _call(name, **clamp) == INVALID_ARG, pgb.lib().b200mp_last_error()


# the sweeps that collect grad_t or grad_p, with a per-channel parameter and its gradient buffer
PARAM_GRAD = {"softmax_aggr_backward_dst": {"t_mode": 2}, "power_mean_backward_dst": {"p_mode": 2},
              "power_mean_backward_src": {"p_mode": 2}}


@pytest.mark.parametrize("feat", [20000, 8191], ids=["vector", "scalar"])
@pytest.mark.parametrize("name", sorted(PARAM_GRAD))
def test_too_wide_parameter_gradient_is_unsupported(name, feat):
    # one fp32 row of F per lane group: 4 groups of a vector CTA or 8 warps of a scalar CTA exceed 227 KB
    assert _call(name, feat=feat, **PARAM_GRAD[name]) == UNSUPPORTED, pgb.lib().b200mp_last_error()
    assert "shared memory" in pgb.lib().b200mp_last_error().decode()


@pytest.mark.parametrize("name", sorted(PARAM_GRAD))
def test_widest_parameter_gradient_gets_past_the_check(name):
    # 4 groups x 14000 channels x 4 bytes = 224000 bytes: within the limit
    assert _call(name, feat=14000, **PARAM_GRAD[name]) not in (INVALID_ARG, UNSUPPORTED), pgb.lib().b200mp_last_error()
