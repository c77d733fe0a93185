"""GCNConv's bias gradient from the transposed sweep (b200mp_spmm_csr_self_colsum, csrc/csr_reduce.cuh SELF_COLSUM).

On a graph with exactly one self-loop per row, the weighted-sum sweep also adds the unweighted row of each self-loop edge
into per-CTA column partials, so that sum_i x[i, :] comes out of the sweep without a second read of x.  The sweep's own
output must stay bit-identical to b200mp_spmm_csr's, and the column sum must match a float64 column sum.  Graphs that
lack the property (no self-loops added, adopted or trimmed CSRs) keep the separate column-sum pass."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from pytorch_geometric_b200 import ops, utils as U  # noqa: E402
from pytorch_geometric_b200.graph import CSRGraph  # noqa: E402
from pytorch_geometric_b200.nn import GCNConv  # noqa: E402

DEV = "cuda"


def gcn_graph(n, e, seed, hubs=True, chunk=64):
    """gcn_norm_graph of a graph whose sources are power-law (a few hub sources hold ~30 % of the edges, so the rows of
    the transposed CSR are cut into chunks) and lie in [0, n / 2): rows n / 2 .. n - 1 of the transposed CSR hold only
    their self-loop."""
    gen = torch.Generator(device=DEV).manual_seed(seed)
    src = torch.randint(0, max(n // 2, 1), (e, ), device=DEV, generator=gen)
    if hubs:
        hub = torch.randint(0, 5, (e, ), device=DEV, generator=gen)
        src = torch.where(torch.rand(e, device=DEV, generator=gen) < 0.3, hub, src)
    dst = torch.randint(0, n, (e, ), device=DEV, generator=gen)
    g = U.gcn_norm_graph(torch.stack([src, dst]), None, n, chunk=chunk)
    g.build_transpose()
    return g


def check_colsum(colsum, x):
    ref = x.double().sum(0)
    tol = 1e-5 * x.double().abs().sum(0) + 1e-30
    err = (colsum.double() - ref).abs()
    assert colsum.dtype == torch.float32 and colsum.shape == (x.size(1), )
    assert bool((err <= tol).all()), float((err / tol).max())


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("F", [1, 64, 256, 264])
def test_out_bit_identical_and_colsum_on_a_chunked_power_law_graph(dtype, F):
    n = 3000
    g = gcn_graph(n, 30000, seed=F)
    assert g.one_self_loop_per_row
    assert g.plan_t.n_long > 0                                         # hub rows of A^T are walked in chunks
    deg_t = (g.rowptr_t[1:] - g.rowptr_t[:-1]).long()
    assert int((deg_t == 1).sum()) >= n // 2 - 5                       # rows whose only edge is the self-loop
    x = torch.randn(n, F, device=DEV, generator=torch.Generator(device=DEV).manual_seed(7)).to(dtype)
    want = ops.spmm_csr(g.rowptr_t, g.col_t, g.val_t, x, n, "sum", g.plan_t)
    out, colsum = ops.spmm_csr_self_colsum(g.rowptr_t, g.col_t, g.val_t, x, g.plan_t)
    assert out.dtype == dtype and torch.equal(out, want)
    check_colsum(colsum, x)
    out2, colsum2 = ops.spmm_csr_self_colsum(g.rowptr_t, g.col_t, g.val_t, x, g.plan_t)
    assert torch.equal(out2, out) and torch.equal(colsum2, colsum)    # deterministic


def test_int64_indices():
    n, F = 2000, 256
    g = gcn_graph(n, 20000, seed=3)
    rowptr, col = g.rowptr_t.long(), g.col_t.long()
    plan = ops.LongRowPlan(rowptr, g.chunk)
    x = torch.randn(n, F, device=DEV)
    out, colsum = ops.spmm_csr_self_colsum(rowptr, col, g.val_t, x, plan)
    assert torch.equal(out, ops.spmm_csr(rowptr, col, g.val_t, x, n, "sum", plan))
    check_colsum(colsum, x)


@pytest.mark.parametrize("F", [64, 256])
@pytest.mark.parametrize("n", [1, 3])
def test_fewer_rows_than_one_ctas_lane_groups(n, F):
    g = gcn_graph(n, 4, seed=n, hubs=False)
    x = torch.randn(n, F, device=DEV)
    out, colsum = ops.spmm_csr_self_colsum(g.rowptr_t, g.col_t, g.val_t, x, g.plan_t)
    assert torch.equal(out, ops.spmm_csr(g.rowptr_t, g.col_t, g.val_t, x, n, "sum", g.plan_t))
    check_colsum(colsum, x)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_no_rows(dtype):
    rowptr = torch.zeros(1, dtype=torch.int32, device=DEV)
    col = torch.zeros(0, dtype=torch.int32, device=DEV)
    val = torch.zeros(0, device=DEV)
    out, colsum = ops.spmm_csr_self_colsum(rowptr, col, val, torch.zeros(0, 256, device=DEV, dtype=dtype))
    assert out.shape == (0, 256) and torch.equal(colsum, torch.zeros(256, device=DEV))


def kernels_timed(fn):
    ops.PROFILE.reset(enabled=True)
    try:
        fn()
        return ops.PROFILE.summary()
    finally:
        ops.PROFILE.reset(enabled=False)


def layer_step(conv, x, graph, gout):
    x = x.detach().clone().requires_grad_()
    conv.zero_grad(set_to_none=True)
    out = conv(x, graph)
    out.backward(gout)
    return out, x.grad, conv.lin.weight.grad, conv.bias.grad


def test_gcnconv_takes_the_bias_gradient_from_the_sweep():
    n, F = 4000, 256
    g = gcn_graph(n, 40000, seed=11)
    torch.manual_seed(0)
    conv = GCNConv(F, F).to(DEV)
    with torch.no_grad():
        conv.bias.normal_()
    x = torch.randn(n, F, device=DEV)
    gout = torch.randn(n, F, device=DEV)
    res = {}
    kern = kernels_timed(lambda: res.update(fused=layer_step(conv, x, g, gout)))
    assert "column_sum" not in kern and kern["spmm_csr"]["calls"] == 2     # forward sweep, transposed sweep
    # the same structure without the property: the separate column sum, as before
    plain = g.with_values(g.val)
    plain.one_self_loop_per_row = False
    kern = kernels_timed(lambda: res.update(plain=layer_step(conv, x, plain, gout)))
    assert kern["column_sum"]["calls"] == 1
    (out_f, gx_f, gw_f, gb_f), (out_p, gx_p, gw_p, gb_p) = res["fused"], res["plain"]
    assert torch.equal(out_f, out_p) and torch.equal(gx_f, gx_p) and torch.equal(gw_f, gw_p)
    assert torch.equal(gb_p, ops.column_sum(gout))
    check_colsum(gb_f, gout)


def test_graphs_without_the_property_keep_the_column_sum():
    n, F = 1000, 64
    gen = torch.Generator(device=DEV).manual_seed(5)
    ei = torch.randint(0, n, (2, 8000), device=DEV, generator=gen)
    torch.manual_seed(0)
    conv = GCNConv(F, F, add_self_loops=False).to(DEV)
    x = torch.randn(n, F, device=DEV)
    gout = torch.randn(n, F, device=DEV)
    g_nl = U.gcn_norm_graph(ei, None, n, add_self_loops=False)
    g = U.gcn_norm_graph(ei, None, n)
    adopted = CSRGraph.from_csr(g.rowptr, g.col, n, g.val)            # same edges, self-loops included
    trimmed = adopted.trim(n, n, g.num_edges)
    assert not g_nl.one_self_loop_per_row and not adopted.one_self_loop_per_row and not trimmed.one_self_loop_per_row
    for graph in (g_nl, adopted, trimmed):
        res = {}
        kern = kernels_timed(lambda: res.update(r=layer_step(conv, x, graph, gout)))
        assert kern["column_sum"]["calls"] == 1
        assert torch.equal(res["r"][3], ops.column_sum(gout))


def test_bias_without_gradient_takes_the_plain_sweep(monkeypatch):
    n, F = 1000, 256
    g = gcn_graph(n, 8000, seed=2)
    conv = GCNConv(F, F).to(DEV)
    conv.bias.requires_grad_(False)
    x = torch.randn(n, F, device=DEV, requires_grad=True)
    gout = torch.randn(n, F, device=DEV)

    def unexpected(*args, **kw):
        raise AssertionError("the bias needs no gradient: no column sum to fuse")

    monkeypatch.setattr(ops, "spmm_csr_self_colsum", unexpected)
    kern = kernels_timed(lambda: conv(x, g).backward(gout))
    assert "column_sum" not in kern and kern["spmm_csr"]["calls"] == 2 and conv.bias.grad is None
