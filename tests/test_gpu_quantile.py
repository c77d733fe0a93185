"""Quantile aggregation on the GPU (csrc/quantile.cu) against the numpy restatement of its contract
(tests/quantile_oracle.py): every interpolation with one and five q, fp32 and bf16, int32 and int64 indices, both
message forms (x gathered through a CSR, edge rows read through perm or in ptr order), rows of 0, 1, 2, short, medium
and hub length with a small chunk so that hub rows take the hub kernel and the transposed plan's combine, widths on
several lane-group shapes, ties, NaN, +-inf and +-0.  Outputs are bit-exact; gradients are exact for lower / higher /
nearest and within 1e-6 (fp32) / 1.6e-2 (bf16) of |g| for linear / midpoint.  Also: a second run's bits, no
device->host sync after warm-up, exact ranks past 2^24 messages, golden/quantile.npz through the nn mirrors, and the
plug-in against the unmodified reference on the CPU."""
import numpy as np
import pytest
import torch

import quantile_oracle as O
from conftest import load_golden

pytestmark = pytest.mark.gpu
DEV = "cuda"
CHUNK = 32
LENS = [0, 1, 2, 3, 5, 9, 17, 31, 40, 0, 1, 150, 700, 2, 0]


def _graph(rng, n_dst=40, n_src=50):
    """Destination rows of every length class, and source 0 a hub of 100 out-edges (more than CHUNK), so that the
    transposed sweep splits it by the transposed plan and folds the chunks."""
    lens = np.concatenate([LENS, rng.integers(0, 12, n_dst - len(LENS))])
    dst = np.repeat(np.arange(n_dst), lens)[rng.permutation(int(lens.sum()))]
    src = rng.integers(1, n_src, dst.size)
    src[rng.choice(dst.size, 100, replace=False)] = 0
    return src, dst, n_src, n_dst


def _values(rng, n, F, bf16):
    v = rng.standard_normal((n, F)).astype(np.float32)
    ties = rng.random((n, F)) < 0.3
    v[ties] = rng.integers(-2, 3, ties.sum()).astype(np.float32)
    special = rng.random((n, F)) < 0.05
    pool = np.array([0.0, -0.0, np.nan, np.inf, -np.inf], dtype=np.float32)
    v[special] = pool[rng.integers(0, len(pool), special.sum())]
    return O.rnd(v, bf16)


def _t(v, bf16):
    return torch.from_numpy(np.ascontiguousarray(v)).to(DEV, torch.bfloat16 if bf16 else torch.float32)


def _np(t):
    return t.detach().float().cpu().numpy()


def _g(rng, shape, bf16, interp):
    g = rng.standard_normal(shape).astype(np.float32)
    return g if O.out_is_f32(bf16, interp) else O.rnd(g, bf16)


def _assert_out(got, want):
    nan = np.isnan(want)
    assert (np.isnan(got) == nan).all(), "NaN positions differ"
    bad = got[~nan] != want[~nan]
    assert not bad.any(), f"{bad.sum()} outputs differ, e.g. {np.argwhere(~nan)[np.flatnonzero(bad)[:3]].tolist()}"


def _assert_grad(got, want, interp, bf16, g, positions=True):
    if positions:
        assert ((got != 0) == (want != 0)).all(), "gradient lands on other elements than the tie rule's"
    if interp in ("lower", "higher", "nearest"):
        assert np.array_equal(got, want)
    else:
        tol = (1.6e-2 if bf16 else 1e-6) * float(np.abs(g).max())
        assert np.abs(got - want).max() <= tol


def _run(form, interp, nq, bf16, idx_dtype, F, seed=0):
    from pytorch_geometric_b200 import functional as Fn
    from pytorch_geometric_b200 import ops
    from pytorch_geometric_b200.graph import CSRGraph
    rng = np.random.default_rng(seed)
    src, dst, n_src, N = _graph(rng)
    E = dst.size
    q = [0.5] if nq == 1 else [0.0, 0.1, 0.5, 0.9, 1.0]
    qt = torch.tensor(q, dtype=torch.float32, device=DEV)
    di = torch.from_numpy(dst).to(DEV, idx_dtype)
    if form == "x":
        x = _values(rng, n_src, F, bf16)
        V = x[src]
        xt = _t(x, bf16).requires_grad_()
        g_ = CSRGraph(torch.from_numpy(src).to(DEV, idx_dtype), di, n_src, N, chunk=CHUNK, idx_dtype=idx_dtype)
        out = Fn.quantile_aggregate(g_, xt, None, qt, interp, 2.5)
        leaf = xt
    else:
        V = _values(rng, E, F, bf16)
        if form == "rows_ptr":                       # destination-sorted messages, grouped by ptr
            order = np.argsort(dst, kind="stable")
            V, dst, src = V[order], dst[order], src[order]
            ptr = torch.from_numpy(np.concatenate([[0], np.cumsum(np.bincount(dst, minlength=N))])).to(DEV, idx_dtype)
            where = (ptr, ops.LongRowPlan(ptr, CHUNK))
        else:                                        # caller order, a CSR over the messages themselves
            e = torch.arange(E, device=DEV, dtype=idx_dtype)
            where = CSRGraph(e, torch.from_numpy(dst).to(DEV, idx_dtype), E, N, chunk=CHUNK, idx_dtype=idx_dtype)
        leaf = _t(V, bf16).requires_grad_()
        out = Fn.quantile_aggregate(where, None, leaf, qt, interp, 2.5)
    want, _ = O.aggregate(V, dst, N, np.array(q, np.float32), interp, 2.5, bf16)
    assert out.dtype == (torch.float32 if O.out_is_f32(bf16, interp) else leaf.dtype)
    _assert_out(_np(out), want)
    g = _g(rng, tuple(out.shape), bf16, interp)
    out.backward(torch.from_numpy(g).to(DEV, out.dtype))
    _, ge = O.aggregate(V, dst, N, np.array(q, np.float32), interp, 2.5, bf16, g)
    if form == "x":
        _assert_grad(_np(leaf.grad), O.sum_out_edges(ge, src, n_src, bf16, CHUNK), interp, bf16, g, positions=False)
    else:
        _assert_grad(_np(leaf.grad), ge, interp, bf16, g)
    return out, leaf.grad


@pytest.mark.parametrize("idx_dtype", [torch.int32, torch.int64], ids=["i32", "i64"])
@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
@pytest.mark.parametrize("nq", [1, 5])
@pytest.mark.parametrize("interp", O.INTERP)
@pytest.mark.parametrize("form", ["x", "rows_ptr", "rows_unsorted"])
def test_matches_the_oracle(form, interp, nq, bf16, idx_dtype):
    _run(form, interp, nq, bf16, idx_dtype, F=37 if nq == 1 else 8)


@pytest.mark.parametrize("F", [1, 4, 32, 33, 64, 100])
@pytest.mark.parametrize("form", ["x", "rows_unsorted"])
def test_widths(form, F):
    _run(form, "linear", 5, False, torch.int32, F, seed=F)
    _run(form, "nearest", 1, True, torch.int64, F, seed=F + 1)


@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
def test_rows_of_ties(bf16):
    from pytorch_geometric_b200 import functional as Fn
    from pytorch_geometric_b200 import ops
    rng = np.random.default_rng(7)
    lens = np.array([5, 154, 1, 300, 64])
    N, E, F = lens.size, int(lens.sum()), 16
    V = np.ones((E, F), dtype=np.float32) * 3.0
    V[:, 1::2] = O.rnd(rng.integers(0, 3, (E, F // 2)) * 0.1, bf16)          # heavy ties after rounding
    V[::7, 2] = -0.0
    V[::11, 2] = 0.0
    dst = np.repeat(np.arange(N), lens)
    ptr = torch.from_numpy(np.concatenate([[0], np.cumsum(lens)])).to(DEV)
    for interp in O.INTERP:
        a = _t(V, bf16).requires_grad_()
        out = Fn.quantile_aggregate((ptr, ops.LongRowPlan(ptr, CHUNK)), None, a, [0.1, 0.5, 0.77], interp)
        want, _ = O.aggregate(V, dst, N, np.array([0.1, 0.5, 0.77], np.float32), interp, 0.0, bf16)
        _assert_out(_np(out), want)
        g = _g(rng, tuple(out.shape), bf16, interp)
        out.backward(torch.from_numpy(g).to(DEV, out.dtype))
        _, ge = O.aggregate(V, dst, N, np.array([0.1, 0.5, 0.77], np.float32), interp, 0.0, bf16, g)
        _assert_grad(_np(a.grad), ge, interp, bf16, g)


def test_second_run_gives_identical_bits():
    for form in ("x", "rows_ptr"):
        o1, g1 = _run(form, "linear", 5, False, torch.int32, 48, seed=3)
        o2, g2 = _run(form, "linear", 5, False, torch.int32, 48, seed=3)
        assert torch.equal(o1.view(torch.int32), o2.view(torch.int32))
        assert torch.equal(g1.view(torch.int32), g2.view(torch.int32))


def test_no_device_to_host_sync_after_warm_up():
    from pytorch_geometric_b200 import functional as Fn
    from pytorch_geometric_b200 import ops
    rng = np.random.default_rng(5)
    lens = rng.integers(0, 90, 500)
    ptr = torch.from_numpy(np.concatenate([[0], np.cumsum(lens)])).to(DEV)
    plan = ops.LongRowPlan(ptr, CHUNK)
    a = torch.randn(int(lens.sum()), 32, device=DEV, requires_grad=True)
    q = torch.tensor([[0.25], [0.5]], device=DEV)

    def step():
        out = Fn.quantile_aggregate((ptr, plan), None, a, q, "midpoint")
        out.backward(torch.ones_like(out))
    step()
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        step()
    finally:
        torch.cuda.set_sync_debug_mode(0)
    torch.cuda.synchronize()


def test_ranks_past_2_24_stay_inside_their_group():
    from pytorch_geometric_b200 import functional as Fn
    from pytorch_geometric_b200 import ops
    n0, k, F = (1 << 24) + 1, 200, 4
    g0 = torch.randperm(n0, device=DEV).float()                          # {0, ..., 2^24}: median 2^23
    small = (torch.arange(3 * k, device=DEV) // 3 * 3).float() + torch.stack(
        [torch.randperm(3, device=DEV) for _ in range(k)]).view(-1).float()
    a = torch.cat([g0, small]).view(-1, 1).expand(-1, F).contiguous()
    ptr = torch.cat([torch.tensor([0, n0], device=DEV), n0 + 3 * torch.arange(1, k + 1, device=DEV)])
    out = Fn.quantile_aggregate((ptr, ops.LongRowPlan(ptr, 4096)), None, a, 0.5, "lower")
    assert torch.equal(out[0], torch.full((F, ), float(1 << 23), device=DEV))
    want = (3 * torch.arange(k, device=DEV) + 1).float().view(-1, 1).expand(-1, F)
    assert torch.equal(out[1:], want)


@pytest.mark.parametrize("chunk", [4096, None], ids=["hub_kernel", "row_kernel"])
def test_q1_past_2_24_picks_the_groups_last_element(chunk):
    # count - 1 = 2^24 + 3 rounds up to 2^24 + 4 in fp32, so q = 1 gives h = count: the rank is clamped to count - 1.
    # One zero-filled group with a unique maximum of 1.0 per channel: q = 1 picks the maximum and q = 0 slot 0 (the
    # first of the tied zeros), for every interpolation (frac is 0 at both q).  Without a plan one lane walks the whole
    # row, so that case takes q = 1 alone, where the first digit already isolates the maximum.
    from pytorch_geometric_b200 import functional as Fn
    from pytorch_geometric_b200 import ops
    n0, hot = (1 << 24) + 4, (12345, (1 << 24) - 3)
    ptr = torch.tensor([0, n0], device=DEV)
    plan = ops.LongRowPlan(ptr, chunk) if chunk else None
    assert chunk is None or plan.n_long == 1
    qs = [0.0, 1.0] if chunk else [1.0]
    want_out = torch.tensor([[0.0, 0.0, 1.0, 1.0]] if chunk else [[1.0, 1.0]], device=DEV)
    g = torch.tensor([[1.0, 2.0, 3.0, 4.0]] if chunk else [[3.0, 4.0]], device=DEV)
    want_grad = torch.zeros(n0, 2, device=DEV)
    if chunk:
        want_grad[0] = torch.tensor([1.0, 2.0], device=DEV)
    want_grad[hot[0], 0], want_grad[hot[1], 1] = 3.0, 4.0
    for interp in O.INTERP if chunk else ("linear", "higher"):
        a = torch.zeros(n0, 2, device=DEV)
        a[hot[0], 0] = a[hot[1], 1] = 1.0
        a.requires_grad_()
        out = Fn.quantile_aggregate((ptr, plan), None, a, qs, interp)
        assert torch.equal(out, want_out), (interp, out)
        out.backward(g)
        assert torch.equal(a.grad, want_grad), interp
        del a, out
    torch.cuda.synchronize()


@pytest.mark.parametrize("name", sorted(O.golden_cases(load_golden("quantile"))))
def test_golden_through_the_mirrors(name):
    from pytorch_geometric_b200.nn import MedianAggregation, QuantileAggregation
    c = O.golden_cases(load_golden("quantile"))[name]
    x, d, idx, n, q, interp, fill, bf16, _ = O.case_args(c)
    mod = MedianAggregation(fill) if bool(c["median"]) else QuantileAggregation(q.tolist(), interp, fill)
    mod = mod.to(DEV)
    xt = _t(x, bf16).requires_grad_()
    it = torch.from_numpy(idx).to(DEV)
    out = mod(xt, it, dim_size=n, dim=int(c["dim"]))
    (out.float() * torch.from_numpy(c["w"]).to(DEV)).sum().backward()
    O.check_golden(c, _np(out), _np(xt.grad))


@pytest.mark.parametrize("grouping", ["ptr", "sorted", "unsorted"])
@pytest.mark.parametrize("bf16", [False, True], ids=["fp32", "bf16"])
def test_mirror_groupings(grouping, bf16):
    from pytorch_geometric_b200.nn import QuantileAggregation
    rng = np.random.default_rng(11)
    lens = np.array(LENS + [4, 6])
    N = lens.size
    idx = np.repeat(np.arange(N), lens)
    if grouping == "unsorted":
        idx = idx[rng.permutation(idx.size)]
    V = _values(rng, idx.size, 24, bf16)
    mod = QuantileAggregation([0.2, 0.5, 0.8], "linear", 1.0).to(DEV)
    xt = _t(V, bf16).requires_grad_()
    it = torch.from_numpy(idx).to(DEV)
    kw = dict(dim_size=N)
    if grouping == "ptr":
        kw["ptr"] = torch.from_numpy(np.concatenate([[0], np.cumsum(lens)])).to(DEV)
    if grouping == "sorted":
        kw["index_sorted"] = True
    out = mod(xt, it, **kw)
    q = np.array([0.2, 0.5, 0.8], np.float32)
    want, _ = O.aggregate(V, idx, N, q, "linear", 1.0, bf16)
    _assert_out(_np(out), want)
    g = _g(rng, tuple(out.shape), bf16, "linear")
    out.backward(torch.from_numpy(g).to(DEV))
    _, ge = O.aggregate(V, idx, N, q, "linear", 1.0, bf16, g)
    _assert_grad(_np(xt.grad), ge, "linear", bf16, g)


# ---------------------------------------------------------------- the plug-in against the reference on the CPU
@pytest.fixture
def plugin(tg):
    from pytorch_geometric_b200 import plugin as P
    yield P
    P.uninstall()


def _count_materialise(monkeypatch):
    from pytorch_geometric_b200.plugin import lazy
    calls = []
    orig = lazy.LazyRows.materialise
    monkeypatch.setattr(lazy.LazyRows, "materialise", lambda self: calls.append(1) or orig(self))
    return calls


def _layers(tg):
    from torch_geometric.nn import MessagePassing, SAGEConv
    from torch_geometric.nn.aggr import MultiAggregation

    class QuantileMP(MessagePassing):
        def __init__(self):
            super().__init__(aggr="quantile", aggr_kwargs={"q": [0.2, 0.8]})

        def forward(self, x, edge_index):
            return self.propagate(edge_index, x=x)

    return {"sage_median": lambda: SAGEConv(16, 16, aggr="median"), "mp_quantile": QuantileMP,
            "sage_multi": lambda: SAGEConv(16, 16, aggr=MultiAggregation(["mean", "median"]))}


@pytest.mark.parametrize("layer", ["sage_median", "mp_quantile", "sage_multi"])
def test_plugin_layers_match_the_reference_on_the_cpu(tg, plugin, monkeypatch, layer):
    torch.manual_seed(0)
    rng = np.random.default_rng(2)
    N, E = 300, 3000
    ei = torch.from_numpy(np.stack([rng.integers(0, N, E), (rng.random(E) ** 2 * N).astype(np.int64)]))
    x = torch.randn(N, 16)
    ref = _layers(tg)[layer]()
    xr = x.clone().requires_grad_()
    want = ref(xr, ei)
    gw = torch.randn(want.shape)
    (want * gw).sum().backward()
    plugin.install()
    calls = _count_materialise(monkeypatch)
    mod = _layers(tg)[layer]()
    mod.load_state_dict(ref.state_dict())
    mod = mod.to(DEV)
    xg = x.to(DEV).requires_grad_()
    got = mod(xg, ei.to(DEV))
    (got * gw.to(DEV)).sum().backward()
    if layer != "sage_multi":               # MultiAggregation's 'mean' member goes through FusedAggregation
        assert not calls, "the lazy x_j was materialised"
    terms = want.abs() + 1.0
    assert (got.detach().cpu() - want).abs().max() <= 1e-5 * terms.max() * 16
    gerr = (xg.grad.cpu() - xr.grad).abs().max()
    assert gerr <= 1e-5 * (xr.grad.abs().max() + 1) * 16, gerr


def test_plugin_median_memory_stays_below_half_an_edge_matrix(tg, plugin, monkeypatch):
    from torch_geometric.nn import SAGEConv
    N, E, F = 1_000_000, 16_000_000, 64
    ei = torch.stack([torch.randint(0, N, (E, ), device=DEV), torch.randint(0, N, (E, ), device=DEV)])
    x = torch.randn(N, F, device=DEV, requires_grad=True)
    plugin.install()
    calls = _count_materialise(monkeypatch)
    conv = SAGEConv(F, F, aggr="median").to(DEV)
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    conv(x, ei).sum().backward()
    torch.cuda.synchronize()
    grew = torch.cuda.max_memory_allocated() - base
    assert not calls
    assert grew < E * F * 4 / 2, f"peak grew by {grew / 2**30:.2f} GiB"
