"""GPU tests of PNAConv's fused aggregation (csrc/pna.cu with the multi-aggregation sweep):

  * `Fn.pna_aggregate` against the reference's formula in fp64 -- every aggregator x scaler block and the gradients of
    x, u | v, c and avg_deg_lin / avg_deg_log, with and without c, for widths on and off the vector path, on a graph
    with a chunked hub row, empty and single-edge rows, exact min / max ties and a row whose shifted minimum is 0;
  * one launch per new entry point;
  * the UNMODIFIED reference PNAConv, deep-copied into `B200PNAConv` on the GPU, against the same layer on the CPU;
  * configurations that must fall through to the reference's own forward;
  * the bf16 scaler degree against the reference's DegreeScalerAggregation, bit for bit;
  * the standalone `nn.PNAConv` against the reference's golden vectors (tests/golden/pna.npz).
"""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

from pytorch_geometric_b200 import functional as Fn  # noqa: E402
from pytorch_geometric_b200 import ops  # noqa: E402
from pytorch_geometric_b200.graph import CSRGraph  # noqa: E402

DEV = "cuda"
AGGRS = ("mean", "min", "max", "std", "sum", "var")
SCALERS = ("identity", "amplification", "attenuation", "linear", "inverse_linear")


class _Profile:
    def __enter__(self):
        ops.PROFILE.reset(enabled=True)
        return self

    def __exit__(self, *a):
        self.calls = {k: v["calls"] for k, v in ops.PROFILE.summary().items()}
        ops.PROFILE.reset(enabled=False)
        return False


def _graph_edges(n=700, e=9000, seed=0):
    """A hub row above two 512-edge chunks, a power-law body, empty rows (>= n - 50), single-edge rows."""
    g = torch.Generator().manual_seed(seed)
    dst = (torch.rand(e, generator=g) ** 2 * (n - 60)).long()
    dst[:1300] = 4
    src = torch.randint(0, n, (e, ), generator=g)
    extra_src = torch.arange(10)
    extra_dst = n - 60 + torch.arange(10)                 # ten single-edge rows
    return torch.cat([src, extra_src]), torch.cat([dst, extra_dst]), n


def _reference(x3, uv, c, src, dst, n, aggrs, scalers, lin, log):
    """pna_conv.py:158-169 with scaler.py:75-109 in fp64 on the CPU, message m_e = u[dst] + v[src] (+ c[e])."""
    N, T, F = x3.shape
    W = T * F
    u, v = uv[:, :W], uv[:, W:]
    m = u[dst] + v[src] + (c if c is not None else 0)
    idx = dst.view(-1, 1).expand(-1, W)
    cnt = torch.zeros(n, dtype=m.dtype).index_add_(0, dst, torch.ones_like(dst, dtype=m.dtype))
    s = torch.zeros(n, W, dtype=m.dtype).index_add(0, dst, m)
    mean = s / cnt.clamp(min=1).view(-1, 1)
    mean2 = torch.zeros(n, W, dtype=m.dtype).index_add(0, dst, m * m) / cnt.clamp(min=1).view(-1, 1)
    var = mean2 - mean * mean
    std = var.clamp(min=1e-5).sqrt()
    std = std.masked_fill(std <= 1e-5 ** 0.5, 0.0)
    out = {"sum": s, "mean": mean, "var": var, "std": std,
           "min": torch.zeros(n, W, dtype=m.dtype).scatter_reduce(0, idx, m, "amin", include_self=False),
           "max": torch.zeros(n, W, dtype=m.dtype).scatter_reduce(0, idx, m, "amax", include_self=False)}
    agg = torch.cat([out[a].view(n, T, F) for a in aggrs], dim=-1)
    deg = cnt.view(-1, 1, 1)
    fac = {"identity": torch.ones_like(deg), "amplification": torch.log(deg + 1) / log,
           "attenuation": log / torch.log(deg.clamp(min=1) + 1), "linear": deg / lin,
           "inverse_linear": lin / deg.clamp(min=1)}
    return torch.cat([x3] + [agg * fac[sc] for sc in scalers], dim=-1)


def _close(a, b, tol, what):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    err = (a - b).abs().max().item()
    scale = max(b.abs().max().item(), 1.0)
    assert err <= tol * scale, f"{what}: max err {err:.3e} vs scale {scale:.3e}"


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("width", [(4, 4), (2, 32), (5, 75), (4, 64), (3, 7)])
@pytest.mark.parametrize("with_c", [False, True])
@pytest.mark.parametrize("sorted_csr", [False, True])
def test_pna_aggregate_against_fp64(dtype, width, with_c, sorted_csr):
    T, F = width
    W = T * F
    src, dst, n = _graph_edges()
    if sorted_csr:
        order = torch.argsort(dst, stable=True)
        src, dst = src[order], dst[order]
    g = torch.Generator().manual_seed(T * 100 + F)
    # small integers: sums are exact, min / max ties are frequent
    x3 = torch.randint(-3, 4, (n, T, F), generator=g).double()
    uv = torch.randint(-4, 5, (n, 2 * W), generator=g).double()
    c = torch.randint(-2, 3, (src.numel(), W), generator=g).double() if with_c else None
    # row 0's shifted minimum is exactly 0: u[0] = -min over its in-edges of w
    w = uv[src, W:] + (c if c is not None else 0)
    rows0 = dst == 0
    if rows0.any():
        uv[0, :W] = -w[rows0].min(dim=0).values
    lin = torch.tensor([2.5], dtype=torch.float64)
    log = torch.tensor([1.1], dtype=torch.float64)
    leaves = [t.clone().requires_grad_() for t in (x3, uv, lin, log)] + ([c.clone().requires_grad_()] if with_c else [])
    want = _reference(leaves[0], leaves[1], leaves[4] if with_c else None, src, dst, n, AGGRS, SCALERS, leaves[2], leaves[3])
    gout = torch.randn(want.shape, generator=g, dtype=torch.float64)
    want.backward(gout)

    gpu = [t.detach().to(DEV, dtype if t.numel() > 1 else torch.float32).requires_grad_() for t in leaves]
    ei = torch.stack([src, dst]).to(DEV)
    if sorted_csr:
        rowptr = torch.zeros(n + 1, dtype=torch.long)
        rowptr[1:] = torch.bincount(dst, minlength=n).cumsum(0)
        graph = CSRGraph.from_csr(rowptr.to(DEV), src.to(DEV), n)
    else:
        graph = CSRGraph.from_edge_index(ei, num_nodes=n)
    with _Profile() as p:
        got = Fn.pna_aggregate(graph, gpu[0], gpu[1], gpu[4] if with_c else None, AGGRS, SCALERS, gpu[2], gpu[3])
        got.backward(gout.to(DEV, dtype))
    for name in ("pna_epilogue", "pna_prologue"):
        assert p.calls.get(name) == 1, p.calls
    assert p.calls.get("pna_edge_stats" if with_c else "multi_aggr_csr") == 1, p.calls
    assert p.calls.get("pna_edge_backward" if with_c else "multi_aggr_backward") == 1, p.calls
    tol = 1e-5 if dtype == torch.float32 else 1.6e-2
    _close(got, want, tol, "out")
    names = ["x", "uv", "avg_deg_lin", "avg_deg_log"] + (["c"] if with_c else [])
    for name, lg, lc in zip(names, gpu, leaves):
        if name.startswith("avg"):
            # a sum over every (row, column, aggregator, scaler): the bar is relative to the sum of its |terms|, which
            # |d factor / d avg| = |factor| / avg bounds
            terms = (gout.abs() * want.detach().abs()).sum().item() / lc.item()
            err = (lg.grad.double().cpu() - lc.grad).abs().item()
            assert err <= tol * terms, f"grad {name}: err {err:.3e} vs sum of |terms| {terms:.3e}"
        else:
            _close(lg.grad, lc.grad, tol, f"grad {name}")


def test_var_is_shift_free():
    """|u| >> spread(w): the engine's var comes from the statistics of w, so it is at least as close as the bar."""
    src, dst, n = _graph_edges(seed=3)
    T, F = 2, 16
    W = T * F
    g = torch.Generator().manual_seed(5)
    x3 = torch.randn(n, T, F, generator=g, dtype=torch.float64)
    uv = torch.cat([torch.full((n, W), 1e4, dtype=torch.float64), torch.randn(n, W, generator=g, dtype=torch.float64)], 1)
    lin, log = torch.tensor([2.0], dtype=torch.float64), torch.tensor([1.0], dtype=torch.float64)
    want = _reference(x3, uv, None, src, dst, n, ("var", "std"), ("identity", ), lin, log)
    graph = CSRGraph.from_edge_index(torch.stack([src, dst]).to(DEV), num_nodes=n)
    got = Fn.pna_aggregate(graph, x3.float().to(DEV), uv.float().to(DEV), None, ("var", "std"), ("identity", ),
                           lin.float().to(DEV), log.float().to(DEV))
    _close(got[..., F:], want[..., F:], 1e-5, "var / std")


def _pna_case(tg, case):
    g = torch.Generator().manual_seed(11)
    n, e = 400, 3000
    src = torch.randint(0, n, (e, ), generator=g)
    dst = (torch.rand(e, generator=g) ** 2 * (n - 20)).long()
    dst[:900] = 2
    ei = torch.stack([src, dst])
    deg = torch.bincount(torch.bincount(dst, minlength=n))
    kw = dict(aggregators=list(AGGRS), scalers=list(SCALERS), deg=deg, edge_dim=3, towers=4)
    fin, fout = 16, 32
    if case == "examples_pna":
        fin = fout = 75
        kw = dict(aggregators=["mean", "min", "max", "std"], scalers=["identity", "amplification", "attenuation"],
                  deg=deg, edge_dim=50, towers=5, post_layers=1, divide_input=False)
    elif case == "divide_input":
        kw["divide_input"] = True
    elif case == "no_edge_dim":
        kw["edge_dim"] = None
    elif case == "train_norm":
        kw["train_norm"] = True
    elif case == "target_to_source":
        kw["flow"] = "target_to_source"
    elif case == "edge_index_sorted":
        ei, _ = tg.EdgeIndex(ei, sparse_size=(n, n)).sort_by("col")
    x = torch.randn(n, fin, generator=g)
    ea = torch.randn(e, kw["edge_dim"], generator=g) if kw.get("edge_dim") else None
    return ei, x, ea, fin, fout, kw


@pytest.mark.parametrize("case", ["reference_test", "divide_input", "examples_pna", "no_edge_dim", "train_norm",
                                  "target_to_source", "edge_index_sorted"])
def test_unmodified_reference_pna_on_the_fused_path(tg, case):
    from pytorch_geometric_b200.plugin import conv as PC
    ei, x, ea, fin, fout, kw = _pna_case(tg, case)
    torch.manual_seed(3)
    ref = tg.nn.PNAConv(fin, fout, **kw)
    gpu = copy.deepcopy(ref).to(DEV)
    gpu.__class__ = PC.B200PNAConv
    xc = x.clone().requires_grad_()
    xg = x.to(DEV).requires_grad_()
    eac = None if ea is None else ea.clone().requires_grad_()
    eag = None if ea is None else ea.to(DEV).requires_grad_()
    want = ref(xc, ei, eac)
    gout = torch.randn_like(want)
    want.backward(gout)
    with _Profile() as p:
        got = gpu(xg, ei.to(DEV), eag)
        got.backward(gout.to(DEV))
    assert p.calls.get("pna_epilogue") == 1 and p.calls.get("pna_prologue") == 1, p.calls
    _close(got, want, 1e-4, f"{case} out")
    _close(xg.grad, xc.grad, 3e-4, f"{case} grad x")
    if ea is not None:
        _close(eag.grad, eac.grad, 3e-4, f"{case} grad edge_attr")
    for (nm, pg), (_, pc) in zip(gpu.named_parameters(), ref.named_parameters()):
        _close(pg.grad, pc.grad, 2e-4, f"{case} grad {nm}")


@pytest.mark.parametrize("kind", ["pre_layers", "hook", "explain"])
def test_configurations_that_fall_through(tg, kind):
    from pytorch_geometric_b200.plugin import conv as PC
    ei, x, ea, fin, fout, kw = _pna_case(tg, "reference_test")
    if kind == "pre_layers":
        kw["pre_layers"] = 2
    torch.manual_seed(3)
    ref = tg.nn.PNAConv(fin, fout, **kw).to(DEV)
    gpu = copy.deepcopy(ref)
    gpu.__class__ = PC.B200PNAConv
    if kind == "hook":
        for m in (ref, gpu):
            m.register_message_forward_hook(lambda mod, inp, out: out)
    if kind == "explain":
        for m in (ref, gpu):
            m.explain = True
            m._edge_mask = torch.ones(ei.size(1), device=DEV)
            m._apply_sigmoid = False
    with _Profile() as p:
        got = gpu(x.to(DEV), ei.to(DEV), ea.to(DEV))
    want = ref(x.to(DEV), ei.to(DEV), ea.to(DEV))
    assert "pna_epilogue" not in p.calls
    # the reference's CUDA scatters use atomics, so two runs of its own forward agree to rounding, not to the bit
    _close(got, want, 1e-5, f"{kind} out")


def test_memory_of_the_op():
    """fwd + bwd growth, beside the [N, T, (1 + A S) F] output itself, below one [E, 2W] tensor without c and below
    [E, 3W] with it (N = 400k, E = 4M)."""
    n, e, T, F = 400_000, 4_000_000, 4, 16
    W = T * F
    g = torch.Generator(device=DEV).manual_seed(0)
    src = torch.randint(0, n, (e, ), device=DEV, generator=g)
    dst = torch.randint(0, n, (e, ), device=DEV, generator=g)
    graph = CSRGraph.from_edge_index(torch.stack([src, dst]), num_nodes=n)
    graph.build_transpose()
    _ = graph.t2csr
    lin = torch.tensor([3.0], device=DEV)
    log = torch.tensor([1.2], device=DEV)
    for with_c in (False, True):
        x3 = torch.randn(n, T, F, device=DEV, requires_grad=True)
        uv = torch.randn(n, 2 * W, device=DEV, requires_grad=True)
        c = torch.randn(e, W, device=DEV, requires_grad=True) if with_c else None
        gout = torch.randn(n, T, (1 + 4 * 3) * F, device=DEV)
        torch.cuda.synchronize()
        base = torch.cuda.memory_allocated()
        torch.cuda.reset_peak_memory_stats()
        out = Fn.pna_aggregate(graph, x3, uv, c, ("mean", "min", "max", "std"), ("identity", "amplification", "attenuation"),
                               lin, log)
        out.backward(gout)
        torch.cuda.synchronize()
        growth = torch.cuda.max_memory_allocated() - base - out.numel() * out.element_size()
        bound = e * (3 if with_c else 2) * W * 4
        assert growth < bound, f"with_c={with_c}: {growth / 1e9:.2f} GB >= {bound / 1e9:.2f} GB"
        del out, x3, uv, c


def test_bf16_degree_rounds_like_the_reference(tg):
    """deg in bf16 is the exact count rounded once, as the reference's degree(..., dtype=bfloat16) gives it on the CPU
    (257 -> 256, 1001 -> 1000, 1300 -> 1296): the identity and linear blocks of a sum over ones equal, bit for bit,
    the reference's DegreeScalerAggregation on the same messages."""
    counts = [1300, 257, 1001, 3, 0, 1]
    dst = torch.repeat_interleave(torch.arange(len(counts)), torch.tensor(counts))
    n, e, F = len(counts), dst.numel(), 8
    src = torch.arange(e) % n
    ref = tg.nn.aggr.DegreeScalerAggregation(["sum"], ["identity", "linear", "amplification"],
                                             torch.bincount(torch.tensor(counts))).to(torch.bfloat16)
    with torch.no_grad():
        ref.avg_deg_lin.fill_(1.0)
        ref.avg_deg_log.fill_(1.0)
    want = ref(torch.ones(e, F, dtype=torch.bfloat16), dst, dim_size=n)
    graph = CSRGraph.from_edge_index(torch.stack([src, dst]).to(DEV), num_nodes=n)
    uv = torch.cat([torch.zeros(n, F), torch.ones(n, F)], 1).to(DEV, torch.bfloat16)
    got = Fn.pna_aggregate(graph, torch.zeros(n, 1, F, device=DEV, dtype=torch.bfloat16), uv, None, ("sum", ),
                           ("identity", "linear", "amplification"), ref.avg_deg_lin.float().to(DEV),
                           ref.avg_deg_log.float().to(DEV))
    assert torch.equal(got[:, 0, F:3 * F].cpu(), want[:, :2 * F])
    _close(got[:, 0, 3 * F:], want[:, 2 * F:], 1e-2, "amplification")


# ------------------------------------------------------------------------------------------------ the standalone mirror
_GOLDEN_CASES = [("all", 16, 32, dict(aggregators=["mean", "min", "max", "std", "sum", "var"],
                                      scalers=["identity", "amplification", "attenuation", "linear", "inverse_linear"],
                                      towers=4, edge_dim=3)),
                 ("divide", 16, 32, dict(aggregators=["sum", "max", "var"], scalers=["identity", "linear"], towers=2,
                                         divide_input=True, post_layers=2)),
                 ("train_norm", 12, 8, dict(aggregators=["mean", "min", "max", "std"],
                                            scalers=["identity", "amplification", "attenuation"], edge_dim=5,
                                            train_norm=True))]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("tag,ic,oc,kw", _GOLDEN_CASES)
def test_standalone_pna_matches_golden(golden, tag, ic, oc, kw, dtype):
    """fp32: the output, grad x, grad edge_attr and every parameter gradient of the reference's golden run.  bf16: the
    output, and the dtype of every gradient."""
    from pytorch_geometric_b200.nn import PNAConv
    z = golden("pna")
    conv = PNAConv(ic, oc, deg=torch.from_numpy(z[f"{tag}_deg"]), **kw)
    conv.load_state_dict({k[len(tag) + 3:]: torch.from_numpy(v) for k, v in z.items() if k.startswith(f"{tag}_p_")})
    conv = conv.to(DEV).to(dtype)
    t = lambda k: torch.from_numpy(z[f"{tag}_{k}"]).to(DEV).to(dtype)      # noqa: E731
    x = t("x").requires_grad_()
    ea = t("ea").requires_grad_() if f"{tag}_ea" in z else None
    with _Profile() as p:
        out = conv(x, torch.from_numpy(z[f"{tag}_ei"]).to(DEV), ea)
        out.backward(t("gout"))
    assert p.calls.get("pna_epilogue") == 1 and p.calls.get("pna_prologue") == 1, p.calls
    got = {"out": out, "gx": x.grad}
    if ea is not None:
        got["gea"] = ea.grad
    got.update({f"g_{n}": q.grad for n, q in conv.named_parameters() if f"{tag}_g_{n}" in z})
    assert len(got) == sum(1 for k in z if k.startswith(f"{tag}_g_")) + (3 if ea is not None else 2)
    if dtype == torch.float32:
        for k, v in got.items():
            _close(v, torch.from_numpy(z[f"{tag}_{k}"]), 1e-4 if k.startswith("g_") else 2e-5, f"{tag} {k}")
    else:
        _close(out, torch.from_numpy(z[f"{tag}_out"]), 6e-2, f"{tag} out vs golden")
        assert all(v.dtype == torch.bfloat16 for v in got.values())
