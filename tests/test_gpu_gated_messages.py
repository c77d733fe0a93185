"""GPU tests of the gated message sigmoid(k_i + q_j) * v_j (ResGatedGraphConv, res_gated_graph_conv.py:13-148) fused
into the CSR sweep:

  * `Fn.aggregate_gated` / `aggregate_gated_qv` against an fp64 formula -- sum / mean, fp32 / bf16, widths on the
    vector and the scalar path, q and v as two tensors or the halves of one [N, 2F] tensor, a bipartite power-law
    graph with destination hubs and a source out-hub (both chunked), adopted and sorted CSRs;
  * the sigmoid's edge cases (s in {0, +-20, +-30, +-inf, NaN}, v = +-inf where the gate is 0) and the memory of
    forward and backward;
  * the UNMODIFIED reference ResGatedGraphConv (`tg` fixture) under `plugin.install()` against the same layer on the
    CPU, and messages that must not fuse;
  * the standalone `nn.ResGatedGraphConv` against the reference's golden vectors (tests/golden/res_gated.npz).
"""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

from pytorch_geometric_b200 import functional as Fn  # noqa: E402
from pytorch_geometric_b200 import ops  # noqa: E402
from pytorch_geometric_b200.graph import CSRGraph  # noqa: E402

DEV = "cuda"
KERNELS = ("gated_csr", "gated_backward_dst", "gated_backward_src")


class _Profile:
    def __enter__(self):
        ops.PROFILE.reset(enabled=True)
        return self

    def __exit__(self, *a):
        self.calls = {k: v["calls"] for k, v in ops.PROFILE.summary().items()}
        ops.PROFILE.reset(enabled=False)
        return False


def _close(a, b, tol=2e-5, what=""):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    err = (a - b).abs().max().item()
    assert err <= tol * max(b.abs().max().item(), 1e-3), f"{what}: max err {err:.3e} vs scale {b.abs().max().item():.3e}"


def _power_law_edges(n_src=3000, n_dst=2500, e=60000, seed=0):
    """Destinations: two hubs far above the 512-edge chunk, a power-law body, a tail of empty rows; sources: one
    out-hub (chunked in the transposed sweep) and a tail without out-edges; a block of duplicated edges."""
    g = torch.Generator().manual_seed(seed)
    dst = (torch.rand(e, generator=g) ** 3 * (n_dst - 200)).long()           # rows >= n_dst - 200 stay empty
    dst[:3000] = 0
    dst[3000:4500] = 7
    src = torch.randint(0, n_src - 100, (e, ), generator=g)                  # sources >= n_src - 100 send nothing
    src[5000:7000] = 11
    src[8000:8100], dst[8000:8100] = src[8100:8200], dst[8100:8200]         # duplicate edges
    return src, dst, n_src, n_dst


def _check(a, b, s, tol, what):
    """|a - b| <= tol * s elementwise (s = sum of |terms|), NaN exactly where the formula has NaN, equal infinities."""
    a, b, s = a.detach().double().cpu(), b.double().cpu(), s.double().cpu()
    assert torch.equal(a.isnan(), b.isnan()), f"{what}: NaN pattern differs"
    fin = b.isfinite()
    assert torch.equal(a[~fin & ~b.isnan()], b[~fin & ~b.isnan()]), f"{what}: infinities differ"
    bad = ((a - b).abs() > tol * s + 1e-30) & fin
    assert not bad.any(), f"{what}: {int(bad.sum())} entries off, first at {bad.nonzero()[:3].tolist()}"


def _sig(s):
    """fp64 sigmoid and its derivative from t = exp(-|s|) (accurate at large |s|)."""
    t = torch.exp(-s.abs())
    r = 1.0 / (1.0 + t)
    return torch.where(s >= 0, r, t * r), t * r * r


def _formula(k, q, v, src, dst, n_src, n_dst, reduce, gout):
    """fp64 out, grad_k, grad_q, grad_v, each with its sum of |terms| (pre-activation rounded to the storage dtype)."""
    s = (k[dst] + q[src]).double()                                           # the add in the storage dtype
    sig, dsig = _sig(s)
    vj = v[src].double()
    deg = torch.bincount(dst, minlength=n_dst).clamp(min=1).double().view(-1, 1)
    g = gout.double()
    F = k.size(1)

    def red(n, idx, t):
        z = torch.zeros(n, F, dtype=torch.float64, device=k.device)
        return z.clone().index_add_(0, idx, t), z.index_add_(0, idx, t.abs())
    out, s_out = red(n_dst, dst, sig * vj)
    if reduce == "mean":
        out, s_out, g = out / deg, s_out / deg, g / deg
    gk, s_gk = red(n_dst, dst, g[dst] * vj * dsig)
    gv, s_gv = red(n_src, src, sig * g[dst])
    gq, s_gq = red(n_src, src, vj * dsig * g[dst])
    return (out, s_out), (gk, s_gk), (gq, s_gq), (gv, s_gv)


def _graph(src, dst, n_src, n_dst, adopted):
    src, dst = src.to(DEV), dst.to(DEV)
    if not adopted:
        return CSRGraph(src, dst, n_src, n_dst), src, dst
    order = torch.sort(dst, stable=True).indices
    src, dst = src[order], dst[order]
    rowptr = torch.zeros(n_dst + 1, dtype=torch.int64, device=DEV)
    rowptr[1:] = torch.bincount(dst, minlength=n_dst).cumsum(0)
    g = CSRGraph.from_csr(rowptr, src, n_src)
    assert g.perm is None
    return g, src, dst


def _run(graph, k, q, v, reduce, gout, layout):
    """out, grad_k, grad_q, grad_v of the op, with q / v as two tensors or the halves of one [N, 2F] leaf."""
    F = k.size(1)
    k = k.clone().requires_grad_()
    if layout == "halves":
        qv = torch.cat([q, v], 1).requires_grad_()
        out = Fn.aggregate_gated_qv(graph, k, qv, reduce)
        out.backward(gout)
        return out, k.grad, qv.grad[:, :F], qv.grad[:, F:]
    q, v = q.clone().requires_grad_(), v.clone().requires_grad_()
    out = Fn.aggregate_gated(graph, k, q, v, reduce)
    out.backward(gout)
    return out, k.grad, q.grad, v.grad


@pytest.mark.parametrize("layout", ["separate", "halves"])
@pytest.mark.parametrize("adopted", [False, True])
@pytest.mark.parametrize("feat", [6, 16, 64, 128, 256, 300])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("reduce", ["sum", "mean"])
def test_op_matches_fp64_formula(reduce, dtype, feat, adopted, layout):
    src, dst, n_src, n_dst = _power_law_edges()
    graph, src, dst = _graph(src, dst, n_src, n_dst, adopted)
    gen = torch.Generator(device=DEV).manual_seed(feat)
    k = (2 * torch.randn(n_dst, feat, device=DEV, generator=gen)).to(dtype)
    q = (2 * torch.randn(n_src, feat, device=DEV, generator=gen)).to(dtype)
    v = torch.randn(n_src, feat, device=DEV, generator=gen).to(dtype)
    gout = torch.randn(n_dst, feat, device=DEV, generator=gen).to(dtype)
    with _Profile() as p:
        got = _run(graph, k, q, v, reduce, gout, layout)
    assert all(p.calls.get(name, 0) == 1 for name in KERNELS), p.calls
    assert graph.plan.n_long >= 2 and graph.plan_t.n_long >= 1
    assert all(t.dtype == dtype for t in got)
    tol = 1e-5 if dtype == torch.float32 else 1.6e-2
    want = _formula(k, q, v, src, dst, n_src, n_dst, reduce, gout)
    for name, t, (ref, s) in zip(("out", "grad_k", "grad_q", "grad_v"), got, want):
        _check(t, ref, s, tol, name)
    assert (got[0][n_dst - 200:] == 0).all() and (got[1][n_dst - 200:] == 0).all()      # empty rows
    assert (got[2][n_src - 100:] == 0).all() and (got[3][n_src - 100:] == 0).all()      # sources without out-edges


def test_inference_trailing_shapes_and_empty_graph():
    src, dst, n_src, n_dst = _power_law_edges(seed=1)
    graph, src, dst = _graph(src, dst, n_src, n_dst, False)
    k = torch.randn(n_dst, 64, device=DEV)
    q, v = torch.randn(n_src, 64, device=DEV), torch.randn(n_src, 64, device=DEV)
    with torch.no_grad(), _Profile() as p:
        o1 = Fn.aggregate_gated(graph, k, q, v)
    assert p.calls == {"gated_csr": 1}, p.calls
    o2 = Fn.aggregate_gated(graph, k.view(n_dst, 4, 16), q.view(n_src, 4, 16), v.view(n_src, 4, 16))
    assert o2.shape == (n_dst, 4, 16) and torch.equal(o2.view(n_dst, 64), o1)
    # only k needs a gradient: the source sweep does not run
    kr = k.clone().requires_grad_()
    with _Profile() as p:
        Fn.aggregate_gated(graph, kr, q, v).sum().backward()
    assert "gated_backward_src" not in p.calls and p.calls.get("gated_backward_dst") == 1, p.calls
    empty = CSRGraph(torch.zeros(0, dtype=torch.long, device=DEV), torch.zeros(0, dtype=torch.long, device=DEV), 5, 4)
    ke = torch.full((4, 32), float("inf"), device=DEV, requires_grad=True)
    qe = torch.randn(5, 32, device=DEV, requires_grad=True)
    ve = torch.full((5, 32), float("nan"), device=DEV, requires_grad=True)
    oe = Fn.aggregate_gated(empty, ke, qe, ve, "mean")
    oe.backward(torch.full_like(oe, float("inf")))
    assert (oe == 0).all() and (ke.grad == 0).all() and (qe.grad == 0).all() and (ve.grad == 0).all()
    with pytest.raises(ValueError, match="sum or mean"):
        Fn.aggregate_gated(graph, k, q, v, "max")
    with pytest.raises(TypeError, match="share a dtype"):
        Fn.aggregate_gated(graph, k, q.bfloat16(), v)
    with pytest.raises(ValueError, match="destination nodes"):
        Fn.aggregate_gated(graph, q, q, v)


@pytest.mark.parametrize("feat", [64, 13])
def test_sigmoid_edge_cases(feat):
    """s = k_i + q_j over {0, +-20, +-30, +-inf, NaN}, and v = +-inf on edges whose gate is 0 (0 * inf = NaN, as the
    reference computes it); every output against the fp64 formula, NaN pattern included."""
    vals = [0.0, 20.0, -20.0, 30.0, -30.0, float("inf"), float("-inf"), float("nan"), float("-inf"), float("-inf")]
    n = len(vals)
    src = torch.tensor(list(range(n)) + [1, 2, 3, 4], device=DEV)
    dst = torch.tensor(list(range(n)) + [0, 0, 9, 9], device=DEV)
    graph = CSRGraph(src, dst, n, n)
    k = torch.zeros(n, feat, device=DEV)
    k[9] = 0.5
    q = torch.tensor(vals, device=DEV).view(-1, 1).repeat(1, feat)
    v = torch.randn(n, feat, device=DEV)
    v[8], v[9] = float("inf"), float("-inf")                 # their gates are sigmoid(-inf) = 0
    gout = torch.randn(n, feat, device=DEV)
    for reduce in ("sum", "mean"):
        got = _run(graph, k, q, v, reduce, gout, "separate")
        want = _formula(k, q, v, src, dst, n, n, reduce, gout)
        for name, t, (ref, s) in zip(("out", "grad_k", "grad_q", "grad_v"), got, want):
            _check(t, ref, s, 1e-5, f"{reduce} {name}")
        o = got[0]
        assert torch.equal(o[5], v[5] if reduce == "sum" else v[5]) and (o[6] == 0).all()   # s = +inf / -inf
        assert o[7].isnan().all() and o[8].isnan().all() and (got[3][8] == 0).all()          # NaN; 0 * inf


def test_memory_of_forward_and_backward():
    """N = 400k, E = 4M, F = 128 fp32: neither the forward nor the backward grows the peak by one [E, F] tensor."""
    n, e, f = 400_000, 4_000_000, 128
    g = torch.Generator(device=DEV).manual_seed(0)
    src = torch.randint(0, n, (e, ), device=DEV, generator=g)
    dst = (torch.rand(e, device=DEV, generator=g) ** 2 * (n - 1)).long()
    graph = CSRGraph(src, dst, n, n)
    del src, dst
    k, q, v = (torch.randn(n, f, device=DEV, generator=g).requires_grad_() for _ in range(3))
    gout = torch.randn(n, f, device=DEV, generator=g)
    one_ef = e * f * 4
    Fn.aggregate_gated(graph, k, q, v, "mean").backward(gout)   # warm: transpose, plans' partials
    k.grad = q.grad = v.grad = None
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    m0 = torch.cuda.memory_allocated()
    out = Fn.aggregate_gated(graph, k, q, v, "mean")
    torch.cuda.synchronize()
    fwd = torch.cuda.max_memory_allocated() - m0
    torch.cuda.reset_peak_memory_stats()
    m1 = torch.cuda.memory_allocated()
    out.backward(gout)
    torch.cuda.synchronize()
    bwd = torch.cuda.max_memory_allocated() - m1
    assert fwd < one_ef and bwd < one_ef, (fwd, bwd, one_ef)


# ------------------------------------------------------------------------------------------------ the reference layer
@pytest.fixture
def plugin(tg):
    from pytorch_geometric_b200 import plugin as P
    yield P
    P.uninstall()


def _no_materialise(monkeypatch):
    from pytorch_geometric_b200.plugin.lazy import GatedRows, LazyRows
    seen = []
    for cls in (LazyRows, GatedRows):
        orig = cls.materialise
        monkeypatch.setattr(cls, "materialise", lambda self, orig=orig: seen.append(1) or orig(self))
    return seen


def _ref_case(tg, case, n_src=400, n_dst=400, e=5000, seed=3):
    g = torch.Generator().manual_seed(seed)
    bip = case == "bipartite"
    if bip:
        n_dst = 250
    src = torch.randint(0, n_src, (e, ), generator=g)
    dst = (torch.rand(e, generator=g) ** 2 * (n_dst - 1)).long()
    dst[:700] = 3                                                       # a hub row above the 512-edge chunk
    src[700:1400] = 5                                                   # a source out-hub
    ei = torch.stack([src, dst])
    if case == "edge_index_sorted":
        ei, _ = tg.EdgeIndex(ei, sparse_size=(n_src, n_dst)).sort_by("col")
    x = torch.randn(n_src, 32, generator=g)
    x_dst = torch.randn(n_dst, 24, generator=g) if bip else None
    kw = {"mean": {"aggr": "mean"}, "bipartite": {"aggr": "mean"}, "no_root_no_bias": {"root_weight": False, "bias": False},
          "target_to_source": {"flow": "target_to_source"}}.get(case, {})
    return ei, x, x_dst, kw


@pytest.mark.parametrize("case", ["plain", "bipartite", "mean", "no_root_no_bias", "edge_index_sorted", "sparse_csc",
                                  "target_to_source"])
def test_unmodified_reference_res_gated_reaches_the_fused_kernels(tg, plugin, monkeypatch, case):
    ei, x, x_dst, kw = _ref_case(tg, case)
    plugin.install()
    seen = _no_materialise(monkeypatch)
    torch.manual_seed(7)
    ic = (32, 24) if x_dst is not None else 32
    ref = tg.nn.ResGatedGraphConv(ic, 16, **kw)
    if ref.bias is not None:
        with torch.no_grad():
            ref.bias.normal_()
    gpu = copy.deepcopy(ref).to(DEV)
    assert type(gpu).__module__.startswith("torch_geometric.")
    leaves_c = [t.clone().requires_grad_() for t in (x, ) + ((x_dst, ) if x_dst is not None else ())]
    leaves_g = [t.detach().clone().to(DEV).requires_grad_() for t in leaves_c]
    n_dst = x_dst.size(0) if x_dst is not None else x.size(0)

    def adj(dev):
        if case == "sparse_csc":       # the reference's own test: to_torch_csc_tensor(edge_index).t()
            return tg.utils.to_torch_csc_tensor(ei.to(dev), size=(x.size(0), n_dst)).t()
        return ei.to(dev)

    def run(mod, leaves, dev):
        xin = (leaves[0], leaves[1]) if x_dst is not None else leaves[0]
        return mod(xin, adj(dev))
    want = run(ref, leaves_c, "cpu")
    gout = torch.randn_like(want)
    want.backward(gout)
    assert not seen                                                      # the CPU run falls through untouched
    with _Profile() as p:
        got = run(gpu, leaves_g, DEV)
        got.backward(gout.to(DEV))
    assert all(p.calls.get(name, 0) == 1 for name in KERNELS), p.calls
    assert not seen, "the message was materialised"
    _close(got, want, what=f"{case} out")
    for i, (lg, lc) in enumerate(zip(leaves_g, leaves_c)):
        _close(lg.grad, lc.grad, tol=5e-5, what=f"{case} grad of input {i}")
    for (n, pg), (_, pc) in zip(gpu.named_parameters(), ref.named_parameters()):
        _close(pg.grad, pc.grad, tol=1e-4, what=f"{case} grad {n}")


def _v_i_layer(tg):
    class GateVi(tg.nn.MessagePassing):
        """sigmoid(k_i + q_j) * v_i: the gated value is the destination's, which the fused sweep does not compute."""

        def __init__(self):
            super().__init__(aggr="add")

        def forward(self, k, q, v, edge_index):
            return self.propagate(edge_index, k=k, q=q, v=v)

        def message(self, k_i, q_j, v_i):
            return torch.sigmoid(k_i + q_j) * v_i
    return GateVi()


@pytest.mark.parametrize("kind", ["edge_dim", "tanh", "v_i", "max", "mixed_dtype"])
def test_messages_that_must_not_fuse_match_the_reference(tg, plugin, kind):
    g = torch.Generator().manual_seed(9)
    n, e, f = 200, 3000, 16
    ei = torch.stack([torch.randint(0, n, (e, ), generator=g), torch.randint(0, n, (e, ), generator=g)])
    x = torch.randn(n, f, generator=g)
    ea = torch.randn(e, 4, generator=g)
    plugin.install()
    torch.manual_seed(1)
    if kind == "v_i":
        ref = _v_i_layer(tg)
        kqv = [torch.randn(n, f, generator=g) for _ in range(3)]
        call = lambda m, dev, leaves: m(*leaves, ei.to(dev))                                        # noqa: E731
        leaves_c = [t.clone().requires_grad_() for t in kqv]
    else:
        kw = {"edge_dim": {"edge_dim": 4}, "tanh": {"act": torch.nn.Tanh()}, "max": {"aggr": "max"}}.get(kind, {})
        ref = tg.nn.ResGatedGraphConv(f, f, **kw)
        if kind == "edge_dim":
            call = lambda m, dev, leaves: m(leaves[0], ei.to(dev), ea.to(dev))                      # noqa: E731
        else:
            call = lambda m, dev, leaves: m(leaves[0], ei.to(dev))                                  # noqa: E731
        leaves_c = [x.clone().requires_grad_()]
    gpu = copy.deepcopy(ref).to(DEV)
    if kind == "mixed_dtype":          # bf16 q / v gathered next to an fp32 k: promoted as in the reference
        gpu.lin_query.bfloat16()
        gpu.lin_value.bfloat16()
        ref.lin_query.bfloat16()
        ref.lin_value.bfloat16()
        call = lambda m, dev, leaves: m((leaves[0].bfloat16(), leaves[0]), ei.to(dev))              # noqa: E731
    leaves_g = [t.detach().clone().to(DEV).requires_grad_() for t in leaves_c]
    want = call(ref, "cpu", leaves_c)
    with _Profile() as p:
        got = call(gpu, DEV, leaves_g)
    assert p.calls.get("gated_csr", 0) == 0, p.calls
    assert got.dtype == want.dtype, (got.dtype, want.dtype)
    tol = 1e-5 if kind != "mixed_dtype" else 2e-2
    _close(got, want, tol=tol, what=kind)
    gout = torch.randn_like(want)
    want.backward(gout)
    got.backward(gout.to(DEV))
    for lg, lc in zip(leaves_g, leaves_c):
        _close(lg.grad, lc.grad, tol=1e-4 if kind != "mixed_dtype" else 3e-2, what=kind + " grad")


# ------------------------------------------------------------------------------------------------ the standalone mirror
_GOLDEN_CASES = [("plain", 16, 32, {}), ("mean_bip", (16, 24), 32, {"aggr": "mean", "root_weight": False}),
                 ("narrow", 16, 6, {"bias": False})]


def _run_mirror(z, tag, ic, oc, kw, dtype):
    from pytorch_geometric_b200.nn import ResGatedGraphConv
    conv = ResGatedGraphConv(ic, oc, **kw)
    conv.load_state_dict({k[len(tag) + 3:]: torch.from_numpy(v) for k, v in z.items() if k.startswith(f"{tag}_p_")})
    conv = conv.to(DEV).to(dtype)
    t = lambda k: torch.from_numpy(z[f"{tag}_{k}"]).to(DEV).to(dtype)      # noqa: E731
    x = t("x").requires_grad_()
    bip = f"{tag}_x_dst" in z
    xd = t("x_dst").requires_grad_() if bip else None
    with _Profile() as p:
        out = conv((x, xd) if bip else x, torch.from_numpy(z[f"{tag}_ei"]).to(DEV))
        out.backward(t("gout"))
    assert all(p.calls.get(name, 0) == 1 for name in KERNELS), p.calls
    res = {"out": out, "gx": x.grad}
    if bip:
        res["gx_dst"] = xd.grad
    res.update({f"g_{n}": p.grad for n, p in conv.named_parameters()})
    return res


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("tag,ic,oc,kw", _GOLDEN_CASES)
def test_standalone_res_gated_matches_golden(golden, tag, ic, oc, kw, dtype):
    """fp32: every array of the reference's golden run.  bf16: the output, and the dtype of every gradient."""
    z = golden("res_gated")
    got = _run_mirror(z, tag, ic, oc, kw, dtype)
    if dtype == torch.float32:
        for k, v in got.items():
            _close(v, torch.from_numpy(z[f"{tag}_{k}"]), tol=1e-4 if k.startswith("g_") else 2e-5, what=k)
    else:
        _close(got["out"], torch.from_numpy(z[f"{tag}_out"]), tol=6e-2, what="out vs golden")
        assert all(v.dtype == torch.bfloat16 for v in got.values())
