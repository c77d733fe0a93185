"""GPU tests of the edge-feature message relu(x_j + e_ji) (GINEConv, gin_conv.py:104-207) fused into the CSR sweep:

  * `Fn.aggregate_edge_relu` against an fp64 formula -- sum / mean, fp32 / bf16, widths on the vector and the scalar
    path, a power-law graph with hub rows (chunked), empty rows and duplicate edges, adopted and sorted CSRs;
  * the ReLU's edge cases (pre-activation exactly 0, NaN, -0.0) and the memory the forward allocates;
  * the UNMODIFIED reference GINEConv (`tg` fixture) under `plugin.install()` against the same layer on the CPU, and
    messages that must not fuse;
  * the standalone `nn.GINEConv` against the reference's golden vectors (tests/golden/gine.npz).
"""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

from pytorch_geometric_b200 import functional as Fn  # noqa: E402
from pytorch_geometric_b200 import ops  # noqa: E402
from pytorch_geometric_b200.graph import CSRGraph  # noqa: E402

DEV = "cuda"
KERNELS = ("edge_relu_csr", "edge_relu_backward_x", "edge_relu_backward_edge")


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
    out-hub (chunked in the transposed sweep); a block of duplicated edges."""
    g = torch.Generator().manual_seed(seed)
    dst = (torch.rand(e, generator=g) ** 3 * (n_dst - 200)).long()           # rows >= n_dst - 200 stay empty
    dst[:3000] = 0
    dst[3000:4500] = 7
    src = torch.randint(0, n_src, (e, ), generator=g)
    src[5000:7000] = 11
    src[8000:8100], dst[8000:8100] = src[8100:8200], dst[8100:8200]         # duplicate edges
    return src, dst, n_src, n_dst


def _bound(a, b, s, tol, what):
    """|a - b| <= tol * s elementwise (s = sum of |terms|), with exact agreement where s == 0."""
    a, b = a.detach().double().cpu(), b.double().cpu()
    bad = (a - b).abs() > tol * s.cpu() + 1e-30
    assert not bad.any(), f"{what}: {int(bad.sum())} entries off, first at {bad.nonzero()[:3].tolist()}"


def _formula(x, a, src, dst, n_dst, reduce, gout):
    """fp64: out, grad_x, grad_a and the sums of |terms| each is bounded by (pre-activation rounded to x's dtype)."""
    pre = (x[src] + a).double()                                              # the add in the storage dtype
    on = ~(pre <= 0)
    term = torch.where(on, pre, torch.zeros_like(pre))
    deg = torch.bincount(dst, minlength=n_dst).clamp(min=1).double().view(-1, 1)
    out = torch.zeros(n_dst, x.size(1), dtype=torch.float64, device=x.device).index_add_(0, dst, term)
    s_out = torch.zeros_like(out).index_add_(0, dst, term.abs())
    g = gout.double()
    if reduce == "mean":
        out, s_out, g = out / deg, s_out / deg, g / deg
    ge = torch.where(on, g[dst], torch.zeros_like(pre))
    gx = torch.zeros(x.size(0), x.size(1), dtype=torch.float64, device=x.device).index_add_(0, src, ge)
    s_gx = torch.zeros_like(gx).index_add_(0, src, ge.abs())
    return out, s_out, gx, s_gx, ge


def _graph(src, dst, n_src, n_dst, adopted):
    """(graph, src, dst) with src / dst in the order the graph expects edge rows in."""
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


@pytest.mark.parametrize("adopted", [False, True])
@pytest.mark.parametrize("feat", [16, 64, 128, 256, 300])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("reduce", ["sum", "mean"])
def test_op_matches_fp64_formula(reduce, dtype, feat, adopted):
    src, dst, n_src, n_dst = _power_law_edges()
    graph, src, dst = _graph(src, dst, n_src, n_dst, adopted)
    assert graph.plan.n_long >= 2
    gen = torch.Generator(device=DEV).manual_seed(feat)
    x = torch.randn(n_src, feat, device=DEV, generator=gen).to(dtype).requires_grad_()
    a = torch.randn(src.numel(), feat, device=DEV, generator=gen).to(dtype).requires_grad_()
    gout = torch.randn(n_dst, feat, device=DEV, generator=gen).to(dtype)
    with _Profile() as p:
        out = Fn.aggregate_edge_relu(graph, x, a, reduce)
        out.backward(gout)
    assert all(p.calls.get(k, 0) == 1 for k in KERNELS), p.calls
    assert out.dtype == dtype and x.grad.dtype == dtype and a.grad.dtype == dtype
    tol = 1e-5 if dtype == torch.float32 else 1.6e-2
    ref, s_out, gx, s_gx, ge = _formula(x.detach(), a.detach(), src, dst, n_dst, reduce, gout)
    _bound(out, ref, s_out, tol, "out")
    _bound(x.grad, gx, s_gx, tol, "grad_x")
    _bound(a.grad, ge, ge.abs(), tol, "grad_edge_rows")
    assert (out[n_dst - 200:] == 0).all()                                    # empty rows


def test_inference_writes_no_mask_and_matches_training():
    src, dst, n_src, n_dst = _power_law_edges(seed=1)
    graph, src, dst = _graph(src, dst, n_src, n_dst, False)
    x = torch.randn(n_src, 64, device=DEV)
    a = torch.randn(src.numel(), 64, device=DEV)
    with torch.no_grad():
        o1 = Fn.aggregate_edge_relu(graph, x, a)
    o2 = Fn.aggregate_edge_relu(graph, x.requires_grad_(), a)
    assert torch.equal(o1, o2.detach())
    # trailing shapes are flattened; E = 0 is valid
    o3 = Fn.aggregate_edge_relu(graph, x.detach().view(n_src, 4, 16), a.view(-1, 4, 16))
    assert o3.shape == (n_dst, 4, 16) and torch.equal(o3.view(n_dst, 64), o1)
    empty = CSRGraph(torch.zeros(0, dtype=torch.long, device=DEV), torch.zeros(0, dtype=torch.long, device=DEV), 5, 4)
    xe = torch.randn(5, 32, device=DEV, requires_grad=True)
    ae = torch.zeros(0, 32, device=DEV, requires_grad=True)
    oe = Fn.aggregate_edge_relu(empty, xe, ae, "mean")
    oe.sum().backward()
    assert (oe == 0).all() and (xe.grad == 0).all() and ae.grad.shape == (0, 32)


@pytest.mark.parametrize("feat", [64, 300, 13])
def test_relu_edge_cases(feat):
    """pre == 0 (a = -x_j exactly): output 0, gradient 0; NaN in a: relu(NaN) = NaN forward and the gradient passes
    through (threshold_backward); -0.0 + -0.0: output +0.0, gradient 0."""
    n = 6
    src = torch.tensor([0, 1, 2, 3, 4, 5, 1], device=DEV)
    dst = torch.tensor([0, 0, 1, 2, 3, 3, 4], device=DEV)
    graph = CSRGraph(src, dst, n, n)
    x = torch.randn(n, feat, device=DEV).abs() + 0.5
    x[4] = -0.0
    a = torch.randn(7, feat, device=DEV)
    a[0] = -x[0]                                   # row 0, edge 0: pre == 0 exactly
    a[2, :5] = float("nan")                        # row 1: NaN pre-activations in the first 5 features
    a[4] = -0.0                                    # row 3, edge 4: -0.0 + -0.0
    a[5] = -x[5] - 1.0                             # row 3, edge 5: negative
    x.requires_grad_()
    a.requires_grad_()
    out = Fn.aggregate_edge_relu(graph, x, a)
    gout = torch.randn(n, feat, device=DEV)
    out.backward(gout)
    o, gx, ga = out.detach(), x.grad, a.grad
    assert torch.equal(o[0], (x[1] + a[1]).relu().detach())
    assert (ga[0] == 0).all() and torch.equal(ga[1], torch.where(x[1] + a[1] > 0, gout[0], 0.0))
    assert o[1, :5].isnan().all() and torch.equal(ga[2, :5], gout[1, :5])
    assert (o[3] == 0).all() and not o[3].signbit().any()
    assert (ga[4] == 0).all() and (ga[5] == 0).all() and (gx[4] == 0).all() and (gx[5] == 0).all()
    assert (o[5] == 0).all() and not o[5].signbit().any()     # empty row
    assert torch.equal(gx[0], torch.zeros_like(gx[0]))        # its only edge had pre == 0


def test_memory_of_the_forward():
    """N = 400k, E = 4M, F = 128 fp32: in training the forward grows the peak by less than one [E, F] tensor (out and
    the E*F/8-byte ReLU mask); under no_grad it allocates only `out` (the hub-row partials are cached by the plan)."""
    n, e, f = 400_000, 4_000_000, 128
    g = torch.Generator(device=DEV).manual_seed(0)
    src = torch.randint(0, n, (e, ), device=DEV, generator=g)
    dst = (torch.rand(e, device=DEV, generator=g) ** 2 * (n - 1)).long()
    graph = CSRGraph(src, dst, n, n)
    del src, dst
    x = torch.randn(n, f, device=DEV, generator=g)
    a = torch.randn(e, f, device=DEV, generator=g)
    one_ef = e * f * 4
    with torch.no_grad():
        Fn.aggregate_edge_relu(graph, x, a)                    # warm: the plan's partials
    torch.cuda.synchronize()
    for grad in (False, True):
        x.requires_grad_(grad)
        a.requires_grad_(grad)
        torch.cuda.reset_peak_memory_stats()
        m0 = torch.cuda.memory_allocated()
        with torch.set_grad_enabled(grad):
            out = Fn.aggregate_edge_relu(graph, x, a)
        torch.cuda.synchronize()
        growth = torch.cuda.max_memory_allocated() - m0
        out_bytes = out.numel() * 4
        if grad:
            assert out_bytes + e * f // 8 <= growth < one_ef, (growth, one_ef)
        else:
            assert growth <= out_bytes + (2 << 20), (growth, out_bytes)
        del out


# ------------------------------------------------------------------------------------------------ the reference layer
@pytest.fixture
def plugin(tg):
    from pytorch_geometric_b200 import plugin as P
    yield P
    P.uninstall()


def _no_materialise(monkeypatch):
    from pytorch_geometric_b200.plugin.lazy import LazyRows
    seen = []
    orig = LazyRows.materialise
    monkeypatch.setattr(LazyRows, "materialise", lambda self: seen.append(1) or orig(self))
    return seen


def _mlp(f_in, f_out=16):
    return torch.nn.Sequential(torch.nn.Linear(f_in, 24), torch.nn.ReLU(), torch.nn.Linear(24, f_out))


def _ref_case(tg, case, f=32, n_src=400, n_dst=400, e=5000, seed=3):
    g = torch.Generator().manual_seed(seed)
    bip = case == "bipartite"
    if bip:
        n_dst = 250
    src = torch.randint(0, n_src, (e, ), generator=g)
    dst = (torch.rand(e, generator=g) ** 2 * (n_dst - 1)).long()
    dst[:700] = 3                                                       # a hub row above the 512-edge chunk
    ei = torch.stack([src, dst])
    fe = 7 if case == "edge_dim" else f
    ea = torch.randn(e, fe, generator=g)
    if case == "edge_index_sorted":
        ei, perm = tg.EdgeIndex(ei, sparse_size=(n_src, n_dst)).sort_by("col")
        ea = ea[perm]
    x = torch.randn(n_src, f, generator=g)
    x_dst = torch.randn(n_dst, f, generator=g) if bip else None
    kw = {"edge_dim": {"edge_dim": 7}, "train_eps": {"train_eps": True, "eps": 0.3}, "mean": {"aggr": "mean"},
          "bipartite": {"aggr": "mean", "eps": -0.2}}.get(case, {})
    return ei, ea, x, x_dst, kw


@pytest.mark.parametrize("case", ["plain", "edge_dim", "train_eps", "mean", "bipartite", "edge_index_sorted"])
def test_unmodified_reference_gineconv_reaches_the_fused_kernels(tg, plugin, monkeypatch, case):
    ei, ea, x, x_dst, kw = _ref_case(tg, case)
    plugin.install()
    seen = _no_materialise(monkeypatch)
    torch.manual_seed(7)
    ref = tg.nn.GINEConv(_mlp(32), **kw)
    gpu = tg.nn.GINEConv(_mlp(32), **kw)
    gpu.load_state_dict(ref.state_dict())
    gpu = gpu.to(DEV)
    assert type(gpu).__module__.startswith("torch_geometric.")
    leaves_c = [t.clone().requires_grad_() for t in (x, ea) + ((x_dst, ) if x_dst is not None else ())]
    leaves_g = [t.detach().clone().to(DEV).requires_grad_() for t in leaves_c]

    def run(mod, leaves, edge_index):
        xin = (leaves[0], leaves[2]) if x_dst is not None else leaves[0]
        return mod(xin, edge_index, leaves[1])
    want = run(ref, leaves_c, ei)
    gout = torch.randn_like(want)
    want.backward(gout)
    assert not seen                                                      # the CPU run falls through untouched
    with _Profile() as p:
        got = run(gpu, leaves_g, ei.to(DEV))
        got.backward(gout.to(DEV))
    assert all(p.calls.get(k, 0) == 1 for k in KERNELS), p.calls
    assert not seen, "the message was materialised"
    _close(got, want, what=f"{case} out")
    for i, (lg, lc) in enumerate(zip(leaves_g, leaves_c)):
        _close(lg.grad, lc.grad, tol=5e-5, what=f"{case} grad of input {i}")
    for (n, pg), (_, pc) in zip(gpu.named_parameters(), ref.named_parameters()):
        _close(pg.grad, pc.grad, tol=1e-4, what=f"{case} grad {n}")


def _unfused_layer(tg, kind):
    class Msg(tg.nn.MessagePassing):
        def __init__(self):
            super().__init__(aggr="add")

        def forward(self, x, edge_index, edge_attr):
            return self.propagate(edge_index, x=x, edge_attr=edge_attr)

        def message(self, x_j, edge_attr):
            if kind == "sigmoid":
                return (x_j + edge_attr).sigmoid()
            if kind == "broadcast":
                return (x_j + edge_attr[:, :1]).relu()
            return (x_j + edge_attr).relu() + 1e-7                     # GENConv's `+ eps` after the ReLU
    return Msg()


@pytest.mark.parametrize("kind", ["sigmoid", "broadcast", "eps_after_relu", "mixed_dtype", "max"])
def test_messages_that_must_not_fuse_match_the_reference(tg, plugin, kind):
    g = torch.Generator().manual_seed(9)
    n, e, f = 200, 3000, 16
    ei = torch.stack([torch.randint(0, n, (e, ), generator=g), torch.randint(0, n, (e, ), generator=g)])
    x = torch.randn(n, f, generator=g)
    ea = torch.randn(e, f, generator=g)
    plugin.install()
    if kind == "mixed_dtype":                      # bf16 x, fp32 edge_attr: promoted to fp32 as in the reference
        torch.manual_seed(1)
        ref = tg.nn.GINEConv(_mlp(f))
        x = x.bfloat16()
    elif kind == "max":
        torch.manual_seed(1)
        ref = tg.nn.GINEConv(_mlp(f), aggr="max")
    else:
        ref = _unfused_layer(tg, kind)
    gpu = copy.deepcopy(ref).to(DEV)
    xc, eac = x.clone().requires_grad_(), ea.clone().requires_grad_()
    xg, eag = x.to(DEV).requires_grad_(), ea.to(DEV).requires_grad_()
    want = ref(xc, ei, eac)
    with _Profile() as p:
        got = gpu(xg, ei.to(DEV), eag)
    assert p.calls.get("edge_relu_csr", 0) == 0, p.calls
    assert got.dtype == want.dtype, (got.dtype, want.dtype)
    _close(got, want, tol=1e-5 if x.dtype == torch.float32 else 2e-2, what=kind)
    gout = torch.randn_like(want)
    want.backward(gout)
    got.backward(gout.to(DEV))
    _close(eag.grad, eac.grad, tol=1e-4 if x.dtype == torch.float32 else 2e-2, what=kind + " grad_edge_attr")


# ------------------------------------------------------------------------------------------------ the standalone mirror
def _run_mirror(z, tag, kw, dtype, through=None):
    """nn.GINEConv loaded with the golden parameters, on the golden inputs (cast to `dtype`, after a round trip
    through `through` when given), forward + backward: {name: tensor}."""
    from pytorch_geometric_b200.nn import GINEConv
    conv = GINEConv(torch.nn.Sequential(torch.nn.Linear(8, 16), torch.nn.ReLU(), torch.nn.Linear(16, 8)), **kw)
    conv.load_state_dict({k[len(tag) + 3:]: torch.from_numpy(v) for k, v in z.items() if k.startswith(f"{tag}_p_")})
    cast = (lambda v: v.to(through).to(dtype)) if through is not None else (lambda v: v.to(dtype))   # noqa: E731
    conv = conv.to(DEV)
    with torch.no_grad():
        for p in conv.parameters():
            p.copy_(cast(p))
    conv = conv.to(dtype)
    t = lambda k: cast(torch.from_numpy(z[f"{tag}_{k}"]).to(DEV))       # noqa: E731
    x, ea = t("x").requires_grad_(), t("ea").requires_grad_()
    bip = f"{tag}_x_dst" in z
    xd = t("x_dst").requires_grad_() if bip else None
    out = conv((x, xd) if bip else x, torch.from_numpy(z[f"{tag}_ei"]).to(DEV), ea)
    out.backward(t("gout"))
    res = {"out": out, "gx": x.grad, "gea": ea.grad}
    if bip:
        res["gx_dst"] = xd.grad
    res.update({f"g_{n}": p.grad for n, p in conv.named_parameters()})
    return res


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("tag,kw", [("plain", {}), ("edge_dim", {"edge_dim": 5, "train_eps": True, "eps": 0.25}),
                                    ("mean_bip", {"aggr": "mean", "eps": -0.5})])
def test_standalone_gineconv_matches_golden(golden, tag, kw, dtype):
    """fp32: every array of the reference's golden run.  bf16: the output against the golden run, and every array
    against the fp32 mirror fed the same bf16-rounded inputs and parameters.  In the mean / bipartite case the MLP's
    hidden pre-activations sit close enough to 0 that bf16 rounding flips that ReLU, which moves a gradient by a whole
    term (the reference's own bf16 run on the CPU is 30% off the golden gradients there), so only its output and
    dtypes are checked in bf16."""
    z = golden("gine")
    got = _run_mirror(z, tag, kw, dtype)
    if dtype == torch.float32:
        for k, v in got.items():
            _close(v, torch.from_numpy(z[f"{tag}_{k}"]), tol=1e-4 if k.startswith("g_") else 2e-5, what=k)
    else:
        _close(got["out"], torch.from_numpy(z[f"{tag}_out"]), tol=6e-2, what="out vs golden")
        want = _run_mirror(z, tag, kw, torch.float32, through=torch.bfloat16)
        for k, v in got.items():
            assert v.dtype == torch.bfloat16, k
            if tag != "mean_bip":
                _close(v, want[k], tol=6e-2 if k.startswith("g_") else 3e-2, what=k)
