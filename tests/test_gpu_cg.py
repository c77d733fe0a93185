"""GPU tests of CGConv's crystal-graph message sigmoid(f) * softplus(s), [f | s] = u_i + v_j (+ c_e) (cg_conv.py:93-98),
fused into the CSR sweep:

  * `Fn.aggregate_cg` / `aggregate_cg_uv` against an fp64 formula -- sum / mean, fp32 / bf16, widths on the vector and
    the scalar path, with and without c (c requiring grad or not, which selects the grad_v route), u and v as two
    tensors or the halves of one [N, 4F] tensor, a bipartite power-law graph with a chunked destination hub and a
    chunked source out-hub, empty and single-edge rows, adopted and sorted CSRs, one launch per entry point;
  * the edge cases of sigmoid and softplus (threshold 20, exp underflow, +-inf, NaN, 0 * inf) against the reference's
    own ops on the CPU, and the memory of forward and training step;
  * an unmodified reference CGConv copied into `plugin.conv.B200CGConv` against the same layer on the CPU, and the
    configurations that must fall through;
  * the standalone `nn.CGConv` against the reference's golden vectors (tests/golden/cg.npz).

bf16 bar: u, v and c are each rounded to bf16 before the sweep adds them, where the reference rounds one Linear output;
the formula takes the rounded u, v and c as its inputs and rounds f and s once, so the bar of 1.6e-2 * sum|terms|
covers the kernel's rounding of sigmoid, softplus and their product and the bf16 output.
"""
import copy
import math

import pytest
import torch
import torch.nn.functional as F

pytestmark = pytest.mark.gpu

from pytorch_geometric_b200 import functional as Fn  # noqa: E402
from pytorch_geometric_b200 import ops  # noqa: E402
from pytorch_geometric_b200.graph import CSRGraph  # noqa: E402

DEV = "cuda"
CG = ("cg_csr", "cg_backward_dst", "cg_backward_src")


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


def _check(a, b, s, tol, what):
    """|a - b| <= tol * s elementwise (s = sum of |terms|), NaN exactly where the formula has NaN, equal infinities."""
    a, b, s = a.detach().double().cpu(), b.detach().double().cpu(), s.detach().double().cpu()
    assert torch.equal(a.isnan(), b.isnan()), f"{what}: NaN pattern differs"
    fin = b.isfinite()
    assert torch.equal(a[~fin & ~b.isnan()], b[~fin & ~b.isnan()]), f"{what}: infinities differ"
    bad = ((a - b).abs() > tol * s + 1e-30) & fin
    assert not bad.any(), f"{what}: {int(bad.sum())} entries off, first at {bad.nonzero()[:3].tolist()}"


def _power_law_edges(n_src=3000, n_dst=2500, e=60000, seed=0):
    """Destinations: a hub far above the 512-edge chunk, a power-law body, single-edge rows and a tail of empty rows;
    sources: one out-hub (chunked in the transposed sweep) and a tail without out-edges; a block of duplicated edges."""
    g = torch.Generator().manual_seed(seed)
    dst = (torch.rand(e, generator=g) ** 3 * (n_dst - 300)).long()           # rows >= n_dst - 300 hold no body edge
    dst[:3000] = 0
    src = torch.randint(0, n_src - 100, (e, ), generator=g)                  # sources >= n_src - 100 send nothing
    src[5000:7000] = 11
    src[8000:8100], dst[8000:8100] = src[8100:8200], dst[8100:8200]         # duplicate edges
    dst[9000:9100] = torch.arange(n_dst - 300, n_dst - 200)                  # single-edge rows; the last 200 stay empty
    return src, dst, n_src, n_dst


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


def _sig(x):
    """fp64 sigmoid and its derivative from t = exp(-|x|)."""
    t = torch.exp(-x.abs())
    r = 1.0 / (1.0 + t)
    return torch.where(x >= 0, r, t * r), t * r * r


def _formula(u, v, c, src, dst, n_src, n_dst, reduce, gout, dtype):
    """fp64 out, grad_u, grad_v, grad_c, each with its sum of |terms|; f and s rounded to the storage dtype once."""
    W = u.size(1)
    Fh = W // 2
    pre = u[dst].double() + v[src].double() + (0 if c is None else c.double())
    if dtype != torch.float32:
        pre = pre.to(dtype).double()
    f, s = pre[:, :Fh], pre[:, Fh:]
    sig, dsig = _sig(f)
    sp = F.softplus(s, threshold=20)
    dsp = torch.where(s > 20, torch.ones_like(s), _sig(s)[0])
    deg = torch.bincount(dst, minlength=n_dst).clamp(min=1).double().view(-1, 1)
    g = gout.double()

    def red(n, idx, t):
        z = torch.zeros(n, t.size(1), dtype=torch.float64, device=u.device)
        return z.clone().index_add_(0, idx, t), z.index_add_(0, idx, t.abs())
    out, s_out = red(n_dst, dst, sig * sp)
    if reduce == "mean":
        out, s_out, g = out / deg, s_out / deg, g / deg
    gi = g[dst]
    d = torch.cat([gi * dsig * sp, gi * sig * dsp], 1)
    return (out, s_out), red(n_dst, dst, d), red(n_src, src, d), (d, d.abs())


def _run(graph, u, v, c, c_grad, reduce, gout, layout):
    """out, grad_u, grad_v, grad_c of the op (grad_c None unless c requires grad)."""
    W = u.size(1)
    c = None if c is None else c.clone().requires_grad_(c_grad)
    if layout == "packed":
        uv = torch.cat([u, v], 1).requires_grad_()
        out = Fn.aggregate_cg_uv(graph, uv, c, reduce)
        out.backward(gout)
        return out, uv.grad[:, :W], uv.grad[:, W:], None if c is None else c.grad
    u, v = u.clone().requires_grad_(), v.clone().requires_grad_()
    out = Fn.aggregate_cg(graph, u, v, c, reduce)
    out.backward(gout)
    return out, u.grad, v.grad, None if c is None else c.grad


@pytest.mark.parametrize("layout", ["separate", "packed"])
@pytest.mark.parametrize("adopted", [False, True])
@pytest.mark.parametrize("c_kind", ["none", "grad", "frozen"])
@pytest.mark.parametrize("feat", [6, 16, 21, 64, 128, 256])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("reduce", ["sum", "mean"])
def test_op_matches_fp64_formula(reduce, dtype, feat, c_kind, adopted, layout):
    src, dst, n_src, n_dst = _power_law_edges()
    if layout == "packed":                       # one [N, 4F] product: as many sources as destinations
        n_dst = n_src
    graph, src, dst = _graph(src, dst, n_src, n_dst, adopted)
    gen = torch.Generator(device=DEV).manual_seed(feat)
    u = (2 * torch.randn(n_dst, 2 * feat, device=DEV, generator=gen)).to(dtype)
    v = (2 * torch.randn(n_src, 2 * feat, device=DEV, generator=gen)).to(dtype)
    c = None if c_kind == "none" else torch.randn(src.numel(), 2 * feat, device=DEV, generator=gen).to(dtype)
    gout = torch.randn(n_dst, feat, device=DEV, generator=gen).to(dtype)
    with _Profile() as p:
        got = _run(graph, u, v, c, c_kind == "grad", reduce, gout, layout)
    # with grad_c, grad_v is the segment sum of its rows (spmm over the transposed CSR); otherwise the transposed sweep
    want_calls = {"cg_csr": 1, "cg_backward_dst": 1, "cg_backward_src": 0 if c_kind == "grad" else 1,
                  "spmm_csr": 1 if c_kind == "grad" else 0}
    assert {k: p.calls.get(k, 0) for k in want_calls} == want_calls, p.calls
    assert graph.plan.n_long >= 1 and graph.plan_t.n_long >= 1
    assert all(t is None or t.dtype == dtype for t in got)
    tol = 1e-5 if dtype == torch.float32 else 1.6e-2
    want = _formula(u, v, c, src, dst, n_src, n_dst, reduce, gout, dtype)
    for name, t, (ref, s) in zip(("out", "grad_u", "grad_v", "grad_c"), got, want):
        if name == "grad_c" and c_kind != "grad":
            assert t is None
            continue
        _check(t, ref, s, tol, name)
    assert (got[0][n_dst - 200:] == 0).all() and (got[1][n_dst - 200:] == 0).all()      # empty rows
    assert (got[2][n_src - 100:] == 0).all()                                            # sources without out-edges


def test_inference_only_needed_sweeps_and_errors():
    src, dst, n_src, n_dst = _power_law_edges(seed=1)
    graph, src, dst = _graph(src, dst, n_src, n_dst, False)
    u = torch.randn(n_dst, 128, device=DEV)
    v = torch.randn(n_src, 128, device=DEV)
    c = torch.randn(src.numel(), 128, device=DEV)
    with torch.no_grad(), _Profile() as p:
        Fn.aggregate_cg(graph, u, v, c)
    assert p.calls == {"cg_csr": 1}, p.calls
    # only u needs a gradient: no transposed sweep
    ur = u.clone().requires_grad_()
    with _Profile() as p:
        Fn.aggregate_cg(graph, ur, v, c).sum().backward()
    assert p.calls == {"cg_csr": 1, "cg_backward_dst": 1}, p.calls
    # only v needs a gradient: no destination sweep
    vr = v.clone().requires_grad_()
    with _Profile() as p:
        Fn.aggregate_cg(graph, u, vr, c, "mean").sum().backward()
    assert p.calls == {"cg_csr": 1, "cg_backward_src": 1}, p.calls
    empty = CSRGraph(torch.zeros(0, dtype=torch.long, device=DEV), torch.zeros(0, dtype=torch.long, device=DEV), 5, 4)
    ue = torch.full((4, 32), float("inf"), device=DEV, requires_grad=True)
    ve = torch.full((5, 32), float("nan"), device=DEV, requires_grad=True)
    oe = Fn.aggregate_cg(empty, ue, ve, None, "mean")
    oe.backward(torch.full_like(oe, float("inf")))
    assert (oe == 0).all() and (ue.grad == 0).all() and (ve.grad == 0).all()
    with pytest.raises(ValueError, match="sum or mean"):
        Fn.aggregate_cg(graph, u, v, c, "max")
    with pytest.raises(ValueError, match="destination nodes"):
        Fn.aggregate_cg(graph, v, v, c)
    with pytest.raises(ValueError, match="c must be"):
        Fn.aggregate_cg(graph, u, v, c[:, :64])
    with pytest.raises(ValueError, match="v must be"):
        Fn.aggregate_cg(graph, u, v.bfloat16(), c)


def _nextafter(x, d):
    return torch.nextafter(torch.tensor(x), torch.tensor(d)).item()


# (f, s) per node: threshold 20 and its neighbours, exp underflow, +-inf, NaN, f = -inf with s = +inf (0 * inf)
_EDGE_PAIRS = [(0.0, 20.0), (0.0, _nextafter(20.0, math.inf)), (0.0, _nextafter(20.0, -math.inf)), (20.0, 0.5),
               (_nextafter(20.0, math.inf), 1.0), (_nextafter(20.0, -math.inf), -1.0), (-20.0, 5.0), (30.0, -100.0),
               (-30.0, -200.0), (math.inf, 3.0), (-math.inf, 3.0), (math.nan, 0.0), (0.0, math.nan),
               (-math.inf, math.inf), (1.0, math.inf), (1.0, -math.inf), (-2.0, -90.0)]


@pytest.mark.parametrize("feat", [64, 13])
@pytest.mark.parametrize("reduce", ["sum", "mean"])
def test_activation_edge_cases_match_the_reference_on_cpu(feat, reduce):
    """Each node i has a self-loop and node 0 also receives every other edge; u carries (f, s), v = 0, so the reference's
    sigmoid(f) * softplus(s), its autograd and its reduction on the CPU give the expected out, grad_u and grad_v."""
    n = len(_EDGE_PAIRS)
    src = torch.tensor(list(range(n)) + list(range(1, n)))
    dst = torch.tensor(list(range(n)) + [0] * (n - 1))
    fs = torch.tensor(_EDGE_PAIRS, dtype=torch.float32)
    u = torch.cat([fs[:, :1].repeat(1, feat), fs[:, 1:].repeat(1, feat)], 1)
    v = torch.zeros(n, 2 * feat)
    gout = torch.randn(n, feat, generator=torch.Generator().manual_seed(2))
    # reference: the pre-activation of edge e is u[dst[e]] (v = 0)
    ur = u.clone().requires_grad_()
    vr = v.clone().requires_grad_()
    z = ur[dst] + vr[src]
    m = z[:, :feat].sigmoid() * F.softplus(z[:, feat:])
    want = torch.zeros(n, feat).index_add_(0, dst, m)
    if reduce == "mean":
        want = want / torch.bincount(dst, minlength=n).clamp(min=1).view(-1, 1)
    want.backward(gout)
    graph = CSRGraph(src.to(DEV), dst.to(DEV), n, n)
    ug, vg = u.to(DEV).requires_grad_(), v.to(DEV).requires_grad_()
    got = Fn.aggregate_cg(graph, ug, vg, None, reduce)
    got.backward(gout.to(DEV))
    for name, a, b in (("out", got, want), ("grad_u", ug.grad, ur.grad), ("grad_v", vg.grad, vr.grad)):
        _check(a, b, b.abs().clamp(min=1.0), 1e-5, f"{reduce} {name}")
    assert got[13].isnan().all()                                  # sigmoid(-inf) * softplus(+inf) = 0 * inf
    assert torch.equal(got[1].cpu(), want[1])                     # s just above 20: softplus(s) = s exactly


def test_memory_of_forward_and_training_step():
    """N = 400k, E = 4M, F = 64 fp32: the forward without c grows the peak by less than one [E, F] tensor beyond out;
    a training step with c grows it by less than [E, 2F] beyond c and grad_c."""
    n, e, f = 400_000, 4_000_000, 64
    g = torch.Generator(device=DEV).manual_seed(0)
    src = torch.randint(0, n, (e, ), device=DEV, generator=g)
    dst = (torch.rand(e, device=DEV, generator=g) ** 2 * (n - 1)).long()
    graph = CSRGraph(src, dst, n, n)
    del src, dst
    u, v = (torch.randn(n, 2 * f, device=DEV, generator=g).requires_grad_() for _ in range(2))
    c = torch.randn(e, 2 * f, device=DEV, generator=g).requires_grad_()
    gout = torch.randn(n, f, device=DEV, generator=g)
    one_ef = e * f * 4
    out_bytes = n * f * 4
    for cc in (None, c):                                           # warm: transpose, plans' partials
        Fn.aggregate_cg(graph, u, v, cc, "mean").backward(gout)
    u.grad = v.grad = c.grad = None
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    m0 = torch.cuda.memory_allocated()
    with torch.no_grad():
        out = Fn.aggregate_cg(graph, u, v, None, "mean")
    torch.cuda.synchronize()
    fwd = torch.cuda.max_memory_allocated() - m0 - out_bytes
    del out
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    m1 = torch.cuda.memory_allocated()
    Fn.aggregate_cg(graph, u, v, c, "mean").backward(gout)
    torch.cuda.synchronize()
    step = torch.cuda.max_memory_allocated() - m1 - 2 * one_ef        # grad_c, the counterpart of c
    assert fwd < one_ef and step < 2 * one_ef, (fwd, step, one_ef)


# ------------------------------------------------------------------------------------------------ the reference layer
@pytest.fixture
def plugin(tg):
    from pytorch_geometric_b200 import plugin as P
    yield P
    P.uninstall()


def _b200(ref):
    from pytorch_geometric_b200.plugin import conv as PC
    m = copy.deepcopy(ref).to(DEV)
    m.__class__ = PC.B200CGConv
    return m


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
    kw = {"dim": {"dim": 7}, "bipartite": {"dim": 4}, "mean": {"aggr": "mean"}, "batch_norm": {"batch_norm": True},
          "target_to_source": {"flow": "target_to_source"}}.get(case, {})
    f_src, f_dst = (24, 32) if bip else (32, 32)
    x = torch.randn(n_src, f_src, generator=g)
    x_dst = torch.randn(n_dst, f_dst, generator=g) if bip else None
    ea = torch.randn(e, kw["dim"], generator=g) if "dim" in kw else None
    return ei, x, x_dst, ea, kw, ((f_src, f_dst) if bip else f_src)


@pytest.mark.parametrize("case", ["plain", "dim", "bipartite", "mean", "batch_norm", "target_to_source",
                                  "edge_index_sorted"])
def test_unmodified_reference_cg_reaches_the_fused_kernels(tg, plugin, case):
    ei, x, x_dst, ea, kw, ch = _ref_case(tg, case)
    plugin.install()
    torch.manual_seed(7)
    ref = tg.nn.CGConv(ch, **kw)
    gpu = _b200(ref)
    leaves_c = [t.clone().requires_grad_() for t in (x, x_dst, ea) if t is not None]
    leaves_g = [t.detach().clone().to(DEV).requires_grad_() for t in leaves_c]

    def run(mod, leaves, dev):
        it = iter(leaves)
        xs = next(it)
        xin = (xs, next(it)) if x_dst is not None else xs
        return mod(xin, ei.to(dev), next(it) if ea is not None else None)
    want = run(ref, leaves_c, "cpu")
    gout = torch.randn_like(want)
    want.backward(gout)
    with _Profile() as p:
        got = run(gpu, leaves_g, DEV)
        got.backward(gout.to(DEV))
    assert p.calls.get("cg_csr") == 1 and p.calls.get("cg_backward_dst") == 1, p.calls
    assert p.calls.get("cg_backward_src", 0) == (0 if ea is not None else 1), p.calls
    _close(got, want, what=f"{case} out")
    for i, (lg, lc) in enumerate(zip(leaves_g, leaves_c)):
        _close(lg.grad, lc.grad, tol=5e-5, what=f"{case} grad of input {i}")
    for (n, pg), (_, pc) in zip(gpu.named_parameters(), ref.named_parameters()):
        _close(pg.grad, pc.grad, tol=1e-4, what=f"{case} grad {n}")
    if case == "batch_norm":
        _close(gpu.bn.running_mean, ref.bn.running_mean, what="running_mean")
        _close(gpu.bn.running_var, ref.bn.running_var, what="running_var")


@pytest.mark.parametrize("kind", ["max", "hook", "fp64", "sparse"])
def test_configurations_that_must_fall_through(tg, plugin, kind):
    g = torch.Generator().manual_seed(9)
    n, e, f = 200, 3000, 16
    ei = torch.stack([torch.randint(0, n, (e, ), generator=g), torch.randint(0, n, (e, ), generator=g)])
    x = torch.randn(n, f, generator=g)
    ea = torch.randn(e, 3, generator=g)
    plugin.install()
    torch.manual_seed(1)
    dim = 0 if kind == "sparse" else 3
    ea = ea if dim else None
    ref = tg.nn.CGConv(f, dim=dim, aggr="max" if kind == "max" else "add")
    gpu = _b200(ref)
    seen = []
    if kind == "hook":
        gpu.register_message_forward_hook(lambda mod, inp, out: seen.append(1))
    dt = torch.float64 if kind == "fp64" else torch.float32
    if kind == "fp64":
        ref, gpu = ref.double(), gpu.double()

    def adj(dev):
        if kind == "sparse":
            return tg.utils.to_torch_csc_tensor(ei.to(dev), size=(n, n)).t()
        return ei.to(dev)
    xc = x.to(dt).clone().requires_grad_()
    xg = x.to(dt).to(DEV).requires_grad_()
    want = ref(xc, adj("cpu"), None if ea is None else ea.to(dt))
    with _Profile() as p:
        got = gpu(xg, adj(DEV), None if ea is None else ea.to(dt).to(DEV))
    assert not any(p.calls.get(k, 0) for k in CG), p.calls
    assert got.dtype == want.dtype
    assert seen == ([1] if kind == "hook" else [])
    _close(got, want, tol=1e-5, what=kind)
    gout = torch.randn_like(want)
    want.backward(gout)
    got.backward(gout.to(DEV))
    _close(xg.grad, xc.grad, tol=1e-4, what=kind + " grad")


# ------------------------------------------------------------------------------------------------ the standalone mirror
_GOLDEN_CASES = [("plain", 16, {}), ("bip_mean_bn", (8, 16), dict(dim=5, aggr="mean", batch_norm=True)),
                 ("narrow", 6, dict(dim=3, bias=False))]


def _run_mirror(z, tag, ch, kw, dtype):
    from pytorch_geometric_b200.nn import CGConv
    conv = CGConv(ch, **kw)
    conv.load_state_dict({k[len(tag) + 3:]: torch.from_numpy(v) for k, v in z.items() if k.startswith(f"{tag}_p_")})
    conv = conv.to(DEV).to(dtype).train()
    t = lambda k: torch.from_numpy(z[f"{tag}_{k}"]).to(DEV).to(dtype)      # noqa: E731
    x = t("x").requires_grad_()
    bip = f"{tag}_x_dst" in z
    xd = t("x_dst").requires_grad_() if bip else None
    ea = t("ea").requires_grad_() if f"{tag}_ea" in z else None
    with _Profile() as p:
        out = conv((x, xd) if bip else x, torch.from_numpy(z[f"{tag}_ei"]).to(DEV), ea)
        out.backward(t("gout"))
    assert p.calls.get("cg_csr") == 1 and p.calls.get("cg_backward_dst") == 1, p.calls
    res = {"out": out, "gx": x.grad}
    if bip:
        res["gx_dst"] = xd.grad
    if ea is not None:
        res["gea"] = ea.grad
    res.update({f"g_{n}": p.grad for n, p in conv.named_parameters()})
    return res


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("tag,ch,kw", _GOLDEN_CASES)
def test_standalone_cg_matches_golden(golden, tag, ch, kw, dtype):
    """fp32: every array of the reference's golden run.  bf16: the output, and the dtype of every gradient."""
    z = golden("cg")
    got = _run_mirror(z, tag, ch, kw, dtype)
    if dtype == torch.float32:
        for k, v in got.items():
            _close(v, torch.from_numpy(z[f"{tag}_{k}"]), tol=1e-4 if k.startswith("g") else 2e-5, what=k)
    else:
        _close(got["out"], torch.from_numpy(z[f"{tag}_out"]), tol=6e-2, what="out vs golden")
        assert all(v.dtype == torch.bfloat16 for v in got.values())
