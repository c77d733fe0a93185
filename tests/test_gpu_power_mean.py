"""GPU tests of the power-mean aggregation (csrc/power_mean.cu, functional.power_mean_aggregate,
nn.aggr.PowerMeanAggregation) and of the fused GENConv (plugin.conv.B200GENConv):

  * the op against an fp64 evaluation of the reference's op sequence for out, grad_x, grad_a and grad_p -- fp32 / bf16,
    widths on the vector and the scalar path, every message form (x only, edge rows only, relu(x) + eps,
    relu(x + a) + eps with a trainable or frozen, which selects the grad_x route), p as the number 1, 2.5 and 0.5 and
    learnable with 1 or F channels, clamp_max 100 and None, adopted and sorted CSRs, and a small chunk so hub rows take
    the combine kernels;
  * one launch per entry point, no device->host sync with a learnable p, and identical bits on a second run;
  * non-finite messages against the reference's own ops on the CPU;
  * PowerMeanAggregation and B200GENConv against the reference modules, and the fall-through configurations.

The formula rounds m, y and M to the storage dtype where the reference materialises them (straight-through for the
gradient), so the bf16 bar covers the kernel's fp32 accumulation and the bf16 outputs.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

from pytorch_geometric_b200 import functional as Fn  # noqa: E402
from pytorch_geometric_b200 import ops  # noqa: E402
from pytorch_geometric_b200.graph import CSRGraph  # noqa: E402
from pytorch_geometric_b200.nn import PowerMeanAggregation  # noqa: E402

DEV = "cuda"
EPS = 1e-7
LO = 1e-4
PM = ("power_mean_csr", "power_mean_backward_dst", "power_mean_backward_src")


class _Profile:
    def __enter__(self):
        ops.PROFILE.reset(enabled=True)
        return self

    def __exit__(self, *a):
        self.calls = {k: v["calls"] for k, v in ops.PROFILE.summary().items()}
        ops.PROFILE.reset(enabled=False)
        return False


def _check(a, b, s, tol, what):
    """|a - b| <= tol * s elementwise (s = sum of |terms|), NaN exactly where the formula has NaN, equal infinities."""
    a, b, s = a.detach().double().cpu(), b.detach().double().cpu(), s.detach().double().cpu()
    assert a.shape == b.shape, (what, a.shape, b.shape)
    assert torch.equal(a.isnan(), b.isnan()), f"{what}: NaN pattern differs"
    fin = b.isfinite()
    assert torch.equal(a[~fin & ~b.isnan()], b[~fin & ~b.isnan()]), f"{what}: infinities differ"
    bad = ((a - b).abs() > tol * s + 1e-30) & fin
    assert not bad.any(), f"{what}: {int(bad.sum())} entries off, first at {bad.nonzero()[:3].tolist()}"


def _edges(n_src=300, n_dst=250, e=6000, seed=0):
    """A destination hub above any chunk, a power-law body, single-edge and empty rows, a source out-hub, duplicates."""
    g = torch.Generator().manual_seed(seed)
    dst = (torch.rand(e, generator=g) ** 2 * (n_dst - 30)).long()
    dst[:700] = 0
    src = torch.randint(0, n_src - 10, (e, ), generator=g)
    src[1000:1400] = 7
    src[2000:2010], dst[2000:2010] = src[2010:2020], dst[2010:2020]
    dst[3000:3010] = torch.arange(n_dst - 30, n_dst - 20)
    return src, dst, n_src, n_dst


def _graph(src, dst, n_src, n_dst, adopted, chunk):
    src, dst = src.to(DEV), dst.to(DEV)
    if not adopted:
        return CSRGraph(src, dst, n_src, n_dst, chunk=chunk), src, dst
    order = torch.sort(dst, stable=True).indices
    src, dst = src[order], dst[order]
    rowptr = torch.zeros(n_dst + 1, dtype=torch.int64, device=DEV)
    rowptr[1:] = torch.bincount(dst, minlength=n_dst).cumsum(0)
    return CSRGraph.from_csr(rowptr, src, n_src, chunk=chunk), src, dst


def _formula(x, a, p, src, dst, n_src, n_dst, form, eps, hi, dtype):
    """fp64 out with autograd (x, a, p: fp64 leaves holding the storage-dtype values) by the reference's op sequence,
    and the sums of |terms| of out, of each message's gradient, of grad_x and of grad_p per channel, given grad_out."""
    def rnd(v):
        return v if dtype == torch.float32 else v + (v.to(dtype).double() - v).detach()

    if form in ("x", "rows"):
        m = x[src] if form == "x" else a
    else:
        s = x[src] if form == "x_relu" else rnd(x[src] + a)
        m = rnd(s.relu() + eps)
    F = m.size(1)
    deg = torch.bincount(dst, minlength=n_dst).clamp(min=1).double().view(-1, 1)
    if p is None:
        y = m
    else:
        c = m.clamp(min=LO, max=hi)
        y = rnd(c.pow(p))
    M = rnd(torch.zeros(n_dst, F, dtype=torch.float64, device=m.device).index_add(0, dst, y) / deg)
    out = M if p is None else rnd(M.clamp(min=LO, max=hi).pow(1.0 / p))
    return out, y.detach(), M.detach(), deg


def _sums(out, y, M, m_abs, deg, p, src, dst, n_src, gout, hi):
    """Sums of |terms| of out, of the message gradient, of grad_x and of grad_p (|ln c| counted as at least 1)."""
    g = gout.double()
    if p is None:
        s_out = torch.zeros_like(out).index_add(0, dst, m_abs) / deg
        s_m = (g / deg)[dst].abs()
    else:
        pa = p.detach().abs().double()
        ip = torch.clamp(1.0 / pa, min=1.0)
        s_out = out.detach().abs() * ip
        C = M.clamp(min=LO, max=hi)
        G = (g * out.detach() / (pa * C * deg)).abs()
        c = m_abs.clamp(min=LO, max=hi)
        s_m = G[dst] * pa * y.abs() / c * ip
    s_x = torch.zeros(n_src, out.size(1), dtype=torch.float64, device=out.device).index_add(0, src, s_m)
    s_p = None
    if p is not None:
        lnc = torch.log(m_abs.clamp(min=LO, max=hi)).abs().clamp(min=1.0)
        lnC = torch.log(M.clamp(min=LO, max=hi)).abs().clamp(min=1.0)
        e_term = torch.zeros_like(out).index_add(0, dst, y.abs() * lnc) * G
        s_p = ((e_term + (g * out.detach()).abs() * lnC / pa ** 2) * ip).sum(0)
    return s_out, s_m, s_x, s_p


FORMS = ("x", "rows", "x_relu", "xa_relu", "xa_relu_frozen")
PS = ("one", "2.5", "0.5", "learn1", "learnF")


@pytest.mark.parametrize("adopted,chunk", [(False, 512), (True, 16), (False, 16)])
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("F", [4, 6, 64, 200])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_op_against_formula(dtype, F, form, adopted, chunk):
    src, dst, n_src, n_dst = _edges(seed=F)
    graph, src, dst = _graph(src, dst, n_src, n_dst, adopted, chunk)
    E = src.numel()
    gen = torch.Generator(device=DEV).manual_seed(F)
    x0 = (torch.randn(n_src, F, device=DEV, generator=gen) * 2).to(dtype)
    a0 = torch.randn(E, F, device=DEV, generator=gen).to(dtype)
    gout = torch.randn(n_dst, F, device=DEV, generator=gen).to(dtype)
    tol = 1e-5 if dtype == torch.float32 else 1.6e-2
    message = "identity" if form in ("x", "rows") else "relu_eps"
    eps = EPS if message == "relu_eps" else 0.0
    for pk in PS:
        for hi in (100.0, None):
            if pk == "one" and hi is None:
                continue
            x = None if form == "rows" else x0.clone().requires_grad_()
            a = None if form in ("x", "x_relu") else a0.clone().requires_grad_(form != "xa_relu_frozen")
            if pk == "one":
                p, pd = 1.0, None
            elif pk in ("2.5", "0.5"):
                p = float(pk)
                pd = torch.tensor([p], dtype=torch.float64, device=DEV)
            else:
                n = 1 if pk == "learn1" else F
                p = (torch.rand(n, device=DEV, generator=gen) * 2.5 + 0.5).to(dtype).requires_grad_()
                pd = p.detach().double().requires_grad_()
            if form == "rows":
                mg = CSRGraph(torch.arange(E, device=DEV), dst, E, n_dst, chunk=chunk)
                out = Fn.power_mean_aggregate(mg, None, a, p, clamp_min=LO, clamp_max=hi)
            else:
                out = Fn.power_mean_aggregate(graph, x, a, p, eps, message, LO, hi)
            xd = None if x is None else x0.double().requires_grad_()
            ad = None if a is None else a0.double().requires_grad_()
            ref, y, M, deg = _formula(xd, ad, pd, src, dst, n_src, n_dst, form, eps, hi, dtype)
            # the message magnitudes per edge
            if form in ("x", "rows"):
                m_abs = (x0.double()[src] if form == "x" else a0.double()).abs()
            else:
                s = x0.double()[src] if form == "x_relu" else (x0.double()[src] + a0.double())
                m_abs = (s.relu() + eps).abs()
            s_out, s_m, s_x, s_p = _sums(ref, y, M, m_abs, deg, pd, src, dst, n_src, gout, hi)
            what = f"{form} p={pk} hi={hi}"
            _check(out, ref, s_out, tol, what + " out")
            out.backward(gout)
            ref.backward(gout.double())
            if x is not None:
                _check(x.grad, xd.grad, s_x, tol, what + " grad_x")
            if a is not None and a.requires_grad:
                _check(a.grad, ad.grad, s_m, tol, what + " grad_a")
            if isinstance(p, torch.Tensor):
                assert p.grad.shape == p.shape and p.grad.dtype == p.dtype
                _check(p.grad, pd.grad, s_p.sum().view(1) if p.numel() == 1 else s_p, tol, what + " grad_p")


def test_empty_rows_give_clamp_min_root():
    src = torch.tensor([0, 1, 2], device=DEV)
    dst = torch.tensor([0, 0, 2], device=DEV)
    g = CSRGraph(src, dst, 3, 4)
    x = torch.rand(3, 8, device=DEV) + 0.5
    out = Fn.power_mean_aggregate(g, x, None, 2.0)
    torch.testing.assert_close(out[1], torch.full((8, ), LO ** 0.5, device=DEV), rtol=1e-5, atol=0)
    torch.testing.assert_close(out[3], torch.full((8, ), LO ** 0.5, device=DEV), rtol=1e-5, atol=0)
    assert torch.equal(Fn.power_mean_aggregate(g, x, None, 1.0)[1], torch.zeros(8, device=DEV))


def _learnable_case():
    src, dst, n_src, n_dst = _edges()
    graph, src, dst = _graph(src, dst, n_src, n_dst, False, 512)
    graph.build_transpose()
    return graph, n_src, src.numel()


def test_one_launch_per_entry_point():
    graph, n_src, E = _learnable_case()
    x = torch.randn(n_src, 64, device=DEV, requires_grad=True)
    a = torch.randn(E, 64, device=DEV)
    p = torch.full((64, ), 2.0, device=DEV, requires_grad=True)
    with _Profile() as prof:
        Fn.power_mean_aggregate(graph, x, a, p, 1e-7, "relu_eps").sum().backward()
    assert {k: prof.calls.get(k, 0) for k in PM} == {"power_mean_csr": 1, "power_mean_backward_dst": 0,
                                                     "power_mean_backward_src": 1}, prof.calls
    a.requires_grad_()
    with _Profile() as prof:
        Fn.power_mean_aggregate(graph, x, a, p, 1e-7, "relu_eps").sum().backward()
    assert {k: prof.calls.get(k, 0) for k in PM} == {"power_mean_csr": 1, "power_mean_backward_dst": 1,
                                                     "power_mean_backward_src": 0}, prof.calls


@pytest.mark.parametrize("trainable_a", [False, True])
def test_no_host_sync_with_learnable_p(trainable_a):
    graph, n_src, E = _learnable_case()
    x = torch.randn(n_src, 64, device=DEV, requires_grad=True)
    a = torch.randn(E, 64, device=DEV, requires_grad=trainable_a)
    p = torch.full((1, ), 1.5, device=DEV, requires_grad=True)
    Fn.power_mean_aggregate(graph, x, a, p, 1e-7, "relu_eps").sum().backward()      # warm: plans' partials
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        Fn.power_mean_aggregate(graph, x, a, p, 1e-7, "relu_eps").sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)


@pytest.mark.parametrize("trainable_a", [False, True])
def test_deterministic(trainable_a):
    src, dst, n_src, n_dst = _edges()
    graph, src, dst = _graph(src, dst, n_src, n_dst, False, 16)
    gen = torch.Generator(device=DEV).manual_seed(5)
    x0 = torch.randn(n_src, 64, device=DEV, generator=gen)
    a0 = torch.randn(src.numel(), 64, device=DEV, generator=gen)
    gout = torch.randn(n_dst, 64, device=DEV, generator=gen)
    runs = []
    for _ in range(2):
        x = x0.clone().requires_grad_()
        a = a0.clone().requires_grad_(trainable_a)
        p = torch.full((64, ), 1.7, device=DEV, requires_grad=True)
        out = Fn.power_mean_aggregate(graph, x, a, p, 1e-7, "relu_eps")
        out.backward(gout)
        runs.append([out, x.grad, p.grad] + ([a.grad] if trainable_a else []))
    for u, v in zip(*runs):
        assert torch.equal(u, v)


def _reference_ops(x, a, src, dst, n_dst, form, p, eps, hi):
    """The reference's op sequence on the CPU: GENConv.message (gen_conv.py:231-239), then PowerMeanAggregation.forward
    (basic.py:279-293) with its scatter mean."""
    from torch_geometric.utils import scatter
    m = x[src] if form == "x" else (x[src] if a is None else x[src] + a).relu() + eps
    if not isinstance(p, (int, float)) or p != 1:
        m = m.clamp(min=LO, max=hi).pow(p)
    out = scatter(m, dst, 0, dim_size=n_dst, reduce="mean")
    if not isinstance(p, (int, float)) or p != 1:
        out = out.clamp(min=LO, max=hi).pow(1. / p)
    return out


@pytest.mark.parametrize("p", [1.0, 2.5, 0.5, "learn"])
@pytest.mark.parametrize("hi", [100.0, None])
@pytest.mark.parametrize("form", ["x", "x_relu", "xa_relu"])
def test_non_finite_against_reference_ops(tg, form, p, hi):
    """+-inf and NaN in x and a against the reference's own ops on the CPU: out, every gradient, NaN positions."""
    torch.manual_seed(1)
    n_src, n_dst, E, F = 20, 12, 120, 8
    src = torch.randint(0, n_src, (E, ))
    dst = torch.randint(0, n_dst - 2, (E, ))
    x = torch.randn(n_src, F) * 3
    a = torch.randn(E, F)
    x[9, 0], x[10, 3], x[11, 5] = float("inf"), float("nan"), -float("inf")
    a[20, 4], a[21, 6], a[22, 7] = float("inf"), float("nan"), -float("inf")
    eps = 1e-7
    aa = a if form == "xa_relu" else None
    pv = torch.tensor([1.3]) if p == "learn" else p
    xr = x.clone().requires_grad_()
    ar = None if aa is None else aa.clone().requires_grad_()
    pr = pv.clone().requires_grad_() if p == "learn" else pv
    want = _reference_ops(xr, ar, src, dst, n_dst, form, pr, eps, hi)
    gout = torch.randn(n_dst, F)
    want.backward(gout)
    for chunk in (2, 512):
        graph = CSRGraph(src.to(DEV), dst.to(DEV), n_src, n_dst, chunk=chunk)
        xg = x.to(DEV).requires_grad_()
        ag = None if aa is None else aa.to(DEV).requires_grad_()
        pg = pv.to(DEV).requires_grad_() if p == "learn" else pv
        got = Fn.power_mean_aggregate(graph, xg, ag, pg, eps, "identity" if form == "x" else "relu_eps", LO, hi)
        got.backward(gout.to(DEV))
        pairs = [(got, want), (xg.grad, xr.grad)] + ([(ag.grad, ar.grad)] if ag is not None else []) + \
            ([(pg.grad, pr.grad)] if p == "learn" else [])
        for k, (u, v) in enumerate(pairs):
            u, v = u.detach().cpu(), v.detach()
            assert torch.equal(u.isnan(), v.isnan()), (k, u, v)
            fin = v.isfinite()
            torch.testing.assert_close(u[fin], v[fin], rtol=1e-4, atol=1e-5)
            assert torch.equal(u[~fin & ~v.isnan()], v[~fin & ~v.isnan()])


@pytest.mark.parametrize("learn,channels,p", [(False, 1, 1.0), (False, 1, 2.5), (True, 1, 1.5), (True, 8, 0.7)])
def test_module_against_reference(tg, learn, channels, p):
    from torch_geometric.nn.aggr import PowerMeanAggregation as RefPM
    torch.manual_seed(channels)
    N, E, F = 40, 600, 8
    index = torch.randint(0, N - 3, (E, ))
    x = torch.randn(E, F).abs() * 3
    g = torch.randn(N, F)
    ref = RefPM(p=p, learn=learn, channels=channels)
    mine = PowerMeanAggregation(p=p, learn=learn, channels=channels).to(DEV)
    assert repr(mine) == repr(ref)
    xr = x.clone().requires_grad_()
    want = ref(xr, index, dim_size=N)
    want.backward(g)
    sidx, order = torch.sort(index, stable=True)
    ptr = torch.zeros(N + 1, dtype=torch.long)
    ptr[1:] = torch.bincount(index, minlength=N).cumsum(0)
    for how in ("index", "ptr", "sorted"):
        if learn:
            mine.p.grad = None
        if how == "index":
            xc = x.to(DEV).requires_grad_()
            got = mine(xc, index.to(DEV), dim_size=N)
        elif how == "ptr":
            xc = x[order].to(DEV).requires_grad_()
            got = mine(xc, ptr=ptr.to(DEV))
        else:
            xc = x[order].to(DEV).requires_grad_()
            got = mine(xc, sidx.to(DEV), dim_size=N, index_sorted=True)
        torch.testing.assert_close(got.cpu(), want.detach(), rtol=1e-4, atol=1e-5)
        got.backward(g.to(DEV))
        gx = xc.grad.cpu() if how == "index" else torch.empty_like(x).index_copy_(0, order, xc.grad.cpu())
        torch.testing.assert_close(gx, xr.grad, rtol=1e-4, atol=1e-5)
        if learn:
            torch.testing.assert_close(mine.p.grad.cpu(), ref.p.grad, rtol=1e-4, atol=1e-5)


@pytest.mark.parametrize("dtype", [torch.float16, torch.float64])
def test_module_other_dtypes_take_the_composed_path(tg, dtype):
    from torch_geometric.nn.aggr import PowerMeanAggregation as RefPM
    torch.manual_seed(2)
    N, E, F = 30, 400, 8
    index = torch.randint(0, N - 2, (E, ))
    x = torch.rand(E, F, dtype=torch.float64) * 2
    want = RefPM(p=2.0)(x.to(dtype), index, dim_size=N)
    got = PowerMeanAggregation(p=2.0)(x.to(DEV, dtype), index.to(DEV), dim_size=N)
    assert got.dtype == want.dtype == dtype
    torch.testing.assert_close(got.cpu().double(), want.double(), rtol=2e-3 if dtype == torch.float16 else 1e-6,
                               atol=2e-3 if dtype == torch.float16 else 1e-8)


def test_module_fp32_p_with_bf16_messages_promotes(tg):
    from torch_geometric.nn.aggr import PowerMeanAggregation as RefPM
    torch.manual_seed(3)
    N, E, F = 30, 400, 8
    index = torch.randint(0, N - 2, (E, ))
    x = (torch.rand(E, F) * 2).to(torch.bfloat16)
    ref = RefPM(p=1.5, learn=True)
    want = ref(x, index, dim_size=N)
    mine = PowerMeanAggregation(p=1.5, learn=True).to(DEV)
    got = mine(x.to(DEV), index.to(DEV), dim_size=N)
    assert got.dtype == want.dtype == torch.float32
    torch.testing.assert_close(got.cpu(), want, rtol=1.6e-2, atol=1e-3)
    got.sum().backward()
    assert mine.p.grad is not None and mine.p.grad.dtype == torch.float32


def test_module_clamp_off_the_fused_path(tg):
    """clamp_min None (bases may be 0 or negative) keeps the reference's ops."""
    from torch_geometric.nn.aggr import PowerMeanAggregation as RefPM
    torch.manual_seed(4)
    N, E, F = 30, 400, 8
    index = torch.randint(0, N - 2, (E, ))
    x = torch.rand(E, F) * 2
    want = RefPM(p=2.0, clamp_min=None, clamp_max=100.)(x, index, dim_size=N)
    got = PowerMeanAggregation(p=2.0, clamp_min=None, clamp_max=100.)(x.to(DEV), index.to(DEV), dim_size=N)
    torch.testing.assert_close(got.cpu(), want, rtol=1e-5, atol=1e-6)


def _gen_pair(tg, kw, seed=0):
    from pytorch_geometric_b200.plugin import conv as PC
    torch.manual_seed(seed)
    ref = tg.nn.GENConv(**kw)
    ours = PC.B200GENConv(**kw)
    ours.load_state_dict(ref.state_dict())
    with torch.no_grad():                                    # learnable t / p away from their initial value
        for m in (ref, ours):
            for n, prm in m.named_parameters():
                if n.endswith(".t") or n.endswith(".p"):
                    prm.fill_(1.3)
    return ref.to(DEV), ours.to(DEV)


GEN_CASES = [
    dict(in_channels=16, out_channels=16, aggr="softmax", learn_t=True, num_layers=2, norm="layer"),
    dict(in_channels=16, out_channels=16, aggr="softmax_sg"),
    dict(in_channels=16, out_channels=16, aggr="powermean", p=2.5),
    dict(in_channels=16, out_channels=16, aggr="powermean", learn_p=True),
    dict(in_channels=8, out_channels=16, aggr="softmax", learn_t=True, edge_dim=4),
    dict(in_channels=16, out_channels=16, aggr="powermean", learn_p=True, msg_norm=True, learn_msg_scale=True),
]


@pytest.mark.parametrize("case", range(len(GEN_CASES)))
def test_gen_conv_against_reference(tg, case):
    kw = GEN_CASES[case]
    ref, ours = _gen_pair(tg, kw, case)
    N, E = 60, 500
    gen = torch.Generator().manual_seed(case)
    ei = torch.randint(0, N, (2, E), generator=gen).to(DEV)
    x = torch.randn(N, kw["in_channels"], generator=gen).to(DEV)
    ea = None
    if "edge_dim" in kw:
        ea = torch.randn(E, kw["edge_dim"], generator=gen).to(DEV)
    elif case in (0, 3):
        ea = torch.randn(E, kw["out_channels"], generator=gen).to(DEV)
    xr, xo = x.clone().requires_grad_(), x.clone().requires_grad_()
    er = eo = None
    if ea is not None:
        er, eo = ea.clone().requires_grad_(), ea.clone().requires_grad_()
    with _Profile() as prof:
        got = ours(xo, ei, eo)
    assert sum(prof.calls.get(k, 0) for k in ("softmax_aggr_csr", "power_mean_csr")) == 1, prof.calls
    want = ref(xr, ei, er)
    torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-5)
    g = torch.randn_like(want)
    want.backward(g)
    got.backward(g)
    torch.testing.assert_close(xo.grad, xr.grad, rtol=1e-4, atol=1e-5)
    if ea is not None:
        torch.testing.assert_close(eo.grad, er.grad, rtol=1e-4, atol=1e-5)
    for (n, pr), (_, po) in zip(ref.named_parameters(), ours.named_parameters()):
        torch.testing.assert_close(po.grad, pr.grad, rtol=1e-4, atol=1e-5, msg=n)


def test_gen_conv_bipartite_and_fall_through(tg):
    from pytorch_geometric_b200.plugin import conv as PC
    kw = dict(in_channels=(8, 12), out_channels=16, aggr="powermean", learn_p=True)
    ref, ours = _gen_pair(tg, kw)
    gen = torch.Generator().manual_seed(7)
    xs = torch.randn(30, 8, generator=gen).to(DEV)
    xd = torch.randn(20, 12, generator=gen).to(DEV)
    ei = torch.stack([torch.randint(0, 30, (200, ), generator=gen), torch.randint(0, 20, (200, ), generator=gen)]).to(DEV)
    torch.testing.assert_close(ours((xs, xd), ei), ref((xs, xd), ei), rtol=1e-4, atol=1e-5)
    for aggr in ("mean", "max"):                                # not fused: the reference's own forward
        torch.manual_seed(0)
        r = tg.nn.GENConv(16, 16, aggr=aggr).to(DEV)
        o = PC.B200GENConv(16, 16, aggr=aggr).to(DEV)
        o.load_state_dict(r.state_dict())
        x = torch.randn(30, 16, device=DEV)
        e2 = torch.randint(0, 30, (2, 100), device=DEV)
        with _Profile() as prof:
            got = o(x, e2)
        assert not any(k in prof.calls for k in ("softmax_aggr_csr", "power_mean_csr"))
        torch.testing.assert_close(got, r(x, e2), rtol=1e-5, atol=1e-6)


def test_memory_of_training_step():
    """N = 400k, E = 4M, F = 64 fp32, x and a both trainable, learnable p: the only [E, F] allocation of a step is
    grad_a."""
    n, e, f = 400_000, 4_000_000, 64
    g = torch.Generator(device=DEV).manual_seed(0)
    src = torch.randint(0, n, (e, ), device=DEV, generator=g)
    dst = (torch.rand(e, device=DEV, generator=g) ** 2 * (n - 1)).long()
    graph = CSRGraph(src, dst, n, n)
    del src, dst
    x = torch.randn(n, f, device=DEV, generator=g).requires_grad_()
    a = torch.randn(e, f, device=DEV, generator=g).requires_grad_()
    p = torch.full((f, ), 1.5, device=DEV).requires_grad_()
    gout = torch.randn(n, f, device=DEV, generator=g)
    one_ef = e * f * 4
    Fn.power_mean_aggregate(graph, x, a, p, 1e-7, "relu_eps").backward(gout)   # warm: transpose, plans' partials
    x.grad = a.grad = p.grad = None
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    m0 = torch.cuda.memory_allocated()
    Fn.power_mean_aggregate(graph, x, a, p, 1e-7, "relu_eps").backward(gout)
    torch.cuda.synchronize()
    step = torch.cuda.max_memory_allocated() - m0 - one_ef                   # grad_a
    assert step < one_ef // 2, (step, one_ef)
