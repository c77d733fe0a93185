"""GPU tests of the online-softmax aggregation (csrc/softmax_aggr.cu, functional.softmax_aggregate, nn.aggr.
SoftmaxAggregation):

  * the op against an fp64 formula for out, grad_x, grad_a and grad_t -- fp32 / bf16, widths on the vector and the
    scalar path, the message forms (x only, edge rows only, relu(x) + eps, relu(x + a) + eps with a trainable or
    frozen, which selects the grad_x route), t as the number 1, as 0.5 and learnable with 1 or F channels, with and
    without semi_grad, adopted and sorted CSRs, and a small chunk so hub rows take the combine kernels on both sides;
  * one launch per entry point, and no device->host sync with a learnable t;
  * non-finite inputs (+-inf and NaN in x and a, t = 0, negative t, a row whose z are all -inf, a -inf in a row's
    first slot) against the reference's own ops;
  * SoftmaxAggregation with ptr, sorted and unsorted index, non-finite messages, against the reference module, and
    the composed path it keeps for fp16 / fp64 messages and for an fp32 t with bf16 messages;
  * the memory of a training step at N = 400k, E = 4M, F = 64.

The formula rounds s, m and z to the storage dtype where the reference materialises them (straight-through for the
gradient), so the bf16 bar covers the kernel's fp32 softmax and the bf16 outputs.
"""
import pytest
import torch

pytestmark = pytest.mark.gpu

from pytorch_geometric_b200 import functional as Fn  # noqa: E402
from pytorch_geometric_b200 import ops  # noqa: E402
from pytorch_geometric_b200.graph import CSRGraph  # noqa: E402
from pytorch_geometric_b200.nn import SoftmaxAggregation  # noqa: E402

DEV = "cuda"
EPS = 1e-7
SM = ("softmax_aggr_csr", "softmax_aggr_backward_dst", "softmax_aggr_backward_src")


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


def _formula(x, a, t, src, dst, n_src, n_dst, form, eps, semi, dtype, gout):
    """fp64 out with autograd (x, a, t: fp64 leaves holding the storage-dtype values), and the sums of |terms| of out,
    of each message's gradient, of grad_x and of grad_t per channel."""
    def rnd(v):
        return v if dtype == torch.float32 else v + (v.to(dtype).double() - v).detach()

    if form in ("x", "rows"):
        m = x[src] if form == "x" else a
    else:
        s = x[src] if form == "x_relu" else rnd(x[src] + a)
        m = rnd(s.relu() + eps)
    z = m if t is None else rnd(m * t)
    F = m.size(1)
    idx = dst.view(-1, 1).expand(-1, F)
    M = torch.full((n_dst, F), -float("inf"), dtype=torch.float64, device=m.device)
    M = M.scatter_reduce(0, idx, z.detach(), "amax")
    w = z if not semi else z.detach()
    ex = (w - M[dst]).exp()
    S = torch.zeros(n_dst, F, dtype=torch.float64, device=m.device).index_add(0, dst, ex) + 1e-16
    p = ex / S[dst]
    out = torch.zeros(n_dst, F, dtype=torch.float64, device=m.device).index_add(0, dst, p * m)
    pd, ma, g = p.detach(), m.detach().abs(), gout.double()[dst].abs()
    s_out = torch.zeros_like(out).index_add(0, dst, pd * ma)
    ta = 1.0 if t is None else t.detach().abs()
    s_m = g * pd if semi else g * pd * (1 + ta * (ma + s_out[dst]))
    s_x = torch.zeros(n_src, F, dtype=torch.float64, device=m.device).index_add(0, src, s_m)
    s_t = (g * pd * ma * (ma + s_out[dst])).sum(0)
    return out, s_out.detach(), s_m, s_x, s_t


FORMS = ("x", "rows", "x_relu", "xa_relu", "xa_relu_frozen")
TS = (("one", False), ("half", False), ("one", True), ("half", True), ("learn1", False), ("learnF", False))


@pytest.mark.parametrize("adopted,chunk", [(False, 512), (True, 16), (False, 16)])
@pytest.mark.parametrize("form", FORMS)
@pytest.mark.parametrize("F", [4, 6, 64, 128, 200, 256])
@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
def test_op_against_formula(dtype, F, form, adopted, chunk):
    src, dst, n_src, n_dst = _edges(seed=F)
    graph, src, dst = _graph(src, dst, n_src, n_dst, adopted, chunk)
    E = src.numel()
    gen = torch.Generator(device=DEV).manual_seed(F)
    x0 = torch.randn(n_src, F, device=DEV, generator=gen).to(dtype)
    a0 = torch.randn(E, F, device=DEV, generator=gen).to(dtype)
    gout = torch.randn(n_dst, F, device=DEV, generator=gen).to(dtype)
    tol = 1e-5 if dtype == torch.float32 else 1.6e-2
    message = "identity" if form in ("x", "rows") else "relu_eps"
    eps = EPS if message == "relu_eps" else 0.0
    for tk, semi in TS:
        x = None if form == "rows" else x0.clone().requires_grad_()
        a = None if form in ("x", "x_relu") else a0.clone().requires_grad_(form != "xa_relu_frozen")
        if tk == "one":
            t, td = 1.0, None
        elif tk == "half":
            t, td = 0.5, torch.tensor([0.5], dtype=torch.float64, device=DEV)
        else:
            n = 1 if tk == "learn1" else F
            t = (torch.rand(n, device=DEV, generator=gen) * 2 + 0.25).to(dtype).requires_grad_()
            td = t.detach().double().requires_grad_()
        if form == "rows":
            # a message matrix in the caller's order: the CSR over the messages themselves (nn.aggr's unsorted path)
            mg = CSRGraph(torch.arange(E, device=DEV), dst, E, n_dst, chunk=chunk)
            out = Fn.softmax_aggregate(mg, None, a, t, semi_grad=semi)
        else:
            out = Fn.softmax_aggregate(graph, x, a, t, eps, message, semi)
        xd = None if x is None else x0.double().requires_grad_()
        ad = None if a is None else a0.double().requires_grad_()
        ref, s_out, s_m, s_x, s_t = _formula(xd, ad, td, src, dst, n_src, n_dst, form, eps, semi, dtype, gout)
        what = f"{form} t={tk} semi={semi}"
        _check(out, ref, s_out, tol, what + " out")
        out.backward(gout)
        ref.backward(gout.double())
        if x is not None:
            _check(x.grad, xd.grad, s_x, tol, what + " grad_x")
        if a is not None and a.requires_grad:
            _check(a.grad, ad.grad, s_m, tol, what + " grad_a")
        if isinstance(t, torch.Tensor):
            assert t.grad.shape == t.shape and t.grad.dtype == t.dtype
            _check(t.grad, td.grad, s_t.sum().view(1) if t.numel() == 1 else s_t, tol, what + " grad_t")


def test_one_launch_per_entry_point():
    src, dst, n_src, n_dst = _edges()
    graph, src, dst = _graph(src, dst, n_src, n_dst, False, 512)
    x = torch.randn(n_src, 64, device=DEV, requires_grad=True)
    a = torch.randn(src.numel(), 64, device=DEV)
    t = torch.ones(64, device=DEV, requires_grad=True)
    graph.build_transpose()
    with _Profile() as p:
        Fn.softmax_aggregate(graph, x, a, t, 1e-7, "relu_eps").sum().backward()
    assert {k: p.calls.get(k, 0) for k in SM} == {k: 1 for k in SM}, p.calls


def test_no_host_sync_with_learnable_t():
    src, dst, n_src, n_dst = _edges()
    graph, src, dst = _graph(src, dst, n_src, n_dst, False, 512)
    graph.build_transpose()
    x = torch.randn(n_src, 64, device=DEV, requires_grad=True)
    a = torch.randn(src.numel(), 64, device=DEV, requires_grad=True)
    t = torch.ones(1, device=DEV, requires_grad=True)
    Fn.softmax_aggregate(graph, x, a, t, 1e-7, "relu_eps").sum().backward()      # warm: plans' partials
    torch.cuda.synchronize()
    torch.cuda.set_sync_debug_mode("error")
    try:
        Fn.softmax_aggregate(graph, x, a, t, 1e-7, "relu_eps").sum().backward()
    finally:
        torch.cuda.set_sync_debug_mode(0)


@pytest.mark.parametrize("learn,channels,semi", [(False, 1, False), (False, 1, True), (True, 1, False), (True, 8, False)])
def test_module_against_reference(tg, learn, channels, semi):
    from torch_geometric.nn.aggr import SoftmaxAggregation as RefSoftmax
    torch.manual_seed(channels)
    N, E, F = 40, 600, 8
    index = torch.randint(0, N - 3, (E, ))
    index[:5] = 1
    x = torch.randn(E, F)
    x[3, 2], x[4, 5], x[10, 1] = float("inf"), float("nan"), -float("inf")    # rows 1 and the row of edge 10
    ref = RefSoftmax(t=0.7, learn=learn, semi_grad=semi, channels=channels)
    mine = SoftmaxAggregation(t=0.7, learn=learn, semi_grad=semi, channels=channels).to(DEV)
    assert repr(mine) == repr(ref)
    want = ref(x, index, dim_size=N)
    sidx, order = torch.sort(index, stable=True)
    ptr = torch.zeros(N + 1, dtype=torch.long)
    ptr[1:] = torch.bincount(index, minlength=N).cumsum(0)
    for got in (mine(x.to(DEV), index.to(DEV), dim_size=N),
                mine(x[order].to(DEV), ptr=ptr.to(DEV)),
                mine(x[order].to(DEV), sidx.to(DEV), dim_size=N, index_sorted=True)):
        got = got.cpu()
        assert torch.equal(got.isnan(), want.isnan())
        fin = want.isfinite()
        torch.testing.assert_close(got[fin], want[fin], rtol=1e-5, atol=1e-6)
        torch.testing.assert_close(got[~fin & ~want.isnan()], want[~fin & ~want.isnan()])


def test_module_gradients_against_reference(tg):
    from torch_geometric.nn.aggr import SoftmaxAggregation as RefSoftmax
    torch.manual_seed(0)
    N, E, F = 50, 900, 16
    index = torch.randint(0, N - 2, (E, ))
    x = torch.randn(E, F, requires_grad=True)
    g = torch.randn(N, F)
    ref = RefSoftmax(t=0.3, learn=True, channels=F)
    mine = SoftmaxAggregation(t=0.3, learn=True, channels=F).to(DEV)
    ref(x, index, dim_size=N).backward(g)
    xc = x.detach().to(DEV).requires_grad_()
    mine(xc, index.to(DEV), dim_size=N).backward(g.to(DEV))
    torch.testing.assert_close(xc.grad.cpu(), x.grad, rtol=1e-4, atol=1e-5)
    torch.testing.assert_close(mine.t.grad.cpu(), ref.t.grad, rtol=1e-4, atol=1e-5)


def _reference_ops(tg, x, a, src, dst, n_dst, form, t, eps):
    """The reference's op sequence on the CPU: GENConv.message (gen_conv.py:231-239), then SoftmaxAggregation.forward
    (basic.py:196-215) with its softmax and scatter."""
    from torch_geometric.utils import scatter, softmax
    if form == "x":
        m = x[src]
    else:
        m = (x[src] if a is None else x[src] + a).relu() + eps
    z = m if t == 1 else m * t
    return scatter(m * softmax(z, dst, num_nodes=n_dst), dst, 0, dim_size=n_dst, reduce="sum")


@pytest.mark.parametrize("t", [1.0, 0.0, -1.5, 0.7])
@pytest.mark.parametrize("form", ["x", "x_relu", "xa_relu"])
def test_non_finite_against_reference_ops(tg, form, t):
    """+-inf and NaN in x and a, t = 0 and negative t, a row whose z are all -inf, and (t < 0) a row whose FIRST CSR
    slot has z = -inf from an fp32 overflow of t * m before finite ones, against the reference's own ops."""
    torch.manual_seed(1)
    n_src, n_dst, E, F = 20, 12, 120, 8
    src = torch.randint(0, n_src, (E, ))
    dst = torch.randint(0, n_dst - 2, (E, ))
    dst[:4] = n_dst - 2                                   # a row of 4 edges whose z are all -inf (identity form)
    src[:4] = torch.tensor([0, 1, 2, 3])
    dst[4:8] = n_dst - 1                                   # first slot -inf, then finite
    src[4:8] = torch.tensor([4, 5, 6, 7])
    x = torch.randn(n_src, F)
    a = torch.randn(E, F)
    x[0:4, 1] = -float("inf")
    src[8:][src[8:] == 4] = 5                              # source 4 feeds edge 4 only
    x[4, 2] = 2.5e38                                       # t < 0: z overflows to -inf while m is finite
    x[9, 0], x[10, 3], x[11, 5] = float("inf"), float("nan"), -float("inf")
    a[20, 4], a[21, 6], a[22, 7] = float("inf"), float("nan"), -float("inf")
    eps = 1e-7
    aa = a if form == "xa_relu" else None
    want = _reference_ops(tg, x, aa, src, dst, n_dst, form, t, eps)
    graph = CSRGraph(src.to(DEV), dst.to(DEV), n_src, n_dst, chunk=2)   # chunk 2: the combine kernel merges parts too
    for g in (graph, CSRGraph(src.to(DEV), dst.to(DEV), n_src, n_dst)):
        got = Fn.softmax_aggregate(g, x.to(DEV), None if aa is None else aa.to(DEV), t, eps,
                                   "identity" if form == "x" else "relu_eps").cpu()
        assert torch.equal(got.isnan(), want.isnan()), (got, want)
        fin = want.isfinite()
        torch.testing.assert_close(got[fin], want[fin], rtol=1e-5, atol=1e-6)
        assert torch.equal(got[~fin & ~want.isnan()], want[~fin & ~want.isnan()])
    if t < 0:
        assert want[n_dst - 1, 2].isfinite()
    if form == "x":
        assert want[n_dst - 2, 1].isnan()


@pytest.mark.parametrize("dtype", [torch.float16, torch.float64])
def test_module_other_dtypes_take_the_composed_path(tg, dtype):
    """fp16 and fp64 messages are not the sweep's: the module composes the reference's ops on the engine's softmax and
    scatter as before."""
    from torch_geometric.nn.aggr import SoftmaxAggregation as RefSoftmax
    torch.manual_seed(2)
    N, E, F = 30, 400, 8
    index = torch.randint(0, N - 2, (E, ))
    x = torch.randn(E, F, dtype=torch.float64)
    want = RefSoftmax(t=0.5)(x, index, dim_size=N)
    got = SoftmaxAggregation(t=0.5)(x.to(DEV, dtype), index.to(DEV), dim_size=N)
    assert got.dtype == torch.promote_types(dtype, torch.float32)         # the engine's softmax computes in fp32
    torch.testing.assert_close(got.cpu().double(), want, rtol=2e-3 if dtype == torch.float16 else 1e-5, atol=2e-3)


def test_module_fp32_t_with_bf16_messages_promotes(tg):
    """learn=True keeps t in fp32; with bf16 messages x * t promotes to fp32, as in the reference, so the module takes
    the composed path and returns fp32."""
    from torch_geometric.nn.aggr import SoftmaxAggregation as RefSoftmax
    torch.manual_seed(3)
    N, E, F = 30, 400, 8
    index = torch.randint(0, N - 2, (E, ))
    x = torch.randn(E, F).to(torch.bfloat16)
    ref = RefSoftmax(t=0.5, learn=True)
    want = ref(x, index, dim_size=N)
    mine = SoftmaxAggregation(t=0.5, learn=True).to(DEV)
    got = mine(x.to(DEV), index.to(DEV), dim_size=N)
    assert got.dtype == want.dtype == torch.float32
    torch.testing.assert_close(got.cpu(), want, rtol=1.6e-2, atol=1e-3)
    got.sum().backward()
    assert mine.t.grad is not None and mine.t.grad.dtype == torch.float32


def test_memory_of_training_step():
    """N = 400k, E = 4M, F = 64 fp32, x and a both trainable: the only [E, F] allocation of a step is grad_a."""
    n, e, f = 400_000, 4_000_000, 64
    g = torch.Generator(device=DEV).manual_seed(0)
    src = torch.randint(0, n, (e, ), device=DEV, generator=g)
    dst = (torch.rand(e, device=DEV, generator=g) ** 2 * (n - 1)).long()
    graph = CSRGraph(src, dst, n, n)
    del src, dst
    x = torch.randn(n, f, device=DEV, generator=g).requires_grad_()
    a = torch.randn(e, f, device=DEV, generator=g).requires_grad_()
    t = torch.ones(f, device=DEV).requires_grad_()
    gout = torch.randn(n, f, device=DEV, generator=g)
    one_ef = e * f * 4
    Fn.softmax_aggregate(graph, x, a, t, 1e-7, "relu_eps").backward(gout)   # warm: transpose, plans' partials
    x.grad = a.grad = t.grad = None
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    m0 = torch.cuda.memory_allocated()
    Fn.softmax_aggregate(graph, x, a, t, 1e-7, "relu_eps").backward(gout)
    torch.cuda.synchronize()
    step = torch.cuda.max_memory_allocated() - m0 - one_ef                   # grad_a
    assert step < one_ef // 2, (step, one_ef)
