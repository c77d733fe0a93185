"""GPU tests of SplineConv on the engine (csrc/spline.cu):

  * the shim ops `Fn.spline_basis` / `Fn.spline_weighting` against the fp64 restatement in tests/spline_oracle.py,
    forward and every gradient, over degrees 1-3, D = 1-3 with closed dimensions, pseudo exactly 0 and 1, E = 0;
    weight indices bit-exact and every output bit-identical from run to run;
  * `Fn.spline_conv_aggregate` (one CSR sweep into P and one GEMM) against an fp64 formula over sum / mean, fp32 / bf16,
    F_in = 1, GEMM widths the wgmma kernel takes and ones it hands to the library GEMM, the K F_in limit and the
    refusal just past it, a power-law graph with chunked hubs and isolated rows, adopted CSRs and several row blocks;
  * the unmodified reference SplineConv after `plugin.install(layers=True)` against the CPU reference with the
    oracle's ops, the fall-through configurations against the shim-only path, and the mirror against the golden data;
  * step memory: nothing of size E F is kept for the backward.

Bar: |got - want| <= tol * sum|terms| elementwise, tol = 1e-5 for fp32 and 1.6e-2 for bf16 (inputs are rounded to
bf16 first and the formula takes the rounded values).
"""
import copy
import os
import sys

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import spline_oracle as SO  # noqa: E402

from pytorch_geometric_b200 import functional as Fn  # noqa: E402
from pytorch_geometric_b200 import ops  # noqa: E402
from pytorch_geometric_b200.graph import CSRGraph  # noqa: E402

DEV = "cuda"
TOL = {torch.float32: 1e-5, torch.bfloat16: 1.6e-2}


class _Profile:
    def __enter__(self):
        ops.PROFILE.reset(enabled=True)
        return self

    def __exit__(self, *a):
        self.calls = {k: v["calls"] for k, v in ops.PROFILE.summary().items()}
        ops.PROFILE.reset(enabled=False)
        return False


def _check(a, b, s, tol, what):
    a, b, s = (torch.as_tensor(t).detach().double().cpu() for t in (a, b, s))
    bad = (a - b).abs() > tol * s + 1e-30
    assert not bad.any(), f"{what}: {int(bad.sum())} entries off, first at {bad.nonzero()[:3].tolist()}, " \
                          f"max err {(a - b).abs().max().item():.3e}"


def _close(a, b, tol, what):
    a, b = a.detach().double().cpu(), torch.as_tensor(b).detach().double().cpu()
    err = (a - b).abs().max().item() if a.numel() else 0.0
    scale = b.abs().max().item() if b.numel() else 0.0
    assert err <= tol * max(scale, 1e-3), f"{what}: max err {err:.3e} vs scale {scale:.3e}"


def _power_law(n_src, n_dst, e, seed, isolated=8):
    g = torch.Generator().manual_seed(seed)
    src = (torch.rand(e, generator=g) ** 3 * n_src).long().clamp(max=n_src - 1)
    dst = (torch.rand(e, generator=g) ** 4 * (n_dst - isolated)).long().clamp(max=n_dst - isolated - 1)
    return src, dst                                     # the last `isolated` destinations have no in-edges


# ---------------------------------------------------------------------------------------------- shim ops
BASIS_CASES = [(1, [5], [1]), (2, [5], [1]), (3, [7], [1]), (1, [5, 4], [1, 0]), (2, [4, 6], [0, 1]),
               (3, [5, 5], [1, 1]), (1, [3, 4, 5], [1, 0, 1]), (2, [5, 3, 4], [0, 1, 1]), (3, [4, 5, 3], [1, 1, 0])]


def _pseudo(e, d, seed):
    g = torch.Generator().manual_seed(seed)
    p = torch.rand(e, d, generator=g)
    p[:4] = 0.0                                         # exactly 0 and 1: the ends of the open and closed ranges
    p[4:8] = 1.0
    return p


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("degree,ks,op", BASIS_CASES)
def test_basis_against_oracle(dtype, degree, ks, op):
    e = 3000
    p = _pseudo(e, len(ks), seed=degree * 10 + len(ks)).to(dtype)
    kst, opt = torch.tensor(ks), torch.tensor(op, dtype=torch.uint8)
    pg = p.to(DEV).requires_grad_()
    b, wi = Fn.spline_basis(pg, kst.to(DEV), opt.to(DEV), degree)
    gb = torch.randn(b.shape, generator=torch.Generator().manual_seed(3)).to(dtype)
    b.backward(gb.to(DEV))
    want_b, want_wi = SO.spline_basis(p.float().numpy(), ks, op, degree)
    assert wi.dtype == torch.int64 and b.dtype == dtype
    assert np.array_equal(wi.cpu().numpy(), want_wi)                                        # bit-exact indices
    _check(b, want_b, np.ones_like(want_b), TOL[dtype], "basis")
    assert (b.double().sum(1) - 1).abs().max() < (1e-5 if dtype == torch.float32 else 3e-2)  # partition of unity
    want_gp = SO.spline_basis_grad(gb.float().numpy(), p.float().numpy(), ks, op, degree)
    scale = np.abs(gb.float().numpy()).sum(1, keepdims=True) * np.asarray(ks, dtype=np.float64)[None, :] * 4
    _check(pg.grad, want_gp, scale, TOL[dtype], "grad_pseudo")
    b2, wi2 = Fn.spline_basis(pg.detach(), kst.to(DEV), opt.to(DEV), degree, torch.int32)
    assert torch.equal(b2, b.detach()) and torch.equal(wi2.long(), wi)


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("degree,ks,op", [(1, [5, 5], [1, 1]), (2, [4, 6], [0, 1]), (3, [3, 4, 5], [1, 0, 1])])
def test_weighting_against_oracle_and_deterministic(dtype, degree, ks, op):
    e, fi, fo = 2000, 12, 20
    K = int(np.prod(ks))
    g = torch.Generator().manual_seed(7)
    p = _pseudo(e, len(ks), seed=8)
    b, wi = SO.spline_basis(p.numpy(), ks, op, degree)
    x = torch.randn(e, fi, generator=g).to(dtype)
    w = (torch.randn(K, fi, fo, generator=g) / fi ** 0.5).to(dtype)
    bt = torch.from_numpy(b).to(dtype)
    gout = torch.randn(e, fo, generator=g).to(dtype)

    def run():
        xg, wg, bg = (t.to(DEV).requires_grad_() for t in (x, w, bt))
        out = Fn.spline_weighting(xg, wg, bg, torch.from_numpy(wi).to(DEV))
        out.backward(gout.to(DEV))
        return out, xg.grad, wg.grad, bg.grad

    got = run()
    xa, wa, ba, ga = (t.float().numpy() for t in (x, w, bt, gout))
    want = SO.spline_weighting(xa, wa, ba, wi)
    wgx, wgw, wgb = SO.spline_weighting_grads(ga, xa, wa, ba, wi)
    s_out = SO.spline_weighting(np.abs(xa), np.abs(wa), np.abs(ba), wi)
    sx, sw, sb = SO.spline_weighting_grads(np.abs(ga), np.abs(xa), np.abs(wa), np.abs(ba), wi)
    tol = TOL[dtype]
    _check(got[0], want, s_out, tol, "out")
    _check(got[1], wgx, sx, tol, "grad_x")
    _check(got[2], wgw, sw, tol, "grad_weight")
    _check(got[3], wgb, sb, tol, "grad_basis")
    again = run()
    for u, v in zip(got, again):
        assert torch.equal(u, v)


def test_shim_ops_with_no_edges():
    p = torch.empty(0, 2, device=DEV, requires_grad=True)
    b, wi = Fn.spline_basis(p, torch.tensor([5, 5], device=DEV), torch.tensor([1, 1], dtype=torch.uint8, device=DEV), 1)
    assert b.shape == (0, 4) and wi.shape == (0, 4)
    x = torch.randn(0, 3, device=DEV, requires_grad=True)
    w = torch.randn(25, 3, 4, device=DEV, requires_grad=True)
    out = Fn.spline_weighting(x, w, b, wi)
    out.sum().backward()
    assert out.shape == (0, 4) and (w.grad == 0).all() and p.grad.shape == (0, 2)


@pytest.mark.parametrize("kind", ["cpu", "fp16", "fp64"])
def test_shim_ops_refuse_other_devices_and_dtypes(kind):
    dev, dt = ("cpu", torch.float32) if kind == "cpu" else (DEV, {"fp16": torch.float16, "fp64": torch.float64}[kind])
    p = torch.rand(4, 2, device=dev, dtype=dt)
    with pytest.raises(RuntimeError, match="CUDA float32 / bfloat16"):
        Fn.spline_basis(p, torch.tensor([5, 5]), torch.tensor([1, 1], dtype=torch.uint8), 1)
    with pytest.raises(RuntimeError, match="CUDA float32 / bfloat16"):
        Fn.spline_weighting(torch.randn(4, 3, device=dev, dtype=dt), torch.randn(25, 3, 2, device=dev, dtype=dt),
                            torch.rand(4, 4, device=dev, dtype=dt), torch.zeros(4, 4, dtype=torch.long, device=dev))


def test_pseudo_outside_the_unit_interval_stays_in_bounds():
    p = torch.tensor([[-0.3, 1.7], [-2.0, 3.25], [float("inf"), float("nan")]], device=DEV)
    b, wi = Fn.spline_basis(p, torch.tensor([5, 4], device=DEV), torch.tensor([1, 0], dtype=torch.uint8, device=DEV), 2)
    assert wi.min() >= 0 and wi.max() < 20
    want_b, want_wi = SO.spline_basis(p[:2].cpu().numpy(), [5, 4], [1, 0], 2)
    assert np.array_equal(wi[:2].cpu().numpy(), want_wi)


# ---------------------------------------------------------------------------------------------- fused aggregate
def _formula(src, dst, n_src, n_dst, x, basis, wi, w, g, mean):
    """fp64 out, grad_w, grad_basis, grad_x and their sums of |terms|, through the dense P."""
    x, basis, w, g = (torch.as_tensor(t).detach().double().cpu() for t in (x, basis, w, g))
    wi = torch.as_tensor(wi).long().cpu()
    src, dst = src.cpu(), dst.cpu()
    (E, S), (K, Fi, Fo) = basis.shape, w.shape
    xj = x[src]
    onehot = torch.zeros(E, K, dtype=torch.float64)
    onehot_a = torch.zeros(E, K, dtype=torch.float64)
    onehot.scatter_add_(1, wi, basis)
    onehot_a.scatter_add_(1, wi, basis.abs())
    outer = (onehot[:, :, None] * xj[:, None, :]).reshape(E, -1)
    outer_a = (onehot_a[:, :, None] * xj.abs()[:, None, :]).reshape(E, -1)
    inv = 1.0 / torch.bincount(dst, minlength=n_dst).clamp(min=1).double() if mean else torch.ones(n_dst, dtype=torch.float64)
    p = torch.zeros(n_dst, K * Fi, dtype=torch.float64).index_add_(0, dst, outer) * inv[:, None]
    pa = torch.zeros(n_dst, K * Fi, dtype=torch.float64).index_add_(0, dst, outer_a) * inv[:, None]
    w2 = w.reshape(K * Fi, Fo)
    res = {"out": (p @ w2, pa @ w2.abs()), "gw": ((p.T @ g).view(K, Fi, Fo), (pa.T @ g.abs()).view(K, Fi, Fo))}
    dp = ((g @ w2.T) * inv[:, None])[dst].view(E, K, Fi)
    dpa = ((g.abs() @ w2.abs().T) * inv[:, None])[dst].view(E, K, Fi)
    idx = wi[:, :, None].expand(E, S, Fi)
    res["gb"] = ((dp.gather(1, idx) * xj[:, None, :]).sum(2), (dpa.gather(1, idx) * xj.abs()[:, None, :]).sum(2))
    q = (basis[:, :, None] * dp.gather(1, idx)).sum(1)
    qa = (basis.abs()[:, :, None] * dpa.gather(1, idx)).sum(1)
    res["gx"] = (torch.zeros(n_src, Fi, dtype=torch.float64).index_add_(0, src, q),
                 torch.zeros(n_src, Fi, dtype=torch.float64).index_add_(0, src, qa))
    return res


def _operands(e, n_src, dim, ks, fi, fo, dtype, seed, degree=1):
    g = torch.Generator().manual_seed(seed)
    p = torch.rand(e, dim, generator=g)
    b, wi = SO.spline_basis(p.numpy(), [ks] * dim, [1] * dim, degree)
    K = ks ** dim
    x = torch.randn(n_src, fi, generator=g).to(dtype)
    w = (torch.randn(K, fi, fo, generator=g) / (fi * 2) ** 0.5).to(dtype)
    return x, torch.from_numpy(b).to(dtype), torch.from_numpy(wi), w


def _run(graph, x, basis, wi, w, gout, reduce):
    xg, bg, wg = (t.to(DEV).requires_grad_() for t in (x, basis, w))
    out = Fn.spline_conv_aggregate(graph, xg, bg, wi.to(DEV), wg, reduce)
    out.backward(gout.to(DEV, out.dtype))
    return out, xg.grad, bg.grad, wg.grad


# (dim, kernel, F_in, F_out): MNIST's first conv (F_in = 1, K = 25: library GEMM); a P width the wgmma GEMM takes
# (K F_in = 25 * 32 = 800, F_out = 64); FAUST's dim 3 (K F_in = 125 * 16 = 2000); an odd width
SHAPES = [(2, 5, 1, 32), (2, 5, 32, 64), (3, 5, 16, 64), (1, 7, 5, 10)]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("reduce", ["sum", "mean"])
@pytest.mark.parametrize("dim,ks,Fi,Fo", SHAPES)
def test_aggregate_against_fp64_on_power_law_graph(dtype, reduce, dim, ks, Fi, Fo):
    n_src, n_dst, e = 900, 700, 9000
    src, dst = _power_law(n_src, n_dst, e, seed=dim + Fi)
    graph = CSRGraph(src.to(DEV), dst.to(DEV), n_src, n_dst)
    assert graph.plan.n_long > 0                               # hub rows above the chunk
    x, basis, wi, w = _operands(e, n_src, dim, ks, Fi, Fo, dtype, seed=1)
    gout = torch.randn(n_dst, Fo, generator=torch.Generator().manual_seed(2))
    with _Profile() as prof:
        out, gx, gb, gw = _run(graph, x, basis, wi, w, gout, reduce)
    assert prof.calls.get("spline_csr") == 2 and prof.calls.get("spline_backward_dst") == 1
    ref = _formula(src, dst, n_src, n_dst, x, basis, wi, w, gout.to(dtype).float(), reduce == "mean")
    tol = TOL[dtype]
    assert out.dtype == dtype and gx.dtype == dtype and gb.dtype == dtype and gw.dtype == dtype
    _check(out, *ref["out"], tol, "out")
    _check(gw, *ref["gw"], tol, "grad_weight")
    _check(gb, *ref["gb"], tol, "grad_basis")
    _check(gx, *ref["gx"], tol, "grad_x")
    assert (out[-8:] == 0).all()                               # isolated destinations


@pytest.mark.parametrize("idx", [torch.int32, torch.int64])
def test_adopted_csr_and_index_dtypes(idx):
    n, e, Fi, Fo = 300, 2500, 16, 64
    src, dst = _power_law(n, n, e, seed=5, isolated=3)
    order = torch.argsort(dst, stable=True)
    src, dst = src[order], dst[order]
    rowptr = torch.zeros(n + 1, dtype=torch.long)
    rowptr[1:] = torch.cumsum(torch.bincount(dst, minlength=n), 0)
    graph = CSRGraph.from_csr(rowptr.to(DEV), src.to(DEV), n, idx_dtype=idx)
    assert graph.perm is None
    x, basis, wi, w = _operands(e, n, 2, 4, Fi, Fo, torch.float32, seed=6, degree=2)
    gout = torch.randn(n, Fo, generator=torch.Generator().manual_seed(7))
    out, gx, gb, gw = _run(graph, x, basis, wi, w, gout, "mean")
    ref = _formula(src, dst, n, n, x, basis, wi, w, gout, True)
    for name, got in (("out", out), ("gw", gw), ("gb", gb), ("gx", gx)):
        _check(got, *ref[name], 1e-5, name)


def test_aggregate_with_no_edges():
    n, Fi, Fo = 50, 8, 16
    graph = CSRGraph(torch.empty(0, dtype=torch.long, device=DEV), torch.empty(0, dtype=torch.long, device=DEV), n, n)
    x, basis, wi, w = _operands(0, n, 2, 5, Fi, Fo, torch.float32, seed=8)
    out, gx, gb, gw = _run(graph, x, basis, wi, w, torch.randn(n, Fo), "sum")
    assert out.shape == (n, Fo) and (out == 0).all()
    assert (gx == 0).all() and gb.shape == (0, 4) and (gw == 0).all()


@pytest.mark.parametrize("dim,ks,Fi,Fo", [(2, 5, 32, 64), (1, 7, 5, 10)])
def test_deterministic_and_blocked(monkeypatch, dim, ks, Fi, Fo):
    """Two runs are bit-identical; with the block cap lowered so that P spans at least 3 blocks, the output is
    bit-identical to the one-block run where the wgmma GEMM runs, and within the bar elsewhere."""
    n_src, n_dst, e = 800, 600, 8000
    src, dst = _power_law(n_src, n_dst, e, seed=11)
    graph = CSRGraph(src.to(DEV), dst.to(DEV), n_src, n_dst)
    x, basis, wi, w = _operands(e, n_src, dim, ks, Fi, Fo, torch.float32, seed=12)
    gout = torch.randn(n_dst, Fo, generator=torch.Generator().manual_seed(13))
    a = _run(graph, x, basis, wi, w, gout, "sum")
    b = _run(graph, x, basis, wi, w, gout, "sum")
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    width = ks ** dim * Fi
    monkeypatch.setattr(Fn, "SPLINE_BLOCK_BYTES", 4 * width * 250)
    assert len(Fn._spline_blocks(n_dst, width)) >= 3
    c = _run(graph, x, basis, wi, w, gout, "sum")
    ref = _formula(src, dst, n_src, n_dst, x, basis, wi, w, gout, False)
    if width % 32 == 0 and Fo == 64:
        assert torch.equal(c[0], a[0])
    for got, name in zip(c, ("out", "gx", "gb", "gw")):
        _check(got, *ref[name], 1e-5, "blocked " + name)


def test_width_limit_and_just_past_it():
    """K F_in = 16384 is the largest P row the sweeps take (64 KiB in shared memory); one more channel is refused with
    B200MP_ERR_UNSUPPORTED, and the layer then falls through to the shim ops."""
    K, Fi, Fo = 256, 64, 32
    assert ops.spline_supported(K, Fi, 4, torch.float32) and not ops.spline_supported(K, Fi + 1, 4, torch.float32)
    n, e = 120, 600
    src, dst = _power_law(n, n, e, seed=17, isolated=2)
    graph = CSRGraph(src.to(DEV), dst.to(DEV), n, n)
    x, basis, wi, w = _operands(e, n, 2, 16, Fi, Fo, torch.float32, seed=18)
    gout = torch.randn(n, Fo, generator=torch.Generator().manual_seed(19))
    got = _run(graph, x, basis, wi, w, gout, "mean")
    ref = _formula(src, dst, n, n, x, basis, wi, w, gout, True)
    for t, name in zip(got, ("out", "gx", "gb", "gw")):
        _check(t, *ref[name], 1e-5, name)
    x2 = torch.randn(n, Fi + 1, device=DEV)
    with pytest.raises(ValueError, match="does not take"):
        Fn.spline_conv_aggregate(graph, x2, basis.to(DEV), wi.to(DEV), torch.randn(K, Fi + 1, Fo, device=DEV))
    with pytest.raises(Exception, match="code -2"):
        ops.spline_csr(graph.rowptr, graph.col, graph.perm, x2, basis.to(DEV), wi.to(DEV, torch.int32), K, 0, n)


# ---------------------------------------------------------------------------------------------- the plug-in layer
@pytest.fixture
def tg_installed(tg):
    from pytorch_geometric_b200 import plugin
    plugin.install(layers=True)
    yield tg
    plugin.uninstall()


@pytest.mark.parametrize("aggr,bip,dim,degree", [("add", False, 3, 1), ("mean", True, 2, 2), ("mean", False, 2, 3)])
def test_reference_layer_reaches_the_fused_path(tg_installed, aggr, bip, dim, degree):
    tg = tg_installed
    from pytorch_geometric_b200.plugin import conv as PC
    n, e, fi, fo = 400, 5000, 16, 32
    src, dst = _power_law(n, n, e, seed=22)
    ei = torch.stack([src, dst])
    x = torch.randn(n, fi)
    ea = torch.rand(e, dim)
    ch = (fi, 12) if bip else fi
    x_dst = torch.randn(n, 12) if bip else None
    torch.manual_seed(21)
    mine = tg.nn.SplineConv(ch, fo, dim, kernel_size=5, degree=degree, aggr=aggr)
    assert type(mine) is PC.B200SplineConv
    with torch.no_grad():
        mine.bias.normal_()
    import torch_geometric.nn.conv.spline_conv as S
    ref = _shim_only(mine)                               # the reference's forward on the CPU, with the oracle's ops
    xc, ec = x.clone().requires_grad_(), ea.clone().requires_grad_()
    saved = S.spline_basis, S.spline_weighting
    S.spline_basis, S.spline_weighting = SO.torch_spline_basis, SO.torch_spline_weighting
    try:
        want = ref(xc if x_dst is None else (xc, x_dst), ei, ec)
    finally:
        S.spline_basis, S.spline_weighting = saved
    gout = torch.randn_like(want)
    want.backward(gout)
    mine = mine.to(DEV)
    xg, eg = x.to(DEV).requires_grad_(), ea.to(DEV).requires_grad_()
    with _Profile() as prof:
        got = mine(xg if x_dst is None else (xg, x_dst.to(DEV)), ei.to(DEV), eg)
        got.backward(gout.to(DEV))
    assert prof.calls.get("spline_csr") and prof.calls.get("spline_backward_dst") and prof.calls.get("spline_basis")
    assert not prof.calls.get("spline_weighting")
    _close(got, want, 1e-4, "out")
    _close(xg.grad, xc.grad, 1e-4, "grad_x")
    _close(eg.grad, ec.grad, 1e-4, "grad_edge_attr")
    for (name, pg), (_, pc) in zip(mine.named_parameters(), ref.named_parameters()):
        _close(pg.grad, pc.grad, 1e-4, name)


def _shim_only(module):
    """The same module run by the reference's own forward (message = the shim ops, then its aggregation)."""
    m = copy.deepcopy(module)
    m.__class__ = type(module).__mro__[1]
    return m


FALL_THROUGH = ["max", "sparse", "hook", "autocast", "decomposed"]


def _dyadic(shape, g, scale):
    """Entries in {0, +-scale}."""
    return (torch.randint(-1, 2, shape, generator=g) * scale).float()


@pytest.mark.parametrize("kind", FALL_THROUGH)
def test_fall_through_configurations(tg_installed, kind):
    """Max aggregation, a torch.sparse adjacency, a message hook, torch.autocast and decomposed layers run the
    reference's forward -- its message through the shim ops -- and give exactly what the reference's own forward gives
    with the same ops (or raise the same error); no fused sweep runs.  Inputs are dyadic (x, weights in {0, +-1/2^k},
    pseudo-coordinates in multiples of 1/8 at kernel size 5, so every basis value is 0, 1/2 or 1): every sum is exact,
    whatever order the reference's scatter adds in."""
    tg = tg_installed
    n, e, fi, fo, dim = 60, 400, 4, 6, 2
    g = torch.Generator().manual_seed(33)
    src, dst = _power_law(n, n, e, seed=31, isolated=2)
    key = torch.unique(dst * n + src)                    # unique edges sorted by (dst, src): a coalesced adj_t's order
    ei = torch.stack([key % n, key // n]).to(DEV)
    x = _dyadic((n, fi), g, 1.0).to(DEV)
    ea = (torch.randint(0, 9, (ei.size(1), dim), generator=g) / 8.0).to(DEV)
    kw = {"aggr": "max"} if kind == "max" else {}
    if kind == "decomposed":
        kw["decomposed_layers"] = 2
    mine = tg.nn.SplineConv(fi, fo, dim, kernel_size=5, **kw)
    with torch.no_grad():
        for p in mine.parameters():
            p.copy_(_dyadic(tuple(p.shape), g, 0.5))
    mine = mine.to(DEV)
    if kind == "hook":
        mine.register_message_forward_hook(lambda mod, inp, out: out)
    ref = _shim_only(mine)

    def call(module):
        if kind == "sparse":
            adj = tg.utils.to_torch_coo_tensor(ei, size=(n, n)).transpose(0, 1).coalesce()
            return module(x, adj, ea)
        if kind == "autocast":
            with torch.autocast("cuda", dtype=torch.bfloat16):
                return module(x, ei, ea)
        return module(x, ei, ea)

    if kind == "decomposed":
        # the reference's decomposed propagate does not take SplineConv's (x, x) pair: both raise the same error
        with _Profile() as prof:
            with pytest.raises(Exception) as a:
                call(mine)
        with pytest.raises(Exception) as b:
            call(ref)
        assert type(a.value) is type(b.value) and str(a.value) == str(b.value)
        assert not prof.calls.get("spline_csr")
        return
    with _Profile() as prof:
        got = call(mine)
    assert not prof.calls.get("spline_csr"), (kind, prof.calls)
    assert prof.calls.get("spline_weighting"), (kind, prof.calls)
    want = call(ref)
    assert got.dtype == want.dtype
    assert torch.equal(got, want), (kind, (got.double() - want.double()).abs().max().item())


def test_training_step_memory_keeps_no_edge_sized_tensor(tg_installed):
    tg = tg_installed
    n, e, f = 20_000, 400_000, 64
    g = torch.Generator(device=DEV).manual_seed(31)
    ei = torch.stack([torch.randint(0, n, (e, ), device=DEV, generator=g),
                      (torch.rand(e, device=DEV, generator=g) ** 2 * (n - 1)).long()])
    x = torch.randn(n, f, device=DEV, generator=g).requires_grad_()
    ea = torch.rand(e, 2, device=DEV, generator=g)
    conv = tg.nn.SplineConv(f, f, 2, kernel_size=5, aggr="add").to(DEV)
    conv(x, ei, ea).sum().backward()                                      # graph build and warm-up
    torch.cuda.synchronize()
    base = torch.cuda.memory_allocated()
    out = conv(x, ei, ea)
    kept = torch.cuda.memory_allocated() - base - out.numel() * 4         # what autograd holds for the backward
    out.sum().backward()
    torch.cuda.synchronize()
    # x, weight, edge_attr, basis [E, 4] and int32 wi [E, 4]: no [E, F] message or gathered x_j
    assert kept < e * f * 4 / 2, kept


# ---------------------------------------------------------------------------------------------- golden data
GOLDEN = [("faust_add", 8, 8, 3, {"kernel_size": 5, "aggr": "add"}),
          ("mnist_mean", 1, 16, 2, {"kernel_size": 5, "aggr": "mean"}),
          ("deg2_mixed", 6, 4, 2, {"kernel_size": [3, 4], "is_open_spline": [True, False], "degree": 2}),
          ("bipartite", (8, 16), 8, 2, {"kernel_size": 3, "aggr": "add"}),
          ("no_root_no_bias", 4, 8, 2, {"kernel_size": 4, "root_weight": False, "bias": False}),
          ("deg3_isolated", 4, 6, 1, {"kernel_size": 6, "degree": 3, "aggr": "mean"})]


@pytest.mark.parametrize("tag,ch,f_out,dim,kw", GOLDEN)
def test_mirror_matches_golden(golden, tag, ch, f_out, dim, kw):
    from pytorch_geometric_b200.nn import SplineConv
    z = golden("spline")
    mine = SplineConv(ch, f_out, dim, **kw)
    mine.load_state_dict({key[len(tag) + 3:]: torch.from_numpy(v) for key, v in z.items() if key.startswith(f"{tag}_p_")})
    mine = mine.to(DEV)
    x = torch.from_numpy(z[f"{tag}_x"]).to(DEV).requires_grad_()
    ea = torch.from_numpy(z[f"{tag}_ea"]).to(DEV).requires_grad_()
    x_dst = torch.from_numpy(z[f"{tag}_x_dst"]).to(DEV).requires_grad_() if f"{tag}_x_dst" in z else None
    ei = torch.from_numpy(z[f"{tag}_ei"]).to(DEV)
    if x_dst is None:
        out = mine(x, ei, ea)
    else:
        out = mine((x, x_dst), ei, ea, size=(x.size(0), x_dst.size(0)))
    out.backward(torch.from_numpy(z[f"{tag}_gout"]).to(DEV))
    _close(out, torch.from_numpy(z[f"{tag}_out"]), 1e-5, "out")
    _close(x.grad, torch.from_numpy(z[f"{tag}_gx"]), 1e-5, "grad_x")
    _close(ea.grad, torch.from_numpy(z[f"{tag}_gea"]), 1e-4, "grad_edge_attr")
    if x_dst is not None:
        _close(x_dst.grad, torch.from_numpy(z[f"{tag}_gx_dst"]), 1e-5, "grad_x_dst")
    for name, p in mine.named_parameters():
        _close(p.grad, torch.from_numpy(z[f"{tag}_g_{name}"]), 1e-5, "grad " + name)


def test_golden_through_the_plugged_reference(tg_installed, golden):
    """The unmodified reference SplineConv after install() (fused path) reproduces the golden data too."""
    tg = tg_installed
    z = golden("spline")
    tag, ch, f_out, dim, kw = GOLDEN[0]
    conv = tg.nn.SplineConv(ch, f_out, dim, **kw)
    conv.load_state_dict({key[len(tag) + 3:]: torch.from_numpy(v) for key, v in z.items() if key.startswith(f"{tag}_p_")})
    conv = conv.to(DEV)
    out = conv(torch.from_numpy(z[f"{tag}_x"]).to(DEV), torch.from_numpy(z[f"{tag}_ei"]).to(DEV),
               torch.from_numpy(z[f"{tag}_ea"]).to(DEV))
    _close(out, torch.from_numpy(z[f"{tag}_out"]), 1e-5, "out")
