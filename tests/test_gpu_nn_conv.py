"""GPU tests of NNConv's edge-conditioned message fused into one CSR sweep into P and one GEMM (nn_conv.py:96-122):

  * `Fn.nn_conv_aggregate` against an fp64 formula -- forward and the gradients of x, h and W' -- over sum / mean,
    fp32 / bf16, F_in = 1 (MNIST's first conv), a P width the wgmma GEMM takes and ones it rejects, a power-law graph
    whose hub rows exceed the plan's chunk with isolated destinations, adopted and sorted CSRs, and E = 0;
  * determinism, and destination-row blocking (P over at least 3 blocks) against the one-block run;
  * unmodified reference NNConv and ECConv under `plugin.install(layers=True)`: the new kernels run, the output and
    every gradient match the CPU reference, and a training step at E = 200k, F_in = F_out = 64 stays below the size of
    one [E, F_in F_out] fp32 tensor; the configurations that must fall through (autocast and torch.sparse included)
    give exactly the reference's result or error;
  * the standalone `nn.NNConv` against the reference's golden vectors (tests/golden/nn_conv.npz).

Bar: |got - want| <= tol * sum|terms| elementwise, tol = 1e-5 for fp32 and 1.6e-2 for bf16 (x and h are rounded to
bf16 as inputs; the formula takes the rounded values, so the bar covers the fp32 sums, the 3xTF32 GEMMs and the bf16
rounding of the output and of grad_h, q and grad_x).
"""
import copy

import pytest
import torch

pytestmark = pytest.mark.gpu

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
    a, b, s = a.detach().double().cpu(), b.detach().double().cpu(), s.detach().double().cpu()
    bad = (a - b).abs() > tol * s + 1e-30
    assert not bad.any(), f"{what}: {int(bad.sum())} entries off, first at {bad.nonzero()[:3].tolist()}, " \
                          f"max err {(a - b).abs().max().item():.3e}"


def _close(a, b, tol, what):
    a, b = a.detach().double().cpu(), b.detach().double().cpu()
    err = (a - b).abs().max().item() if a.numel() else 0.0
    scale = b.abs().max().item() if b.numel() else 0.0
    assert err <= tol * max(scale, 1e-3), f"{what}: max err {err:.3e} vs scale {scale:.3e}"


def _power_law(n_src, n_dst, e, seed, isolated=8):
    g = torch.Generator().manual_seed(seed)
    src = (torch.rand(e, generator=g) ** 3 * n_src).long().clamp(max=n_src - 1)              # source out-hubs too
    dst = (torch.rand(e, generator=g) ** 4 * (n_dst - isolated)).long().clamp(max=n_dst - isolated - 1)
    return src, dst                                     # the last `isolated` destinations have no in-edges


def _formula(src, dst, n_src, n_dst, x, h, wp, g, mean):
    """fp64 out, dW', grad_h, grad_x and their sums of |terms|."""
    x, h, wp, g = (t.detach().double().cpu() for t in (x, h, wp, g))
    src, dst = src.cpu(), dst.cpu()
    E, K, Fi = src.numel(), h.size(1), x.size(1)
    ht = torch.cat([h, torch.ones(E, 1, dtype=h.dtype)], 1)
    xj = x[src]
    outer = (ht[:, :, None] * xj[:, None, :]).reshape(E, -1)
    inv = 1.0 / torch.bincount(dst, minlength=n_dst).clamp(min=1).double() if mean else torch.ones(n_dst, dtype=torch.float64)
    p = torch.zeros(n_dst, outer.size(1), dtype=torch.float64).index_add_(0, dst, outer) * inv[:, None]
    pa = torch.zeros_like(p).index_add_(0, dst, outer.abs()) * inv[:, None]
    res = {"out": (p @ wp, pa @ wp.abs()), "gw": (p.T @ g, pa.T @ g.abs())}
    dp = ((g @ wp.T) * inv[:, None])[dst].view(E, K + 1, Fi)
    dpa = ((g.abs() @ wp.abs().T) * inv[:, None])[dst].view(E, K + 1, Fi)
    res["gh"] = (torch.einsum("ekf,ef->ek", dp[:, :K], xj), torch.einsum("ekf,ef->ek", dpa[:, :K], xj.abs()))
    q = torch.einsum("ek,ekf->ef", ht, dp)
    qa = torch.einsum("ek,ekf->ef", ht.abs(), dpa)
    res["gx"] = (torch.zeros(n_src, Fi, dtype=torch.float64).index_add_(0, src, q),
                 torch.zeros(n_src, Fi, dtype=torch.float64).index_add_(0, src, qa))
    return res


def _operands(src, n_src, e, K, Fi, Fo, dtype, seed):
    g = torch.Generator().manual_seed(seed)
    x = torch.randn(n_src, Fi, generator=g).to(dtype)
    h = torch.randn(e, K, generator=g).to(dtype)
    wp = (torch.randn((K + 1) * Fi, Fo, generator=g) / (K * Fi) ** 0.5).to(dtype)
    return x, h, wp


def _run(graph, x, h, wp, gout, reduce):
    xg, hg, wg = (t.to(DEV).requires_grad_() for t in (x, h, wp))
    out = Fn.nn_conv_aggregate(graph, xg, hg, wg, reduce)
    out.backward(gout.to(DEV, out.dtype))
    return out, xg.grad, hg.grad, wg.grad


# (K, F_in, F_out): F_in = 1 as in MNIST's first conv ((K+1) F_in = 26: library GEMM); a width the wgmma GEMM takes
# ((K+1) F_in = 256, F_out = 64); odd widths it rejects
SHAPES = [(25, 1, 32), (31, 8, 64), (5, 6, 10)]


@pytest.mark.parametrize("dtype", [torch.float32, torch.bfloat16])
@pytest.mark.parametrize("reduce", ["sum", "mean"])
@pytest.mark.parametrize("K,Fi,Fo", SHAPES)
def test_op_against_fp64_on_power_law_graph(dtype, reduce, K, Fi, Fo):
    n_src, n_dst, e = 900, 700, 9000
    src, dst = _power_law(n_src, n_dst, e, seed=K + Fi)
    graph = CSRGraph(src.to(DEV), dst.to(DEV), n_src, n_dst)
    assert graph.plan.n_long > 0                               # hub rows above the chunk
    x, h, wp = _operands(src, n_src, e, K, Fi, Fo, dtype, seed=1)
    gout = torch.randn(n_dst, Fo, generator=torch.Generator().manual_seed(2))
    with _Profile() as prof:
        out, gx, gh, gw = _run(graph, x, h, wp, gout, reduce)
    assert prof.calls.get("nn_conv_csr") == 2 and prof.calls.get("nn_conv_backward_dst") == 1
    ref = _formula(src, dst, n_src, n_dst, x, h, wp, gout.to(dtype).float(), reduce == "mean")
    tol = TOL[dtype]
    assert out.dtype == dtype and gx.dtype == dtype and gh.dtype == dtype and gw.dtype == dtype
    _check(out, *ref["out"], tol, "out")
    _check(gw, *ref["gw"], tol, "grad_w'")
    _check(gh, *ref["gh"], tol, "grad_h")
    _check(gx, *ref["gx"], tol, "grad_x")
    assert (out[-8:] == 0).all()                               # isolated destinations


@pytest.mark.parametrize("idx", [torch.int32, torch.int64])
def test_adopted_csr_and_index_dtypes(idx):
    n, e, K, Fi, Fo = 300, 2500, 7, 16, 64
    src, dst = _power_law(n, n, e, seed=5, isolated=3)
    order = torch.argsort(dst, stable=True)
    src, dst = src[order], dst[order]
    rowptr = torch.zeros(n + 1, dtype=torch.long)
    rowptr[1:] = torch.cumsum(torch.bincount(dst, minlength=n), 0)
    graph = CSRGraph.from_csr(rowptr.to(DEV), src.to(DEV), n, idx_dtype=idx)
    assert graph.perm is None
    x, h, wp = _operands(src, n, e, K, Fi, Fo, torch.float32, seed=6)
    gout = torch.randn(n, Fo, generator=torch.Generator().manual_seed(7))
    out, gx, gh, gw = _run(graph, x, h, wp, gout, "mean")
    ref = _formula(src, dst, n, n, x, h, wp, gout, True)
    for name, got in (("out", out), ("gw", gw), ("gh", gh), ("gx", gx)):
        _check(got, *ref[name], 1e-5, name)


def test_no_edges():
    n, K, Fi, Fo = 50, 4, 8, 16
    graph = CSRGraph(torch.empty(0, dtype=torch.long, device=DEV), torch.empty(0, dtype=torch.long, device=DEV), n, n)
    x, h, wp = _operands(None, n, 0, K, Fi, Fo, torch.float32, seed=8)
    out, gx, gh, gw = _run(graph, x, h, wp, torch.randn(n, Fo), "sum")
    assert out.shape == (n, Fo) and (out == 0).all()
    assert (gx == 0).all() and gh.shape == (0, K) and (gw == 0).all()


@pytest.mark.parametrize("K,Fi,Fo", [(31, 8, 64), (5, 6, 10)])
def test_deterministic_and_blocked(monkeypatch, K, Fi, Fo):
    """Two runs are bit-identical; with the block cap lowered so that P spans at least 3 blocks, the output is
    bit-identical to the one-block run where the wgmma GEMM runs ((K+1) F_in = 256, F_out = 64), and within the bar
    where the library GEMM runs; the gradients are within the bar."""
    n_src, n_dst, e = 800, 600, 8000
    src, dst = _power_law(n_src, n_dst, e, seed=11)
    graph = CSRGraph(src.to(DEV), dst.to(DEV), n_src, n_dst)
    x, h, wp = _operands(src, n_src, e, K, Fi, Fo, torch.float32, seed=12)
    gout = torch.randn(n_dst, Fo, generator=torch.Generator().manual_seed(13))
    a = _run(graph, x, h, wp, gout, "sum")
    b = _run(graph, x, h, wp, gout, "sum")
    for u, v in zip(a, b):
        assert torch.equal(u, v)
    width = (K + 1) * Fi
    monkeypatch.setattr(Fn, "NN_CONV_BLOCK_BYTES", 4 * width * 250)
    assert len(Fn._nn_conv_blocks(n_dst, width)) >= 3
    c = _run(graph, x, h, wp, gout, "sum")
    ref = _formula(src, dst, n_src, n_dst, x, h, wp, gout, False)
    if width % 32 == 0 and Fo == 64:
        assert torch.equal(c[0], a[0])
    _check(c[0], *ref["out"], 1e-5, "blocked out")
    for got, name in zip(c[1:], ("gx", "gh", "gw")):
        _check(got, *ref[name], 1e-5, "blocked " + name)


def test_unsupported_shape_is_refused():
    graph = CSRGraph(torch.tensor([0], device=DEV), torch.tensor([0], device=DEV), 1, 1)
    x = torch.randn(1, 64, device=DEV)
    h = torch.randn(1, 256, device=DEV)
    assert not ops.nn_conv_supported(256, 64, torch.float32)
    with pytest.raises(ValueError, match="does not take"):
        Fn.nn_conv_aggregate(graph, x, h, torch.randn(257 * 64, 8, device=DEV))
    with pytest.raises(Exception, match="code -2"):
        ops.nn_conv_csr(graph.rowptr, graph.col, graph.perm, x, h, 0, 1)


# ---------------------------------------------------------------------------------------------- the plug-in layer
@pytest.fixture
def tg_installed(tg):
    from pytorch_geometric_b200 import plugin
    plugin.install(layers=True)
    yield tg
    plugin.uninstall()


def _net(d, k, fi, fo, bare=False):
    from torch.nn import Linear, ReLU, Sequential
    return Linear(d, fi * fo) if bare else Sequential(Linear(d, k), ReLU(), Linear(k, fi * fo))


def _cpu_and_gpu(tg, cls_name, layer_args, kw, x, ei, ea, x_dst=None):
    from pytorch_geometric_b200 import plugin
    torch.manual_seed(21)
    mine = getattr(tg.nn.conv, cls_name)(*layer_args, **kw)
    plugin.uninstall()
    ref = getattr(tg.nn.conv, cls_name)(*copy.deepcopy(layer_args), **kw)     # its own edge network
    plugin.install(layers=True)
    ref.load_state_dict(mine.state_dict())
    with torch.no_grad():
        if ref.bias is not None:
            ref.bias.normal_()
            mine.bias.copy_(ref.bias)
    mine = mine.to(DEV)
    xc = x.clone().requires_grad_()
    ec = ea.clone().requires_grad_()
    xin_c = xc if x_dst is None else (xc, x_dst)
    want = ref(xin_c, ei, ec)
    gout = torch.randn_like(want)
    want.backward(gout)
    xg = x.to(DEV).requires_grad_()
    eg = ea.to(DEV).requires_grad_()
    xin_g = xg if x_dst is None else (xg, x_dst.to(DEV))
    with _Profile() as prof:
        got = mine(xin_g, ei.to(DEV), eg)
        got.backward(gout.to(DEV))
    return mine, ref, (got, xg.grad, eg.grad), (want, xc.grad, ec.grad), prof


@pytest.mark.parametrize("cls_name,aggr,bare,bip", [("NNConv", "add", False, False), ("NNConv", "mean", False, True),
                                                    ("ECConv", "mean", True, False), ("ECConv", "add", False, True)])
def test_reference_layer_reaches_the_fused_path(tg_installed, cls_name, aggr, bare, bip):
    tg = tg_installed
    from pytorch_geometric_b200.plugin import conv as PC
    n, e, d, k, fi, fo = 400, 5000, 5, 16, 16, 32
    src, dst = _power_law(n, n, e, seed=22)
    ei = torch.stack([src, dst])
    x = torch.randn(n, fi)
    ea = torch.randn(e, d)
    ch = (fi, 12) if bip else fi
    x_dst = torch.randn(n, 12) if bip else None
    mine, ref, got, want, prof = _cpu_and_gpu(tg, cls_name, (ch, fo, _net(d, k, fi, fo, bare)), {"aggr": aggr}, x, ei, ea,
                                              x_dst)
    assert type(mine) is PC.B200NNConv
    assert prof.calls.get("nn_conv_csr") and prof.calls.get("nn_conv_backward_dst")
    for a, b, name in zip(got, want, ("out", "grad_x", "grad_edge_attr")):
        _close(a, b, 1e-4, name)
    for (name, pg), (_, pc) in zip(mine.named_parameters(), ref.named_parameters()):
        _close(pg.grad, pc.grad, 1e-4, name)


def test_training_step_memory_is_below_one_edge_weight_tensor(tg_installed):
    tg = tg_installed
    n, e, d, k, f = 20_000, 200_000, 8, 64, 64
    g = torch.Generator(device=DEV).manual_seed(31)
    ei = torch.stack([torch.randint(0, n, (e, ), device=DEV, generator=g),
                      (torch.rand(e, device=DEV, generator=g) ** 2 * (n - 1)).long()])
    x = torch.randn(n, f, device=DEV, generator=g).requires_grad_()
    ea = torch.randn(e, d, device=DEV, generator=g)
    conv = tg.nn.NNConv(f, f, _net(d, k, f, f), aggr="add").to(DEV)
    conv(x, ei, ea).sum().backward()                                      # graph build and warm-up
    torch.cuda.synchronize()
    torch.cuda.reset_peak_memory_stats()
    base = torch.cuda.memory_allocated()
    conv(x, ei, ea).sum().backward()
    torch.cuda.synchronize()
    assert torch.cuda.max_memory_allocated() - base < e * f * f * 4


def _dyadic(shape, g, scale):
    """Entries in {0, +-scale}: every product and sum the layer forms on them is exact in fp16 and bf16 at these sizes,
    so the result does not depend on the order in which any reduction adds."""
    return (torch.randint(-1, 2, shape, generator=g) * scale).float()


def _fall_through_inputs(n=60, d=3, fi=4):
    g = torch.Generator().manual_seed(41)
    dst = torch.arange(n).repeat_interleave(2)                 # in-degree 2, no duplicate edges
    src = (dst * 7 + 1 + torch.arange(2 * n) % 2 * 3) % n
    perm = torch.randperm(2 * n, generator=g)
    return torch.stack([src[perm], dst[perm]]), _dyadic((n, fi), g, 1.0), _dyadic((2 * n, d), g, 1.0)


def _dyadic_layer(tg, kw, net, fi=4, fo=5):
    conv = tg.nn.NNConv(fi, fo, net, **kw)
    g = torch.Generator().manual_seed(42)
    with torch.no_grad():
        for p in conv.parameters():
            p.copy_(_dyadic(tuple(p.shape), g, 0.5))
    return conv


FALL_THROUGH = ["max", "not_linear", "fp64", "fp16", "cpu", "autocast", "autocast_bare", "sparse"]


@pytest.mark.parametrize("kind", FALL_THROUGH)
def test_fall_through_configurations(tg_installed, kind):
    """Max aggregation, an edge network not ending in a Linear, fp64 and fp16 tensors, CPU tensors, torch.autocast
    (with a Sequential and with a bare Linear edge network) and a torch.sparse adjacency run the reference's code (no
    NNConv kernel) and give exactly its result: the same module with the plug-in uninstalled."""
    tg = tg_installed
    from pytorch_geometric_b200 import plugin
    from torch.nn import Linear, ReLU, Sequential
    d, fi, fo = 3, 4, 5
    ei, x, ea = _fall_through_inputs(d=d, fi=fi)
    n = x.size(0)
    net = {"not_linear": Sequential(Linear(d, fi * fo), ReLU()), "autocast_bare": Linear(d, fi * fo)}.get(
        kind, Sequential(Linear(d, 4), ReLU(), Linear(4, fi * fo)))
    kw = {"aggr": "max"} if kind == "max" else ({"aggr": "mean"} if kind in ("fp16", "sparse") else {})
    dt = {"fp64": torch.float64, "fp16": torch.float16}.get(kind, torch.float32)
    dev = "cpu" if kind == "cpu" else DEV
    mine = _dyadic_layer(tg, kw, net, fi, fo).to(dev, dt)
    plugin.uninstall()
    ref = copy.deepcopy(mine)
    ref.__class__ = tg.nn.NNConv
    plugin.install(layers=True)

    def call(module):
        xi, ai = x.to(dev, dt), ea.to(dev, dt)
        if kind == "sparse":
            adj = tg.utils.to_torch_coo_tensor(ei.to(dev), ai, size=(n, n)).transpose(0, 1).coalesce()
            return module(xi, adj)
        if kind.startswith("autocast"):
            with torch.autocast("cuda", dtype=torch.bfloat16):
                return module(xi, ei.to(dev), ai)
        return module(xi, ei.to(dev), ai)

    with _Profile() as prof:
        got = call(mine)
    assert not any(k.startswith("nn_conv") for k in prof.calls), (kind, prof.calls)
    plugin.uninstall()
    want = call(ref)
    plugin.install(layers=True)
    assert got.dtype == want.dtype and got.device == want.device, (got.dtype, want.dtype)
    assert torch.equal(got, want), (kind, (got.double() - want.double()).abs().max().item())


def test_missing_edge_attr_raises_the_reference_error(tg_installed):
    tg = tg_installed
    from pytorch_geometric_b200 import plugin
    from torch.nn import Linear
    ei, x, _ = _fall_through_inputs()
    conv = tg.nn.NNConv(4, 5, Linear(3, 20)).to(DEV)
    with pytest.raises(Exception) as mine_err:
        conv(x.to(DEV), ei.to(DEV))
    plugin.uninstall()
    ref = copy.deepcopy(conv)
    ref.__class__ = tg.nn.NNConv
    with pytest.raises(Exception) as ref_err:
        ref(x.to(DEV), ei.to(DEV))
    plugin.install(layers=True)
    assert type(mine_err.value) is type(ref_err.value) and str(mine_err.value) == str(ref_err.value)


# ---------------------------------------------------------------------------------------------- golden data
GOLDEN = [("qm9_add", 8, 8, 5, 16, {}), ("qm9_mean", 8, 8, 5, 16, {"aggr": "mean"}), ("bipartite", (8, 16), 32, 3, 8, {}),
          ("bare_linear", 6, 4, 3, None, {}), ("no_root_no_bias", 4, 8, 2, 6, {"root_weight": False, "bias": False}),
          ("isolated", 8, 8, 5, 16, {"aggr": "mean"})]


@pytest.mark.parametrize("tag,ch,f_out,d,k,kw", GOLDEN)
def test_mirror_matches_golden(golden, tag, ch, f_out, d, k, kw):
    from pytorch_geometric_b200.nn import NNConv
    z = golden("nn_conv")
    f_src = ch if isinstance(ch, int) else ch[0]
    mine = NNConv(ch, f_out, _net(d, k, f_src, f_out, bare=k is None), **kw)
    mine.load_state_dict({key[len(tag) + 3:]: torch.from_numpy(v) for key, v in z.items() if key.startswith(f"{tag}_p_")})
    mine = mine.to(DEV)
    x = torch.from_numpy(z[f"{tag}_x"]).to(DEV).requires_grad_()
    ea = torch.from_numpy(z[f"{tag}_ea"]).to(DEV).requires_grad_()
    x_dst = torch.from_numpy(z[f"{tag}_x_dst"]).to(DEV).requires_grad_() if f"{tag}_x_dst" in z else None
    ei = torch.from_numpy(z[f"{tag}_ei"]).to(DEV)
    out = mine(x if x_dst is None else (x, x_dst), ei, ea)
    out.backward(torch.from_numpy(z[f"{tag}_gout"]).to(DEV))
    _close(out, torch.from_numpy(z[f"{tag}_out"]), 1e-5, "out")
    _close(x.grad, torch.from_numpy(z[f"{tag}_gx"]), 1e-5, "grad_x")
    _close(ea.grad, torch.from_numpy(z[f"{tag}_gea"]), 1e-5, "grad_edge_attr")
    if x_dst is not None:
        _close(x_dst.grad, torch.from_numpy(z[f"{tag}_gx_dst"]), 1e-5, "grad_x_dst")
    for name, p in mine.named_parameters():
        _close(p.grad, torch.from_numpy(z[f"{tag}_g_{name}"]), 1e-5, "grad " + name)
