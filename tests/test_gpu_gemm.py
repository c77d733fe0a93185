"""GPU parity of the wgmma 3xTF32 dense transform (csrc/gemm_tf32x3.cu) against an fp64
reference of the same products: fp32-class accuracy (1e-5 relative to sum |a||b|, the bound an
fp32 GEMM itself satisfies), ragged row counts, all supported widths, forward and both gradients,
and the layer-level equivalence with the strict-fp32 library path."""
import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from pytorch_geometric_b200 import dense  # noqa: E402
from pytorch_geometric_b200.nn import GCNConv  # noqa: E402

DEV = "cuda"
DEFAULT_GEMM_MODE = dense.DEFAULT_GEMM_MODE


def _check(got, ref64, scale64, tol=1e-5):
    err = (got.double() - ref64).abs()
    bound = tol * scale64 + 1e-30
    assert (err <= bound).all(), f"max err/scale {float((err / (scale64 + 1e-30)).max()):.3e}"


@pytest.fixture(params=["ss-bk32", "ss-bk16", "ts"])
def gemm_bk(request):
    """Every setting of the GEMM options the library accepts (gemm_mode, gemm_bk, gemm_prefetch) must give the
    fp32-accurate result; the sm_90a kernel has one configuration, so they must not change it either."""
    from pytorch_geometric_b200 import ops
    ops.set_option("gemm_mode", 1 if request.param == "ts" else 0)
    ops.set_option("gemm_bk", 16 if request.param == "ss-bk16" else 32)
    ops.set_option("gemm_prefetch", 0 if request.param == "ss-bk32" else 8)     # TMA L2 prefetch distance
    yield request.param
    ops.set_option("gemm_bk", 32)
    ops.set_option("gemm_prefetch", dense.DEFAULT_GEMM_PREFETCH)
    ops.set_option("gemm_mode", DEFAULT_GEMM_MODE)


@pytest.mark.parametrize("m", [1, 127, 128, 129, 1000, 20011])
@pytest.mark.parametrize("n,k", [(256, 256), (128, 256), (256, 128), (128, 64), (512, 256)])
def test_linear_tf32x3_forward_and_grads(m, n, k, gemm_bk):
    g = torch.Generator(device=DEV).manual_seed(m * 7 + n + k)
    x = torch.randn(m, k, device=DEV, generator=g)
    w = torch.randn(n, k, device=DEV, generator=g) / k ** 0.5
    go = torch.randn(m, n, device=DEV, generator=g)
    assert dense.supported(x, w)
    w_hi, w_lo = dense.split_tf32(w)
    assert torch.equal(w_hi + w_lo, w)                                   # the split is exact
    assert torch.equal(w_hi.view(torch.int32) & 0x1fff, torch.zeros_like(w_hi, dtype=torch.int32))  # tf32-representable
    y = dense.linear_forward(x, w_hi, w_lo)
    _check(y, x.double() @ w.double().t(), x.double().abs() @ w.double().abs().t())
    gx = dense.linear_grad_input(go, w_hi, w_lo)
    _check(gx, go.double() @ w.double(), go.double().abs() @ w.double().abs())
    gw = dense.linear_grad_weight(go, x)
    _check(gw, go.double().t() @ x.double(), go.double().abs().t() @ x.double().abs(), tol=2e-5)
    # determinism of the split-K reduction
    assert torch.equal(gw, dense.linear_grad_weight(go, x))


@pytest.mark.parametrize("m", [1, 129, 1000, 20011])
@pytest.mark.parametrize("n,k", [(256, 256), (128, 256), (256, 128), (512, 256)])
def test_unsplit_weight_gives_the_same_bits(m, n, k):
    """w_lo == NULL: the kernel splits each B tile itself (hi in place, lo next to it).  The split is the same
    arithmetic, so the results must be bit-identical to the pre-split path (both B layouts)."""
    from pytorch_geometric_b200 import ops
    ops.set_option("gemm_mode", 1)
    g = torch.Generator(device=DEV).manual_seed(m + n + k)
    x = torch.randn(m, k, device=DEV, generator=g)
    w = torch.randn(n, k, device=DEV, generator=g) / k ** 0.5
    go = torch.randn(m, n, device=DEV, generator=g)
    w_hi, w_lo = dense.split_tf32(w)
    assert torch.equal(dense.linear_forward(x, w, None), dense.linear_forward(x, w_hi, w_lo))
    assert torch.equal(dense.linear_grad_input(go, w, None), dense.linear_grad_input(go, w_hi, w_lo))
    dense.set_b_split(True)
    try:
        assert dense.prepare_weight(w)[1] is None
        conv = GCNConv(k, n).to(DEV)
        ei = torch.randint(0, m, (2, 4 * m), device=DEV)
        xr = x.clone().requires_grad_()
        out = conv(xr, ei)
        out.backward(go)
        g1, gw1 = xr.grad.clone(), conv.lin.weight.grad.clone()
        dense.set_b_split(False)
        xr.grad = None
        conv.zero_grad()
        out2 = conv(xr, ei)
        out2.backward(go)
        assert torch.equal(out, out2) and torch.equal(g1, xr.grad) and torch.equal(gw1, conv.lin.weight.grad)
    finally:
        dense.set_b_split(False)
        ops.set_option("gemm_mode", DEFAULT_GEMM_MODE)


def test_tf32x3_is_fp32_class_not_tf32_class():
    """A single-pass TF32 product is ~1e-3 accurate; the 3x split must be ~100x better than that."""
    g = torch.Generator(device=DEV).manual_seed(0)
    x = torch.randn(4096, 256, device=DEV, generator=g)
    w = torch.randn(256, 256, device=DEV, generator=g)
    ref = x.double() @ w.double().t()
    y = dense.linear(x, w)
    rel = ((y.double() - ref).abs().max() / ref.abs().max()).item()
    y32 = torch.nn.functional.linear(x, w)
    rel32 = ((y32.double() - ref).abs().max() / ref.abs().max()).item()
    assert rel < 2e-6 and rel < 8 * rel32 + 1e-7, (rel, rel32)


def test_gcn_layer_same_result_with_both_dense_backends():
    torch.manual_seed(3)
    N, E = 5000, 60000
    ei = torch.stack([torch.randint(0, N, (E, ), device=DEV), (torch.rand(E, device=DEV) ** 3 * (N - 1)).long()])
    x = torch.randn(N, 256, device=DEV)
    go = torch.randn(N, 256, device=DEV)
    conv = GCNConv(256, 256).to(DEV)
    outs = {}
    for backend in ("tf32x3", "cublas"):
        dense.set_backend(backend)
        xt = x.clone().requires_grad_()
        conv.zero_grad()
        out = conv(xt, ei)
        out.backward(go)
        outs[backend] = (out.detach(), xt.grad, conv.lin.weight.grad.clone())
    dense.set_backend("tf32x3")
    for a, b in zip(outs["tf32x3"], outs["cublas"]):
        torch.testing.assert_close(a, b, rtol=1e-4, atol=1e-4)


def test_unsupported_shapes_use_the_library_gemm():
    x = torch.randn(100, 48, device=DEV)
    w = torch.randn(24, 48, device=DEV)
    assert not dense.supported(x, w)
    torch.testing.assert_close(dense.linear(x, w), torch.nn.functional.linear(x, w))
