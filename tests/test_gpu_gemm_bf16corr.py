"""GPU accuracy of the dense products' correction arithmetic (csrc/gemm_tf32x3.cu): per k-step one BF16 wgmma carries
both correction products bf16(a_lo) bf16(b_hi) + bf16(a_hi) bf16(b_lo), and one TF32 wgmma the product a_hi b_hi.

Every check is against fp64 at 2e-6 * sum |terms| (a CPU emulation of the BF16 correction gives <= 7e-7 on random
inputs; a dropped correction instruction gives ~5e-4, a dropped half of the pair ~2e-4), over every way the kernel gets
its B operand: pre-split K-major (forward, K-major input gradient: the correction packed once per call and staged by
TMA), pre-split MN-major (pair form, layout 1), unsplit K-major and unsplit MN-major (split in the kernel, e.g. the
weight gradient's x)."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from pytorch_geometric_b200 import dense  # noqa: E402

DEV = "cuda"
TOL = 2e-6
TERM_BOUND = 2.0**-17 + 2.0**-21          # worst case per term (tests/test_gemm_bf16corr_numerics_cpu.py)


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _rel(got, a, b):
    """max |got - a b| / (|a| |b|), a [M, K], b [K, N], in fp64."""
    a64, b64 = a.double(), b.double()
    return float(((got.double() - a64 @ b64).abs() / (a64.abs() @ b64.abs() + 1e-300)).max())


def _all_products(x, w, go):
    """{name: max relative error} of every product form the layer and the pair / unsplit paths run."""
    n, k = w.shape
    w_hi, w_lo = dense.split_tf32(w)
    res = {
        "forward": _rel(dense.linear_forward(x, w_hi, w_lo), x, w.t()),
        "forward_unsplit": _rel(dense.linear_forward(x, w, None), x, w.t()),
        "grad_input_mn": _rel(dense.linear_grad_input(go, w_hi, w_lo), go, w),
        "grad_input_mn_unsplit": _rel(dense.linear_grad_input(go, w, None), go, w),
        "grad_input": _rel(dense.linear_grad_input_w(go, w, w_hi, w_lo), go, w),
    }
    if n % 128 == 0:                                  # weight gradient (A = g^T MN-major, B = x MN-major, unsplit)
        res["grad_weight"] = _rel(dense.linear_grad_weight(go, x), go.t(), x)
        # pair form, B = W^T pre-split MN-major
        wt = w.t().contiguous()
        wt_hi, wt_lo = dense.split_tf32(wt)
        res["pair_mn"] = _rel(dense.gemm_pair(x, None, wt_hi, wt_lo, 1, n)[0], x, w.t())
    return res


def _assert_within(res, tol):
    bad = {name: r for name, r in res.items() if not r <= tol}
    assert not bad, f"max err / sum|terms| above {tol:.1e}: {bad}"


@pytest.mark.parametrize("n,k", [(64, 256), (128, 128), (128, 64), (256, 256), (512, 256), (256, 512)])
def test_random_inputs_every_width(n, k):
    m = 5000 + 37
    gen = _gen(n * 3 + k)
    x = torch.randn(m, k, device=DEV, generator=gen)
    w = torch.randn(n, k, device=DEV, generator=gen) / k ** 0.5
    go = torch.randn(m, n, device=DEV, generator=gen)
    _assert_within(_all_products(x, w, go), TOL)


@pytest.mark.parametrize("exact", ["x", "w", "g"])
def test_each_half_of_the_correction_pair(exact):
    """One operand TF32-representable (its a_lo = 0): in each product only one half of the BF16 pair corrects --
    x exact: the forward's a_hi b_lo, the weight gradient's a_lo b_hi; W exact: the forward's and input gradient's
    a_lo b_hi; g exact: the input gradient's a_hi b_lo and the weight gradient's a_hi b_lo."""
    m, n, k = 3000, 256, 256
    gen = _gen({"x": 1, "w": 2, "g": 3}[exact])
    x = torch.randn(m, k, device=DEV, generator=gen)
    w = torch.randn(n, k, device=DEV, generator=gen) / k ** 0.5
    go = torch.randn(m, n, device=DEV, generator=gen)
    if exact == "x":
        x = dense.split_tf32(x)[0]
    elif exact == "w":
        w = dense.split_tf32(w)[0]
    else:
        go = dense.split_tf32(go)[0]
    _assert_within(_all_products(x, w, go), TOL)


def _worst_residuals(shape, gen, signed):
    """Values whose TF32 residual is 0.9 .. 0.999 of half a TF32 ulp, with significands just above 1: |a_lo| ~ 2^-11 |a|."""
    e = torch.randint(-3, 3, shape, device=DEV, generator=gen)
    hi = torch.ldexp(1.0 + torch.randint(1, 5, shape, device=DEV, generator=gen).double() * 2.0**-10, e)
    u = 0.9 + 0.099 * torch.rand(shape, device=DEV, generator=gen, dtype=torch.float64)
    u = u * (torch.randint(0, 2, shape, device=DEV, generator=gen) * 2 - 1)
    v = hi + u * torch.ldexp(torch.ones_like(hi), e - 11)
    if signed:
        s = torch.randint(0, 2, shape, device=DEV, generator=gen) * 2 - 1
        hi, v = hi * s, v * s
    v = v.float()
    assert torch.equal(dense.split_tf32(v)[0], hi.float())                # still rounds to hi: a residual, not a carry
    return v


@pytest.mark.parametrize("signed", [False, True])
def test_worst_case_residuals(signed):
    """Every operand carries a residual near +-2^-11 of its value: within the worst-case per-term bound of the
    BF16 correction plus fp32 accumulation."""
    m, n, k = 4000, 256, 256
    gen = _gen(10 + int(signed))
    x = _worst_residuals((m, k), gen, signed)
    w = _worst_residuals((n, k), gen, signed)
    go = _worst_residuals((m, n), gen, signed)
    res = _all_products(x, w, go)
    _assert_within(res, TERM_BOUND + 1e-6)
