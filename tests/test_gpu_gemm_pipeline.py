"""GPU checks of the pipelined 3xTF32 GEMM (csrc/gemm_tf32x3.cu): the transposed weight split, the B operand read
straight from the TMA stages against the B-preparation warps (same bits), and the shapes that stress the ring of
stages: long K with a tensor-map switch inside the ring, CTAs with 1, 2 or a ragged number of tiles, grouped
segments that are empty or one row long, uneven split-K, and bias / ReLU epilogues on a ragged last tile.
Accuracy is checked against fp64 at 1e-5 * sum |terms|."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from pytorch_geometric_b200 import dense  # noqa: E402
from pytorch_geometric_b200._lib import lib  # noqa: E402

DEV = "cuda"


def _check(got, ref64, scale64, tol=1e-5):
    err = (got.double() - ref64).abs()
    assert (err <= tol * scale64 + 1e-30).all(), f"max err/scale {float((err / (scale64 + 1e-30)).max()):.3e}"


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


@pytest.mark.parametrize("rows,cols", [(256, 256), (128, 512), (64, 256), (33, 70)])
def test_transposed_split_is_exact(rows, cols):
    w = torch.randn(rows, cols, device=DEV, generator=_gen(rows + cols))
    wt_hi, wt_lo = dense.split_tf32_transposed(w)
    assert wt_hi.shape == (cols, rows)
    assert torch.equal(wt_hi + wt_lo, w.t())
    assert torch.equal(wt_hi.view(torch.int32) & 0x1fff, torch.zeros_like(wt_hi, dtype=torch.int32))
    hi, lo = dense.split_tf32(w)
    assert torch.equal(wt_hi, hi.t()) and torch.equal(wt_lo, lo.t())


@pytest.mark.parametrize("m", [1, 128, 129, 3000, 40000])
@pytest.mark.parametrize("n,k", [(256, 256), (128, 512), (512, 128)])
def test_kmajor_grad_input_matches_mn_major_bits(m, n, k):
    """gx = g W from the stage-resident K-major W^T and from the transposed-in-kernel MN-major W: same bits."""
    gen = _gen(m + n + k)
    w = torch.randn(n, k, device=DEV, generator=gen) / n ** 0.5
    go = torch.randn(m, n, device=DEV, generator=gen)
    w_hi, w_lo = dense.split_tf32(w)
    ref = dense.linear_grad_input(go, w_hi, w_lo)
    assert torch.equal(dense.linear_grad_input_w(go, w, w_hi, w_lo), ref)
    assert torch.equal(dense.linear_grad_input(go, w, None), ref)
    _check(ref, go.double() @ w.double(), go.double().abs() @ w.double().abs())


@pytest.mark.parametrize("layout", [0, 1])
def test_long_k_pair_switches_stream_mid_ring(layout):
    """K = 2048 split 1376 + 672: the switch from a1 to a2 lands on k-block 43, not on a multiple of the ring depth."""
    m, k1, k2, n = 1000, 1376, 672, 256
    gen = _gen(7 + layout)
    a1 = torch.randn(m, k1, device=DEV, generator=gen)
    a2 = torch.randn(m, k2, device=DEV, generator=gen)
    w = torch.randn(n, k1 + k2, device=DEV, generator=gen) / (k1 + k2) ** 0.5     # [N, K]
    b = w if layout == 0 else w.t().contiguous()
    hi, lo = dense.split_tf32(b)
    y, _ = dense.gemm_pair(a1, a2, hi, lo, layout, n)
    a = torch.cat([a1, a2], 1).double()
    _check(y, a @ w.double().t(), a.abs() @ w.double().abs().t())
    y_raw, _ = dense.gemm_pair(a1, a2, b, None, layout, n)
    assert torch.equal(y_raw, y)


@pytest.mark.parametrize("tiles_per_cta", [1, 2, 5])
def test_tiles_per_cta(tiles_per_cta):
    """M chosen so that each CTA gets 1, 2 or 5 tiles (5 k-blocks-per-tile multiples do not divide the ring)."""
    sms = torch.cuda.get_device_properties(0).multi_processor_count
    n, k = 256, 160                                               # 2 column tiles, 5 k-blocks per tile
    m = (sms * tiles_per_cta // 2) * 128 - 37
    gen = _gen(tiles_per_cta)
    x = torch.randn(m, k, device=DEV, generator=gen)
    w = torch.randn(n, k, device=DEV, generator=gen) / k ** 0.5
    hi, lo = dense.split_tf32(w)
    y = dense.linear_forward(x, hi, lo)
    _check(y, x.double() @ w.double().t(), x.double().abs() @ w.double().abs().t())
    assert torch.equal(dense.linear_forward(x, w, None), y)


@pytest.mark.parametrize("layout", [0, 1])
def test_grouped_empty_and_one_row_segments(layout):
    sizes = [0, 1, 300, 0, 128, 1, 129, 0]
    k, n = 96, 256
    gen = _gen(11 + layout)
    m = sum(sizes)
    a = torch.randn(m, k, device=DEV, generator=gen)
    ws = torch.randn(len(sizes), k, n, device=DEV, generator=gen) / k ** 0.5    # c = a w[r]
    b = ws if layout == 1 else ws.transpose(1, 2).contiguous()                  # layout 0: [R, N, K]
    hi, lo = dense.split_tf32(b)
    ptr = torch.tensor([0] + sizes, device=DEV, dtype=torch.int64).cumsum(0)
    c = dense._grouped(a, ptr, hi, lo, layout, n)
    row = 0
    for r, s in enumerate(sizes):
        seg = a[row:row + s].double()
        _check(c[row:row + s], seg @ ws[r].double(), seg.abs() @ ws[r].double().abs())
        row += s


@pytest.mark.parametrize("m", [32 * 7 * 132 + 5, 100003])
def test_split_k_uneven(m):
    """grad_W's split-K where the number of splits does not divide the k-blocks; deterministic."""
    n, k = 256, 256
    gen = _gen(m)
    x = torch.randn(m, k, device=DEV, generator=gen)
    go = torch.randn(m, n, device=DEV, generator=gen)
    gw = dense.linear_grad_weight(go, x)
    _check(gw, go.double().t() @ x.double(), go.double().abs().t() @ x.double().abs(), tol=2e-5)
    assert torch.equal(gw, dense.linear_grad_weight(go, x))


@pytest.mark.parametrize("relu", [False, True])
@pytest.mark.parametrize("m", [77, 1000, 5000 + 13])
def test_bias_relu_epilogue_ragged(m, relu):
    n, k = 384, 128
    gen = _gen(m + int(relu))
    x = torch.randn(m, k, device=DEV, generator=gen)
    w = torch.randn(n, k, device=DEV, generator=gen) / k ** 0.5
    bias = torch.randn(n, device=DEV, generator=gen)
    hi, lo = dense.split_tf32(w)
    y, y2 = dense.gemm_pair(x, None, hi, lo, 0, 256, 128, bias=bias, relu=relu)
    ref = x.double() @ w.double().t() + bias.double()
    scale = x.double().abs() @ w.double().abs().t() + bias.double().abs()
    if relu:
        ref = ref.clamp_min(0)
    _check(torch.cat([y, y2], 1), ref, scale)


def test_transposed_split_rejects_bad_arguments():
    assert lib().b200mp_split_tf32_transposed(None, None, None, 4, 4, None) != 0
