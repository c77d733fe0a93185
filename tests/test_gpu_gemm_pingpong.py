"""GPU checks of the 3xTF32 GEMM's 256-row tiles (csrc/gemm_tf32x3.cu): each consumer warpgroup owns 128 rows of a
tile as two m64 halves that share the stage's B tile.  The shapes cover what that schedule adds: CTAs with 1, 2 or an
odd number of tiles (and, in the grouped form, CTAs with none), tiles
whose second warpgroup holds no valid row, a single k-block per tile, the pair form's output switch on either half of
a tile, grouped segments of 0, 1 and 129 rows and split-K with an uneven last split and a 128-row output (half a tile,
fewer TMA boxes).  Every result is held to fp64 at 2e-6 * sum |terms|, and bit-for-bit to the path that computes the
same (hi, correction) products another way."""
import pytest
import torch

pytestmark = pytest.mark.gpu

from pytorch_geometric_b200 import dense  # noqa: E402

DEV = "cuda"
BM = 256


def _check(got, ref64, scale64, tol=2e-6):
    err = (got.double() - ref64).abs()
    assert (err <= tol * scale64 + 1e-30).all(), f"max err/scale {float((err / (scale64 + 1e-30)).max()):.3e}"


def _gen(seed):
    return torch.Generator(device=DEV).manual_seed(seed)


def _sms():
    return torch.cuda.get_device_properties(0).multi_processor_count


def _forward_case(m, n, k, seed):
    gen = _gen(seed)
    x = torch.randn(m, k, device=DEV, generator=gen)
    w = torch.randn(n, k, device=DEV, generator=gen) / k ** 0.5
    hi, lo = dense.split_tf32(w)
    y = dense.linear_forward(x, hi, lo)
    _check(y, x.double() @ w.double().t(), x.double().abs() @ w.double().abs().t())
    assert torch.equal(dense.linear_forward(x, w, None), y)       # unsplit B: split by the preparation warps
    return y


@pytest.mark.parametrize("tiles_per_cta", [1, 2, 3])
def test_tiles_per_cta(tiles_per_cta):
    """Every CTA gets 1, 2 or 3 tiles (the last one ragged).  The grid never exceeds the tiles here; CTAs with no tile
    occur in the grouped form, whose work count is an upper bound (test_grouped_segments)."""
    n, k = 256, 96                                                # 2 column tiles, 3 k-blocks per tile
    m = (_sms() * tiles_per_cta // 2) * BM - 77
    _forward_case(m, n, k, tiles_per_cta)


@pytest.mark.parametrize("m", [1, 100, 128, 129, 255, 256, 257, 383])
def test_second_warpgroup_rows_masked(m):
    """Tiles whose rows end inside the first warpgroup's half (m <= 128), on the half boundary or inside the second."""
    _forward_case(m, 128, 64, m)


@pytest.mark.parametrize("m", [5, 300, 20011])
def test_single_k_block(m):
    """K = 32: one k-block, so every group is the first and last of its tile."""
    _forward_case(m, 256, 32, 31 + m)


@pytest.mark.parametrize("m", [200, 1000])
def test_kmajor_grad_input_matches_mn_major_bits(m):
    n, k = 256, 128
    gen = _gen(m)
    w = torch.randn(n, k, device=DEV, generator=gen) / n ** 0.5
    go = torch.randn(m, n, device=DEV, generator=gen)
    w_hi, w_lo = dense.split_tf32(w)
    ref = dense.linear_grad_input(go, w_hi, w_lo)
    assert torch.equal(dense.linear_grad_input_w(go, w, w_hi, w_lo), ref)
    _check(ref, go.double() @ w.double(), go.double().abs() @ w.double().abs())


@pytest.mark.parametrize("n1,n2", [(128, 256), (256, 128), (128, 128)])
@pytest.mark.parametrize("relu", [False, True])
def test_pair_output_switch_bias_relu(n1, n2, relu):
    """[c1 | c2] with the switch after an odd or even number of column tiles, two A streams, bias and ReLU on a
    ragged last tile."""
    m, k1, k2 = 3 * BM + 131, 96, 64
    gen = _gen(n1 + 3 * n2 + int(relu))
    a1 = torch.randn(m, k1, device=DEV, generator=gen)
    a2 = torch.randn(m, k2, device=DEV, generator=gen)
    w = torch.randn(n1 + n2, k1 + k2, device=DEV, generator=gen) / (k1 + k2) ** 0.5
    bias = torch.randn(n1 + n2, device=DEV, generator=gen)
    hi, lo = dense.split_tf32(w)
    y1, y2 = dense.gemm_pair(a1, a2, hi, lo, 0, n1, n2, bias=bias, relu=relu)
    a = torch.cat([a1, a2], 1).double()
    ref = a @ w.double().t() + bias.double()
    scale = a.abs() @ w.double().abs().t() + bias.double().abs()
    if relu:
        ref = ref.clamp_min(0)
    _check(torch.cat([y1, y2], 1), ref, scale)
    r1, r2 = dense.gemm_pair(a1, a2, w, None, 0, n1, n2, bias=bias, relu=relu)
    assert torch.equal(r1, y1) and torch.equal(r2, y2)


@pytest.mark.parametrize("layout", [0, 1])
def test_grouped_segments(layout):
    sizes = [0, 1, 129, 0, 256, 1, 129, 257]
    k, n = 64, 128
    gen = _gen(5 + layout)
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


@pytest.mark.parametrize("n", [128, 256, 384])
@pytest.mark.parametrize("m", [31, 32 * 5 * 132 + 7, 100003])
def test_split_k_uneven(m, n):
    """grad_W = g^T x: n = 128 fills half a 256-row tile (half the TMA boxes), 384 one and a half; the last split is
    short; two calls give the same bits."""
    k = 128
    gen = _gen(m + n)
    x = torch.randn(m, k, device=DEV, generator=gen)
    go = torch.randn(m, n, device=DEV, generator=gen)
    gw = dense.linear_grad_weight(go, x)
    _check(gw, go.double().t() @ x.double(), go.double().abs().t() @ x.double().abs())
    assert torch.equal(gw, dense.linear_grad_weight(go, x))
