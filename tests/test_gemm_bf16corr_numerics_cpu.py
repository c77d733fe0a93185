"""CPU emulation of the dense products' arithmetic (csrc/gemm_tf32x3.cu), pinning its error bound without a GPU.

Per k-step of 8 the kernel issues one BF16 wgmma (k = 16) holding both correction products of the split a = a_hi + a_lo,
    bf16(a_lo) * bf16(b_hi) + bf16(a_hi) * bf16(b_lo),
then the TF32 wgmma a_hi * b_hi, both accumulated into one fp32 accumulator.  The emulation rounds a_hi with rna to TF32,
rounds the pair members to nearest-even BF16, sums each instruction's exact products and rounds once per instruction
into the fp32 accumulator.  The tensor core's internal order is not modelled; the GPU tests decide that part."""
import numpy as np
import pytest

# per term: two correction products of at most 2^-11 |a b|, each off by two BF16 roundings of at most 2^-8, plus the
# dropped a_lo * b_lo (2^-22): 2^-17 + 2^-22, and second-order terms far below the 2^-22 of slack added here
TERM_BOUND = 2.0**-17 + 2.0**-21


def rna_tf32(x):
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    return ((b + np.uint32(0x1000)) & np.uint32(0xFFFFE000)).view(np.float32)


def rn_bf16(x):
    b = np.ascontiguousarray(x, dtype=np.float32).view(np.uint32)
    r = (b + np.uint32(0x7FFF) + ((b >> np.uint32(16)) & np.uint32(1))) & np.uint32(0xFFFF0000)
    return r.view(np.float32)


def split(x):
    hi = rna_tf32(x)
    return hi, (x - hi).astype(np.float32)


def gemm_bf16corr(a, b):
    """a [M, K] . b [N, K]^T as the kernel computes it."""
    a_hi, a_lo = split(a)
    b_hi, b_lo = split(b)
    ca_lo, ca_hi, cb_hi, cb_lo = (rn_bf16(v).astype(np.float64) for v in (a_lo, a_hi, b_hi, b_lo))
    acc = np.zeros((a.shape[0], b.shape[0]), dtype=np.float32)
    for k0 in range(0, a.shape[1], 8):
        s = slice(k0, k0 + 8)
        corr = ca_lo[:, s] @ cb_hi[:, s].T + ca_hi[:, s] @ cb_lo[:, s].T     # one k16 BF16 instruction
        acc = (acc + corr).astype(np.float32)
        main = a_hi[:, s].astype(np.float64) @ b_hi[:, s].astype(np.float64).T
        acc = (acc + main).astype(np.float32)
    return acc


def gemm_tf32x3(a, b):
    """The three-TF32-product split, for comparison."""
    a_hi, a_lo = (v.astype(np.float64) for v in split(a))
    b_hi, b_lo = (v.astype(np.float64) for v in split(b))
    acc = np.zeros((a.shape[0], b.shape[0]), dtype=np.float32)
    for k0 in range(0, a.shape[1], 8):
        s = slice(k0, k0 + 8)
        for p, q in ((a_lo, b_hi), (a_hi, b_lo), (a_hi, b_hi)):
            acc = (acc + p[:, s] @ q[:, s].T).astype(np.float32)
    return acc


def rel_err(got, a, b):
    a64, b64 = a.astype(np.float64), b.astype(np.float64)
    return float((np.abs(got - a64 @ b64.T) / (np.abs(a64) @ np.abs(b64).T + 1e-300)).max())


def test_rounding_helpers():
    x = np.array([1.0 + 2.0**-11, 1.0 + 2.0**-11 - 2.0**-23, -(1.0 + 2.0**-11), 1.0 + 2.0**-8, 1.0 + 3 * 2.0**-8],
                 dtype=np.float32)
    np.testing.assert_array_equal(rna_tf32(x), np.float32([1 + 2.0**-10, 1, -(1 + 2.0**-10), 1 + 2.0**-8, 1 + 3 * 2.0**-8]))
    np.testing.assert_array_equal(rn_bf16(x[3:]), np.float32([1.0, 1 + 2.0**-6]))      # ties to even


def test_per_term_bound_with_worst_case_residuals():
    """|bf16(a_lo) bf16(b_hi) + bf16(a_hi) bf16(b_lo) + a_hi b_hi - a b| <= TERM_BOUND |a b|, residuals at +-2^-11 |a|."""
    rng = np.random.default_rng(0)
    n = 200_000
    hi = (np.ldexp(1.0 + rng.integers(1, 5, (2, n)) * 2.0**-10, rng.integers(-6, 6, (2, n)))
          * rng.choice([-1.0, 1.0], (2, n)))
    u = rng.uniform(0.9, 0.999, (2, n)) * rng.choice([-1.0, 1.0], (2, n))
    v = (hi + u * np.ldexp(1.0, np.floor(np.log2(np.abs(hi))).astype(int) - 11)).astype(np.float32)
    a, b = v
    a_hi, a_lo = split(a)
    b_hi, b_lo = split(b)
    np.testing.assert_array_equal(a_hi, hi[0].astype(np.float32))           # the residual stays below half a TF32 ulp
    assert np.abs(a_lo / a).max() > 0.99 * 2.0**-11
    f = lambda x: rn_bf16(x).astype(np.float64)
    got = f(a_lo) * f(b_hi) + f(a_hi) * f(b_lo) + a_hi.astype(np.float64) * b_hi
    err = np.abs(got - a.astype(np.float64) * b) / np.abs(a.astype(np.float64) * b)
    assert err.max() <= TERM_BOUND, err.max()
    assert err.max() > 0.25 * TERM_BOUND                                    # the cases do reach toward the bound


@pytest.mark.parametrize("m,n,k", [(512, 256, 256), (512, 128, 64), (256, 64, 1024)])
def test_random_products_are_fp32_class(m, n, k):
    rng = np.random.default_rng(m + n + k)
    a = rng.standard_normal((m, k)).astype(np.float32)
    b = (rng.standard_normal((n, k)) / np.sqrt(k)).astype(np.float32)
    rel = rel_err(gemm_bf16corr(a, b), a, b)
    assert rel <= 2e-6, rel
    rel3 = rel_err(gemm_tf32x3(a, b), a, b)
    assert rel <= 4 * rel3 + 1e-7, (rel, rel3)


@pytest.mark.parametrize("side", ["a", "b"])
def test_each_correction_half_is_needed(side):
    """With one operand TF32-representable only one half of the BF16 pair carries the correction; dropping the
    correction instruction must then be visible far above the bar the GPU tests use."""
    rng = np.random.default_rng(1)
    a = rng.standard_normal((128, 256)).astype(np.float32)
    b = (rng.standard_normal((64, 256)) / 16).astype(np.float32)
    if side == "a":
        a = rna_tf32(a)
    else:
        b = rna_tf32(b)
    assert rel_err(gemm_bf16corr(a, b), a, b) <= 2e-6
    plain = rna_tf32(a).astype(np.float64) @ rna_tf32(b).astype(np.float64).T
    assert rel_err(plain.astype(np.float32), a, b) > 5e-5
