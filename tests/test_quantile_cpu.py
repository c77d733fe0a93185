"""Quantile aggregation on the CPU: the numpy restatement of the contract (tests/quantile_oracle.py) against the
unmodified reference's outputs and gradients (golden/quantile.npz), its rank arithmetic against quantile.py:88's fp32
arithmetic, the 2^24 divergence, the nn mirrors' errors, state and repr against the reference, the plug-in's rebinding
of QuantileAggregation.forward with CPU tensors falling through bit for bit, and the C ABI's argument checks."""
import numpy as np
import pytest
import torch

import quantile_oracle as O
from conftest import load_golden

CASES = O.golden_cases(load_golden("quantile"))


@pytest.mark.parametrize("name", sorted(CASES))
def test_oracle_reproduces_the_reference(name):
    c = CASES[name]
    x, d, idx, n, q, interp, fill, bf16, g = O.case_args(c)
    out, grad = O.aggregate(O.fold(x, d), idx, n, q, interp, fill, bf16, g)
    O.check_golden(c, O.layout(out, len(q), x.shape, d), O.unfold(grad, x.shape, d))


def test_golden_covers_the_contract():
    names = set(CASES)
    for interp in O.INTERP:
        assert {f"{interp}_q05", f"{interp}_q5", f"{interp}_q5_bf16", f"{interp}_special", f"{interp}_unsorted",
                f"{interp}_3d_dim0", f"{interp}_3d_dim1", f"{interp}_fill10_dimsize"} <= names
    assert {"nearest_half_offsets", "median", "median_bf16"} <= names


def _reference_ranks(q, count, ptr):
    """quantile.py:88 on torch CPU tensors: q * (count - 1) + ptr in fp32, then floor / ceil / round / frac."""
    P = torch.tensor(q, dtype=torch.float32).view(-1, 1) * (torch.tensor(count) - 1) + torch.tensor(ptr)
    return P.floor().long(), P.ceil().long(), P.round().long(), P.frac()


def test_rank_arithmetic_matches_the_reference_below_2_24():
    rng = np.random.default_rng(1)
    qs = np.concatenate([[0.0, 0.1, 0.25, 0.5, 0.75, 0.9, 1.0], rng.random(25)]).astype(np.float32)
    counts = np.concatenate([[1, 2, 3, 4, 5, 7, 1000, 65537], rng.integers(1, 1 << 20, 40)])
    ptrs = np.concatenate([[0, 1, 2, 3, 1 << 23, (1 << 23) + 1], rng.integers(0, 1 << 23, 40)])
    count = np.repeat(counts, ptrs.size)
    ptr = np.tile(ptrs, counts.size)
    keep = ptr + count - 1 < (1 << 24)
    count, ptr = count[keep], ptr[keep]
    fl, ce, ne, fr = (t.numpy() for t in _reference_ranks(qs.tolist(), count, ptr))
    for a, qv in enumerate(qs):
        for b in range(count.size):
            c, p = int(count[b]), int(ptr[b])
            lo, hi, frac = O.ranks(float(qv), p, c, "linear")
            assert (lo, hi) == (fl[a, b] - p, ce[a, b] - p) and frac == fr[a, b]
            assert O.ranks(float(qv), p, c, "nearest")[0] == ne[a, b] - p
            assert O.ranks(float(qv), p, c, "higher")[0] == ce[a, b] - p


def test_nearest_rounds_half_to_even_of_the_global_offset():
    # a group of 3 at q = 0.25: P = ptr + 0.5 rounds up at an odd offset, down at an even one, like the reference
    for ptr in range(0, 12):
        ne = _reference_ranks([0.25], [3], [ptr])[2].item()
        assert O.ranks(0.25, ptr, 3, "nearest")[0] == ne - ptr == (1 if ptr % 2 else 0)


def test_ranks_stay_inside_the_group_past_2_24():
    # one group of 2^24 + 1 messages, then groups of 3: the reference's fp32 P leaves these groups; the contract does
    # not, and the median of {3k, 3k + 1, 3k + 2} is rank 1
    ptr0 = (1 << 24) + 1
    escaped = 0
    for k in range(200):
        ptr = ptr0 + 3 * k
        lo, hi, frac = O.ranks(0.5, ptr, 3, "lower")
        assert lo == hi == 1 and frac == 0
        for interp in O.INTERP:
            lo, hi, _ = O.ranks(0.5, ptr, 3, interp)
            assert 0 <= lo <= hi <= 2
        ref_lo = _reference_ranks([0.5], [3], [ptr])[0].item() - ptr
        escaped += ref_lo != 1
    assert escaped > 100                       # the reference's fp32 offset is wrong for most of these groups


def test_ranks_are_clamped_into_the_group():
    # past 2^24 fl32(count - 1) may round up: count = 2^24 + 4 and q = 1 give h = fl32(2^24 + 3) = 2^24 + 4 = count
    n = (1 << 24) + 4
    assert np.float32(1.0) * np.float32(n - 1) == np.float32(n)
    for interp in O.INTERP:
        lo, hi, frac = O.ranks(1.0, 0, n, interp)
        assert lo == hi == n - 1 and frac == 0
    qs = [0.0, 0.1, 0.5, 0.9, 0.999999, 1.0]
    for count in list(range((1 << 24) - 2, (1 << 24) + 70)) + [(1 << 25) + 3, (1 << 30) + 1]:
        for ptr in (0, 1, (1 << 24) + 7):
            for q in qs:
                for interp in O.INTERP:
                    lo, hi, _ = O.ranks(q, ptr, count, interp)
                    assert 0 <= lo <= hi <= count - 1, (q, ptr, count, interp, lo, hi)


def test_keys_order_like_torch_sort():
    v = np.array([np.nan, np.inf, 1.0, 0.0, -0.0, -1.0, -np.inf, 3e-38, -3e-38, 2.5], dtype=np.float32)
    for bf16 in (False, True):
        vv = O.rnd(v, bf16)
        k = O.keys(vv, bf16)
        t = torch.from_numpy(vv).to(torch.bfloat16 if bf16 else torch.float32)
        order = torch.sort(t, stable=True).indices.numpy()
        assert (np.diff(k[order].astype(np.int64)) >= 0).all()
        assert k[3] == k[4] and k[0] > k[1]


def test_mirror_errors_state_and_repr_match_the_reference(tg):
    from torch_geometric.nn.aggr import MedianAggregation as TM
    from torch_geometric.nn.aggr import QuantileAggregation as TQ

    from pytorch_geometric_b200.nn import MedianAggregation, QuantileAggregation, aggregation_resolver
    for args in (([], ), ([0.5, 1.5], ), (-0.1, ), (0.5, "cubic")):
        with pytest.raises(ValueError) as theirs:
            TQ(*args)
        with pytest.raises(ValueError) as ours:
            QuantileAggregation(*args)
        assert str(ours.value) == str(theirs.value)
    for ctor in ((lambda m: m(0.3)), (lambda m: m([0.1, 0.9], "midpoint", 2.0))):
        a, b = ctor(TQ), ctor(QuantileAggregation)
        assert repr(a) == repr(b)
        sa, sb = a.state_dict(), b.state_dict()
        assert list(sa) == list(sb) == ["q"]
        assert sa["q"].dtype == sb["q"].dtype == torch.float32 and torch.equal(sa["q"], sb["q"])
        b.load_state_dict(sa)
    assert repr(TM()) == repr(MedianAggregation()) == "MedianAggregation()"
    assert torch.equal(TM().q, MedianAggregation().q) and MedianAggregation().interpolation == "lower"
    assert isinstance(aggregation_resolver("median"), MedianAggregation)
    r = aggregation_resolver("quantile", q=[0.2, 0.8], interpolation="nearest")
    assert isinstance(r, QuantileAggregation) and r.interpolation == "nearest" and r.q.shape == (2, 1)
    x = torch.randn(4, 3)
    with pytest.raises(NotImplementedError, match="requires 'index'"):
        TQ(0.5)(x, ptr=torch.tensor([0, 2, 4]))
    with pytest.raises(NotImplementedError, match="requires 'index'"):
        QuantileAggregation(0.5)(x, ptr=torch.tensor([0, 2, 4]))


def test_mirror_refuses_other_dtypes():
    from pytorch_geometric_b200.nn import MedianAggregation
    for dt in (torch.float16, torch.float64):
        with pytest.raises(TypeError):
            MedianAggregation()(torch.randn(4, 3).to(dt), torch.tensor([0, 0, 1, 1]), dim_size=2)


def test_install_rebinds_quantile_forward_and_cpu_falls_through(tg):
    from torch_geometric.nn.aggr import MedianAggregation as TM
    from torch_geometric.nn.aggr import QuantileAggregation as TQ

    from pytorch_geometric_b200 import plugin
    orig = TQ.forward
    x = torch.randn(12, 5, requires_grad=True)
    idx = torch.tensor([0, 0, 1, 1, 1, 2, 3, 3, 3, 3, 0, 2])
    mods = (TQ([0.25, 0.5], "linear", 3.0), TQ(0.7, "nearest"), TM())
    want = [m(x, idx, dim_size=5) for m in mods]
    gw = [torch.autograd.grad(w.sum(), x)[0] for w in want]
    try:
        c = plugin.install()
        assert c["quantile_aggregation"] == 1
        assert TQ.forward is not orig and TQ.forward.__wrapped__ is orig and TM.forward is TQ.forward
        for m, w, g in zip(mods, want, gw):
            got = m(x, idx, dim_size=5)
            assert torch.equal(got, w)
            assert torch.equal(torch.autograd.grad(got.sum(), x)[0], g)
    finally:
        plugin.uninstall()
    assert TQ.forward is orig


# The entry points' argument checks, with host buffers where device buffers are expected: anything that slips through
# fails at the launch without a device.
_ARGS_SKIP = pytest.mark.skipif(torch.cuda.is_available(), reason="passes host buffers as device pointers")
_BUF = np.zeros(1 << 12, dtype=np.uint8)
_P = _BUF.ctypes.data + (-_BUF.ctypes.data) % 16


def _fwd(**kw):
    import pytorch_geometric_b200 as pgb
    a = dict(rowptr=_P, col=_P, perm=None, x=_P, edge_rows=None, q=_P, n_q=1, interp=1, fill=0.0, out=_P, bits=None,
             n_rows=4, n_cols=4, n_edges=8, feat=8, plan_rows=None, plan_chunk_ptr=None, n_long=0, n_chunks=0,
             chunk=4, idx=1, val=0, stream=None)
    a.update(kw)
    return pgb.lib().b200mp_quantile_csr(*a.values())


@_ARGS_SKIP
@pytest.mark.parametrize("bad", [dict(n_q=0), dict(q=None), dict(interp=5), dict(interp=-1), dict(edge_rows=_P),
                                 dict(x=None), dict(n_long=-1), dict(n_long=1, n_chunks=1),
                                 dict(n_long=1, n_chunks=1, plan_rows=_P, plan_chunk_ptr=_P, chunk=0)],
                         ids=["no_q", "null_q", "interp_high", "interp_low", "both_forms", "no_form", "negative_long",
                              "no_plan_rows", "zero_chunk"])
def test_quantile_csr_rejects_bad_arguments(bad):
    assert _fwd(**bad) == -1


@_ARGS_SKIP
def test_quantile_csr_valid_arguments_pass_the_checks():
    assert _fwd() != -1
    assert _fwd(n_long=1, n_chunks=1, plan_rows=_P, plan_chunk_ptr=_P) != -1


def test_bits_words():
    import pytorch_geometric_b200 as pgb
    f = pgb.lib().b200mp_quantile_bits_words
    assert f(10, 3, 0, 64) == 10 * 2 * 3 * 2 and f(10, 3, 1, 65) == 10 * 3 * 3 and f(0, 1, 4, 8) == 0
    assert f(10, 0, 1, 8) == -1 and f(10, 1, 5, 8) == -1
