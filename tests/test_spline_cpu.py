"""CPU checks of SplineConv on the engine: the fp64 oracle of the B-spline basis (tests/spline_oracle.py) against the
worked anchors of its convention, partition of unity and finite-difference derivatives; the standalone `nn.SplineConv`
mirror's checkpoint layout, buffers, initialisation and repr against the reference; and the plug-in's binding of
`spline_basis` / `spline_weighting`, its WITH_SPLINE flag, and the fusability predicate with every hook that disables
it.  No engine compute runs here."""
import json
import os
import sys

import numpy as np
import pytest
import torch

sys.path.insert(0, os.path.dirname(os.path.abspath(__file__)))
import spline_oracle as SO  # noqa: E402

from pytorch_geometric_b200.nn import SplineConv  # noqa: E402

# (degree, kernel_size, is_open_spline, pseudo) -> [(weight_index, basis)] per slot, in slot order
ANCHORS = [(1, [5], [1], [0.3], [(1, 0.8), (2, 0.2)]),
           (1, [5, 5], [1, 1], [0.3, 0.9], [(16, 0.32), (17, 0.08), (21, 0.48), (22, 0.12)]),
           (1, [4], [0], [0.9], [(3, 0.4), (0, 0.6)]),
           (1, [5], [1], [1.0], [(4, 1.0), (0, 0.0)]),
           (2, [5], [1], [0.5], [(1, 0.125), (2, 0.75), (3, 0.125)]),
           (3, [5], [1], [0.5], [(1, 1 / 6), (2, 2 / 3), (3, 1 / 6), (4, 0)])]


@pytest.mark.parametrize("degree,ks,op,pseudo,want", ANCHORS)
def test_oracle_reproduces_the_anchor_table(degree, ks, op, pseudo, want):
    b, wi = SO.spline_basis(np.asarray([pseudo], dtype=np.float32), ks, op, degree)
    assert wi[0].tolist() == [w for w, _ in want]
    np.testing.assert_allclose(b[0], [v for _, v in want], rtol=0, atol=1e-6)


CASES = [(d, deg, ks, op) for deg in (1, 2, 3)
         for d, ks, op in ((1, [7], [1]), (2, [5, 3], [1, 0]), (3, [4, 6, 5], [0, 1, 1]))]


@pytest.mark.parametrize("dim,degree,ks,op", CASES)
def test_oracle_partition_of_unity_and_indices_in_range(dim, degree, ks, op):
    p = np.random.default_rng(dim * 10 + degree).random((500, dim)).astype(np.float32)
    p[:3] = 0.0
    p[3:6] = 1.0
    b, wi = SO.spline_basis(p, ks, op, degree)
    np.testing.assert_allclose(b.sum(1), 1.0, rtol=0, atol=1e-12)
    assert wi.min() >= 0 and wi.max() < int(np.prod(ks))


@pytest.mark.parametrize("dim,degree,ks,op", CASES)
def test_oracle_derivative_matches_finite_differences_away_from_knots(dim, degree, ks, op):
    rng = np.random.default_rng(dim + 7 * degree)
    scale = np.asarray(ks) - degree * np.asarray(op)
    # pseudo-coordinates whose v = pseudo * scale sits at least 0.1 away from an integer knot
    v = rng.integers(0, scale, size=(200, dim)) + 0.1 + 0.8 * rng.random((200, dim))
    p = (v / scale).astype(np.float32)
    g = rng.standard_normal((200, (degree + 1) ** dim))
    got = SO.spline_basis_grad(g, p, ks, op, degree)
    h = 1e-5
    for d in range(dim):
        hi, lo = p.astype(np.float64).copy(), p.astype(np.float64).copy()
        hi[:, d] += h
        lo[:, d] -= h
        # fp64 central difference on the basis pieces (the oracle's v is fp32; restate it in fp64 here)
        fd = (_basis64(hi, ks, op, degree) - _basis64(lo, ks, op, degree)) / (2 * h)
        np.testing.assert_allclose(got[:, d], (fd * g).sum(1), rtol=1e-5, atol=1e-5)


def _basis64(p, ks, op, degree):
    scale = np.asarray(ks, dtype=np.float64) - degree * np.asarray(op)
    v = p * scale[None, :]
    t = v - np.floor(v)
    E, D = p.shape
    out = np.ones((E, (degree + 1) ** D))
    for s in range(out.shape[1]):
        for d, km in enumerate(SO._digits(s, D, degree)):
            out[:, s] *= SO.piece(degree, t[:, d], km)
    return out


def test_torch_oracle_equals_the_numpy_oracle():
    p = torch.rand(300, 2)
    b, wi = SO.torch_spline_basis(p.double(), torch.tensor([5, 4]), torch.tensor([1, 0], dtype=torch.uint8), 2)
    nb, nwi = SO.spline_basis(p.numpy(), [5, 4], [1, 0], 2)
    assert np.array_equal(wi.numpy(), nwi)
    np.testing.assert_allclose(b.numpy(), nb, rtol=0, atol=1e-12)


# ---------------------------------------------------------------------------------------------- the mirror
GOLDEN = [("faust_add", 8, 8, 3, {"kernel_size": 5, "aggr": "add"}),
          ("mnist_mean", 1, 16, 2, {"kernel_size": 5, "aggr": "mean"}),
          ("deg2_mixed", 6, 4, 2, {"kernel_size": [3, 4], "is_open_spline": [True, False], "degree": 2}),
          ("bipartite", (8, 16), 8, 2, {"kernel_size": 3, "aggr": "add"}),
          ("no_root_no_bias", 4, 8, 2, {"kernel_size": 4, "root_weight": False, "bias": False}),
          ("deg3_isolated", 4, 6, 1, {"kernel_size": 6, "degree": 3, "aggr": "mean"})]


@pytest.mark.parametrize("tag,ch,f_out,dim,kw", GOLDEN)
def test_mirror_layout_and_repr_match_golden(golden, tag, ch, f_out, dim, kw):
    z = golden("spline")
    mine = SplineConv(ch, f_out, dim, **kw)
    assert {n: list(p.shape) for n, p in mine.state_dict().items()} == json.loads(str(z[f"{tag}_shapes"]))
    assert list(mine.state_dict()) == list(json.loads(str(z[f"{tag}_shapes"])))
    assert repr(mine) == str(z[f"{tag}_repr"])
    state = {key[len(tag) + 3:]: torch.from_numpy(v) for key, v in z.items() if key.startswith(f"{tag}_p_")}
    for name in ("kernel_size", "is_open_spline"):
        assert torch.equal(mine.state_dict()[name], state[name])
    mine.load_state_dict(state)


@pytest.fixture
def placeholder(tg):
    """The reference's spline module with a placeholder bound, so that its constructor runs without pyg-lib."""
    import torch_geometric.nn.conv.spline_conv as S
    saved = S.spline_basis, S.spline_weighting
    S.spline_basis, S.spline_weighting = SO.torch_spline_basis, SO.torch_spline_weighting
    yield S
    S.spline_basis, S.spline_weighting = saved


@pytest.mark.parametrize("ch,f_out,dim,kw", [(8, 16, 3, {"kernel_size": 5}), ((4, 6), 3, 2, {"kernel_size": [3, 5]}),
                                             (2, 4, 1, {"kernel_size": 4, "root_weight": False, "bias": False})])
def test_mirror_initialises_as_the_reference(placeholder, ch, f_out, dim, kw):
    torch.manual_seed(3)
    ref = placeholder.SplineConv(ch, f_out, dim, **kw)
    torch.manual_seed(3)
    mine = SplineConv(ch, f_out, dim, **kw)
    assert repr(mine) == repr(ref) and mine.K == ref.K
    rs, ms = ref.state_dict(), mine.state_dict()
    assert list(rs) == list(ms)
    for k in rs:
        assert torch.equal(rs[k], ms[k]), k


@pytest.mark.parametrize("kw,match", [({"aggr": "max"}, "aggr"), ({"degree": 4}, "degree"),
                                      ({"kernel_size": 129}, "outside"), ({"in_channels": -1}, "lazy")])
def test_mirror_refuses_what_it_does_not_fuse(kw, match):
    kw = dict(kw)
    ch = kw.pop("in_channels", 128)
    with pytest.raises(ValueError, match=match):
        SplineConv(ch, 4, 2, **{"kernel_size": 5, **kw})


# ---------------------------------------------------------------------------------------------- the plug-in
@pytest.fixture
def plugin(tg):
    from pytorch_geometric_b200 import plugin as P
    yield P
    P.uninstall()


def test_install_binds_the_spline_ops_and_flag_and_uninstall_restores(tg, plugin):
    import torch_geometric.nn.conv.spline_conv as S
    import torch_geometric.typing as T
    assert S.spline_basis is None and S.spline_weighting is None and T.WITH_SPLINE is False
    c = plugin.install(layers=True, flip_flags=True)
    assert c["spline_ops"] == 2 and c["spline_flag"] == 1 and T.WITH_SPLINE is True
    assert S.spline_basis.__name__ == "_pl_spline_basis" and S.spline_weighting.__name__ == "_pl_spline_weighting"
    from torch_geometric.nn.conv.spline_conv import SplineConv as Ref
    from pytorch_geometric_b200.plugin import conv as PC
    assert tg.nn.SplineConv is PC.B200SplineConv and issubclass(PC.B200SplineConv, Ref)
    tg.nn.SplineConv(4, 4, 2, kernel_size=3)                              # the constructor no longer raises
    plugin.uninstall()
    assert S.spline_basis is None and S.spline_weighting is None and T.WITH_SPLINE is False
    assert tg.nn.SplineConv is Ref
    with pytest.raises(ImportError, match="pyg-lib"):
        tg.nn.SplineConv(4, 4, 2, kernel_size=3)
    c = plugin.install()
    assert c["spline_ops"] == 2 and "spline_flag" not in c and T.WITH_SPLINE is False


def test_pyg_lib_shim_has_the_spline_ops(plugin):
    from pytorch_geometric_b200.plugin import shims
    m = shims.pyg_lib_module()
    assert callable(m.ops.spline_basis) and callable(m.ops.spline_weighting)
    with pytest.raises(RuntimeError, match="CUDA float32 / bfloat16"):
        m.ops.spline_basis(torch.rand(3, 2), torch.tensor([5, 5]), torch.tensor([1, 1], dtype=torch.uint8), 1)


def _fusable(plugin, conv, x, ei, ea):
    from pytorch_geometric_b200.plugin import conv as PC
    return PC._spline_fusable(conv, PC._pair(x), ei, ea)


@pytest.fixture
def layer(tg, plugin, monkeypatch):
    plugin.install(layers=True)
    from pytorch_geometric_b200.plugin import routing
    conv = tg.nn.SplineConv(4, 6, 2, kernel_size=5)
    x, ei, ea = torch.randn(10, 4), torch.tensor([[0, 1, 2], [1, 2, 3]]), torch.rand(3, 2)
    # the predicate's device and dtype check, with CPU tensors standing in for CUDA ones
    monkeypatch.setattr(routing, "engine_ok", lambda t: t.dtype in (torch.float32, torch.bfloat16))
    return conv, x, ei, ea


def test_fusable_predicate_covers_the_fused_configuration(tg, plugin, layer):
    conv, x, ei, ea = layer
    assert _fusable(plugin, conv, x, ei, ea)
    assert _fusable(plugin, conv, (x, None), ei, ea)
    assert not _fusable(plugin, conv, x, ei, None)                        # no pseudo-coordinates
    assert not _fusable(plugin, conv, x, ei, ea[:, :1])                   # edge_attr narrower than dim
    assert not _fusable(plugin, conv, x, ei, ea.double())                 # mixed dtypes
    assert not _fusable(plugin, conv, x.half(), ei, ea.half())
    sp = torch.sparse_coo_tensor(ei, torch.ones(3), (10, 10))
    assert not _fusable(plugin, conv, x, sp, ea)
    with torch.autocast("cpu", dtype=torch.bfloat16):
        assert not _fusable(plugin, conv, x, ei, ea)
    big = tg.nn.SplineConv(128, 4, 2, kernel_size=12)                     # K F_in = 18432 > 16384
    assert not _fusable(plugin, big, torch.randn(10, 128), ei, ea)
    mx = tg.nn.SplineConv(4, 6, 2, kernel_size=5, aggr="max")
    assert not _fusable(plugin, mx, x, ei, ea)


@pytest.mark.parametrize("hook", ["propagate_pre", "propagate", "message_pre", "message", "aggregate_pre", "aggregate",
                                  "explain", "decomposed"])
def test_every_hook_disables_the_fused_path(tg, plugin, layer, hook):
    conv, x, ei, ea = layer
    fn = {"propagate_pre": conv.register_propagate_forward_pre_hook, "propagate": conv.register_propagate_forward_hook,
          "message_pre": conv.register_message_forward_pre_hook, "message": conv.register_message_forward_hook,
          "aggregate_pre": conv.register_aggregate_forward_pre_hook, "aggregate": conv.register_aggregate_forward_hook}
    if hook in fn:
        fn[hook](lambda *a: None)
    elif hook == "explain":
        conv.explain = True
    else:
        conv.decomposed_layers = 2
    assert not _fusable(plugin, conv, x, ei, ea)
