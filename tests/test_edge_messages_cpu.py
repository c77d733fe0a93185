"""CPU-side checks of the edge-feature message path (GINEConv's relu(x_j + e_ji)): the LazyRows fold rules, built
directly on CPU tensors, and the standalone GINEConv mirror's checkpoint layout and argument errors."""
import json

import pytest
import torch
import torch.nn.functional as F

from pytorch_geometric_b200.nn import GINEConv
from pytorch_geometric_b200.plugin.lazy import LazyRows

N, E, FEAT = 7, 12, 5


def _inputs(dtype=torch.float32):
    g = torch.Generator().manual_seed(3)
    x = torch.randn(N, FEAT, generator=g).to(dtype)
    idx = torch.randint(0, N, (E, ), generator=g)
    t = torch.randn(E, FEAT, generator=g).to(dtype)
    return x, idx, t


def _same(got, want):
    assert type(got) is torch.Tensor, type(got)
    assert got.dtype == want.dtype and got.shape == want.shape
    assert torch.equal(got, want) or torch.equal(got.isnan(), want.isnan()) and torch.equal(
        got.nan_to_num(), want.nan_to_num())


@pytest.mark.parametrize("form", ["lazy+t", "t+lazy", "torch.add", "Tensor.add"])
@pytest.mark.parametrize("act", ["Tensor.relu", "torch.relu", "F.relu"])
def test_add_then_relu_folds(form, act):
    x, idx, t = _inputs()
    lz = LazyRows(x, idx)
    added = {"lazy+t": lambda: lz + t, "t+lazy": lambda: t + lz, "torch.add": lambda: torch.add(lz, t),
             "Tensor.add": lambda: lz.add(t)}[form]()
    assert isinstance(added, LazyRows) and added._add is t and not added._relu
    r = {"Tensor.relu": lambda a: a.relu(), "torch.relu": torch.relu, "F.relu": F.relu}[act](added)
    assert isinstance(r, LazyRows) and r._add is t and r._relu and r._scale is None
    _same(r.materialise(), (x.index_select(0, idx) + t).relu())


def _cases():
    x, idx, t = _inputs()
    w = torch.rand(E)
    xj = x.index_select(0, idx)
    return {
        # mismatched dtype: the reference's type promotion (fp32 + fp64 -> fp64)
        "dtype": (lambda lz: lz + t.double(), lambda: xj + t.double()),
        # broadcast rows
        "broadcast": (lambda lz: lz + t[0], lambda: xj + t[0]),
        "broadcast_E1": (lambda lz: lz + t[:, :1], lambda: xj + t[:, :1]),
        "alpha": (lambda lz: torch.add(lz, t, alpha=2.0), lambda: torch.add(xj, t, alpha=2.0)),
        "inplace_add": (lambda lz: lz.add_(t), lambda: xj.clone().add_(t)),
        "inplace_relu": (lambda lz: F.relu(lz + t, inplace=True), lambda: F.relu(xj + t)),
        "relu_": (lambda lz: (lz + t).relu_(), lambda: (xj + t).relu_()),
        "mul_after_add": (lambda lz: (lz + t) * w.view(-1, 1), lambda: (xj + t) * w.view(-1, 1)),
        "eps_after_relu": (lambda lz: (lz + t).relu() + 1e-7, lambda: (xj + t).relu() + 1e-7),
        "sigmoid": (lambda lz: (lz + t).sigmoid(), lambda: (xj + t).sigmoid()),
        "relu_without_add": (lambda lz: lz.relu(), lambda: xj.relu()),
        "add_after_scale": (lambda lz: (w.view(-1, 1) * lz) + t, lambda: (w.view(-1, 1) * xj) + t),
        "second_add": (lambda lz: (lz + t) + t, lambda: (xj + t) + t),
        "max_reduce": (lambda lz: (lz + t).relu().max(dim=0).values, lambda: (xj + t).relu().max(dim=0).values),
        "sub": (lambda lz: lz - t, lambda: xj - t),
        "parameter": (lambda lz: lz + torch.nn.Parameter(t.clone()), lambda: xj + t),
    }


@pytest.mark.parametrize("case", list(_cases()))
def test_other_operations_materialise_exactly_as_the_reference(case):
    x, idx, _ = _inputs()
    fn, ref = _cases()[case]
    got = fn(LazyRows(x, idx))
    want = ref()
    if case == "parameter":
        got = got.detach()
    _same(got, want)


def test_mul_fold_refuses_a_lazy_carrying_an_add():
    x, idx, t = _inputs()
    w = torch.rand(E)
    lz = LazyRows(x, idx) + t
    assert isinstance(lz, LazyRows)
    assert lz._scaled_by(w) is None
    assert lz._scaled_by(w.view(-1, 1)) is None
    got = w.view(-1, 1) * lz
    _same(got, w.view(-1, 1) * (x.index_select(0, idx) + t))
    # a lazy without an add still folds its scale, as before
    s = LazyRows(x, idx) * w.view(-1, 1)
    assert isinstance(s, LazyRows) and s._add is None and torch.equal(s._scale, w)


def test_bf16_fold_and_materialise():
    x, idx, t = _inputs(torch.bfloat16)
    r = (LazyRows(x, idx) + t).relu()
    assert isinstance(r, LazyRows)
    _same(r.materialise(), (x.index_select(0, idx) + t).relu())
    # fp32 edge rows with bf16 x do not fold and keep the reference's promotion to fp32
    got = LazyRows(x, idx) + t.float()
    _same(got, x.index_select(0, idx) + t.float())


def _mlp():
    return torch.nn.Sequential(torch.nn.Linear(8, 16), torch.nn.ReLU(), torch.nn.Linear(16, 8))


@pytest.mark.parametrize("tag,kw", [("plain", {}), ("edge_dim", {"edge_dim": 5, "train_eps": True, "eps": 0.25}),
                                    ("mean_bip", {"aggr": "mean", "eps": -0.5})])
def test_gine_state_dict_matches_reference_layout(golden, tag, kw):
    z = golden("gine")
    want = json.loads(str(z[f"{tag}_shapes"]))
    conv = GINEConv(_mlp(), **kw)
    assert {k: list(v.shape) for k, v in conv.state_dict().items()} == want
    # a reference checkpoint loads strictly and carries its values
    conv.load_state_dict({k: torch.from_numpy(z[f"{tag}_p_{k}"]) for k in want})
    assert float(conv.eps.detach()) == kw.get("eps", 0.0)
    assert isinstance(conv.eps, torch.nn.Parameter) == kw.get("train_eps", False)


def test_gine_argument_errors_match_reference_messages():
    x = torch.randn(4, 8)
    ei = torch.tensor([[0, 1, 2], [1, 2, 3]])
    with pytest.raises(ValueError, match="Node and edge feature dimensionalities do not match"):   # gin_conv.py:197-200
        GINEConv(_mlp())(x, ei, torch.randn(3, 5))
    with pytest.raises(ValueError, match="Could not infer input channels from `nn`."):             # gin_conv.py:157
        GINEConv(torch.nn.ReLU(), edge_dim=3)
    assert GINEConv(torch.nn.Linear(8, 4), edge_dim=3).lin.weight.shape == (8, 3)
    assert repr(GINEConv(torch.nn.Linear(8, 4))) == "GINEConv(nn=Linear(in_features=8, out_features=4, bias=True))"
    # no CPU fallback
    with pytest.raises(RuntimeError, match="CUDA"):
        GINEConv(_mlp())(x, ei, torch.randn(3, 8))
