"""CPU-side checks of the gated message path (ResGatedGraphConv's sigmoid(k_i + q_j) * v_j): the GatedRows fold
rules, built directly on CPU tensors, and the standalone ResGatedGraphConv mirror's checkpoint layout, argument errors
and repr."""
import json

import pytest
import torch
import torch.nn.functional as F

from pytorch_geometric_b200.nn import ResGatedGraphConv
from pytorch_geometric_b200.plugin.lazy import GatedRows, LazyRows

N, E, FEAT = 7, 12, 5


def _inputs(dtype=torch.float32):
    g = torch.Generator().manual_seed(5)
    k, q, v = (torch.randn(N, FEAT, generator=g).to(dtype) for _ in range(3))
    i = torch.randint(0, N, (E, ), generator=g)
    j = torch.randint(0, N, (E, ), generator=g)
    return k, q, v, i, j


def _same(got, want):
    assert type(got) is torch.Tensor, type(got)
    assert got.dtype == want.dtype and got.shape == want.shape
    assert torch.equal(got, want) or torch.equal(got.isnan(), want.isnan()) and torch.equal(
        got.nan_to_num(), want.nan_to_num())


def _ref(k, q, v, i, j):
    return torch.sigmoid(k.index_select(0, i) + q.index_select(0, j)) * v.index_select(0, j)


_ADD = {"a+b": lambda a, b: a + b, "b+a": lambda a, b: b + a, "torch.add": torch.add, "Tensor.add": lambda a, b: a.add(b)}
_SIG = {"Tensor.sigmoid": lambda s: s.sigmoid(), "torch.sigmoid": torch.sigmoid, "F.sigmoid": F.sigmoid,
        "nn.Sigmoid": torch.nn.Sigmoid()}
_MUL = {"gate*v": lambda g, v: g * v, "v*gate": lambda g, v: v * g, "torch.mul": torch.mul}


@pytest.mark.parametrize("add", list(_ADD))
@pytest.mark.parametrize("sig", list(_SIG))
@pytest.mark.parametrize("mul", list(_MUL))
def test_sum_sigmoid_product_fold(add, sig, mul):
    k, q, v, i, j = _inputs()
    ki, qj, vj = LazyRows(k, i), LazyRows(q, j), LazyRows(v, j)
    s = _ADD[add](ki, qj)
    assert isinstance(s, GatedRows) and s._stage == "sum" and {id(s._a), id(s._b)} == {id(ki), id(qj)}
    gate = _SIG[sig](s)
    assert isinstance(gate, GatedRows) and gate._stage == "gate"
    m = _MUL[mul](gate, vj)
    assert isinstance(m, GatedRows) and m._stage == "message" and m._v is vj
    assert isinstance(m, LazyRows)                     # every isinstance(x, LazyRows) site in routing.py sees it
    _same(m.materialise(), _ref(k, q, v, i, j))
    # the pending stages materialise as the reference's partial results
    _same(s.materialise(), k.index_select(0, i) + q.index_select(0, j))
    _same(gate.materialise(), torch.sigmoid(k.index_select(0, i) + q.index_select(0, j)))


def _cases():
    k, q, v, i, j = _inputs()
    ki, qj, vj = k.index_select(0, i), q.index_select(0, j), v.index_select(0, j)
    w = torch.rand(E)
    t = torch.randn(E, FEAT)
    return {
        "relu_gate": (lambda K, Q, V: (K + Q).relu() * V, lambda: (ki + qj).relu() * vj),
        "tanh_gate": (lambda K, Q, V: torch.tanh(K + Q) * V, lambda: torch.tanh(ki + qj) * vj),
        "sigmoid_": (lambda K, Q, V: (K + Q).sigmoid_() * V, lambda: (ki + qj).sigmoid_() * vj),
        "sigmoid_out": (lambda K, Q, V: torch.sigmoid(K + Q, out=torch.empty(E, FEAT)) * V,
                        lambda: torch.sigmoid(ki + qj) * vj),
        "gate_times_plain": (lambda K, Q, V: torch.sigmoid(K + Q) * t, lambda: torch.sigmoid(ki + qj) * t),
        "gate_times_weight": (lambda K, Q, V: torch.sigmoid(K + Q) * w.view(-1, 1), lambda: torch.sigmoid(ki + qj) * w.view(-1, 1)),
        "three_way_add": (lambda K, Q, V: torch.sigmoid(K + Q + V) * V, lambda: torch.sigmoid(ki + qj + vj) * vj),
        "sub": (lambda K, Q, V: torch.sigmoid(K - Q) * V, lambda: torch.sigmoid(ki - qj) * vj),
        "scaled_lazy": (lambda K, Q, V: torch.sigmoid(w.view(-1, 1) * K + Q) * V,
                        lambda: torch.sigmoid(w.view(-1, 1) * ki + qj) * vj),
        "gate_times_scaled_v": (lambda K, Q, V: torch.sigmoid(K + Q) * (w.view(-1, 1) * V),
                                lambda: torch.sigmoid(ki + qj) * (w.view(-1, 1) * vj)),
        "gate_times_gate": (lambda K, Q, V: torch.sigmoid(K + Q) * torch.sigmoid(K + Q),
                            lambda: torch.sigmoid(ki + qj) * torch.sigmoid(ki + qj)),
        "message_plus_eps": (lambda K, Q, V: torch.sigmoid(K + Q) * V + 1e-7, lambda: torch.sigmoid(ki + qj) * vj + 1e-7),
        "sum_times_v": (lambda K, Q, V: (K + Q) * V, lambda: (ki + qj) * vj),
        "mixed_dtype_sum": (lambda K, Q, V: torch.sigmoid(K + LazyRows(q.double(), j)) * V,
                            lambda: torch.sigmoid(ki + qj.double()) * vj),
        "mixed_dtype_v": (lambda K, Q, V: torch.sigmoid(K + Q) * LazyRows(v.double(), j),
                          lambda: torch.sigmoid(ki + qj) * vj.double()),
        "alpha": (lambda K, Q, V: torch.sigmoid(torch.add(K, Q, alpha=2.0)) * V,
                  lambda: torch.sigmoid(torch.add(ki, qj, alpha=2.0)) * vj),
        "max_reduce": (lambda K, Q, V: (torch.sigmoid(K + Q) * V).max(dim=0).values,
                       lambda: (torch.sigmoid(ki + qj) * vj).max(dim=0).values),
    }


@pytest.mark.parametrize("case", list(_cases()))
def test_other_operations_materialise_exactly_as_the_reference(case):
    k, q, v, i, j = _inputs()
    fn, ref = _cases()[case]
    got = fn(LazyRows(k, i), LazyRows(q, j), LazyRows(v, j))
    _same(got, ref())


def test_existing_add_fold_is_unchanged():
    k, q, v, i, j = _inputs()
    t = torch.randn(E, FEAT)
    lz = LazyRows(q, j) + t                        # GINEConv's fold still applies to a plain tensor
    assert type(lz) is LazyRows and lz._add is t
    s = (LazyRows(q, j) + t).sigmoid()             # and its sigmoid still materialises
    _same(s, (q.index_select(0, j) + t).sigmoid())


def test_bf16_fold_and_materialise():
    k, q, v, i, j = _inputs(torch.bfloat16)
    m = torch.sigmoid(LazyRows(k, i) + LazyRows(q, j)) * LazyRows(v, j)
    assert isinstance(m, GatedRows) and m._stage == "message"
    _same(m.materialise(), _ref(k, q, v, i, j))
    # a fp32 v with bf16 k and q does not fold and keeps the reference's promotion
    got = torch.sigmoid(LazyRows(k, i) + LazyRows(q, j)) * LazyRows(v.float(), j)
    _same(got, torch.sigmoid(k.index_select(0, i) + q.index_select(0, j)) * v.float().index_select(0, j))


_GOLDEN_CASES = [("plain", 16, 32, {}), ("mean_bip", (16, 24), 32, {"aggr": "mean", "root_weight": False}),
                 ("narrow", 16, 6, {"bias": False})]


@pytest.mark.parametrize("tag,ic,oc,kw", _GOLDEN_CASES)
def test_res_gated_state_dict_and_repr_match_reference(golden, tag, ic, oc, kw):
    z = golden("res_gated")
    want = json.loads(str(z[f"{tag}_shapes"]))
    conv = ResGatedGraphConv(ic, oc, **kw)
    assert {k: list(v.shape) for k, v in conv.state_dict().items()} == want
    conv.load_state_dict({k: torch.from_numpy(z[f"{tag}_p_{k}"]) for k in want})    # strict
    assert repr(conv) == str(z[f"{tag}_repr"])
    assert list(dict(conv.named_parameters())) == [k for k in want]


def test_res_gated_argument_errors():
    with pytest.raises(ValueError, match="edge_dim"):
        ResGatedGraphConv(8, 4, edge_dim=3)
    with pytest.raises(ValueError, match="act="):
        ResGatedGraphConv(8, 4, act=torch.nn.Tanh())
    for aggr in ("max", "min", "mul", "softmax"):
        with pytest.raises(ValueError, match=f"aggr='{aggr}'"):
            ResGatedGraphConv(8, 4, aggr=aggr)
    for act in (torch.sigmoid, F.sigmoid, torch.nn.Sigmoid()):
        ResGatedGraphConv(8, 4, act=act)
    for aggr in ("add", "sum", "mean"):
        ResGatedGraphConv(8, 4, aggr=aggr)
    assert repr(ResGatedGraphConv(8, 32)) == "ResGatedGraphConv(8, 32)"
    assert repr(ResGatedGraphConv((8, 32), 32)) == "ResGatedGraphConv((8, 32), 32)"
    # no CPU fallback
    with pytest.raises(RuntimeError, match="CUDA"):
        ResGatedGraphConv(8, 4)(torch.randn(4, 8), torch.tensor([[0, 1, 2], [1, 2, 3]]))
