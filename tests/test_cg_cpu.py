"""CPU checks of the CGConv layers: the standalone `nn.CGConv` mirror's checkpoint layout, repr and errors against the
golden data of the reference, `plugin.conv.B200CGConv` falling through bit for bit on CPU tensors (hooks included),
and the fusability predicate."""
import copy
import json

import pytest
import torch

from pytorch_geometric_b200.nn import CGConv

GOLDEN_CASES = [("plain", 16, {}), ("bip_mean_bn", (8, 16), dict(dim=5, aggr="mean", batch_norm=True)),
                ("narrow", 6, dict(dim=3, bias=False))]


@pytest.mark.parametrize("tag,ch,kw", GOLDEN_CASES)
def test_mirror_layout_and_repr_match_golden(golden, tag, ch, kw):
    z = golden("cg")
    mine = CGConv(ch, **kw)
    assert {n: list(p.shape) for n, p in mine.state_dict().items()} == json.loads(str(z[f"{tag}_shapes"]))
    assert repr(mine) == str(z[f"{tag}_repr"])
    mine.load_state_dict({k[len(tag) + 3:]: torch.from_numpy(v) for k, v in z.items() if k.startswith(f"{tag}_p_")})


@pytest.mark.parametrize("aggr", ["max", "min", ["sum", "mean"]])
def test_mirror_rejects_aggregations_it_does_not_fuse(aggr):
    with pytest.raises(ValueError, match="aggr"):
        CGConv(8, aggr=aggr)


def test_mirror_accepts_sum_add_and_mean():
    assert CGConv(8, aggr="sum").aggr == "sum" and CGConv(8).aggr == "sum" and CGConv(8, aggr="mean").aggr == "mean"


def _b200(ref):
    from pytorch_geometric_b200.plugin import conv as PC
    mine = copy.deepcopy(ref)
    mine.__class__ = PC.B200CGConv
    return mine


@pytest.mark.parametrize("ch,kw,bip", [(16, {}, False), ((8, 16), dict(dim=5, aggr="mean", batch_norm=True), True),
                                       (6, dict(dim=3, bias=False), False)])
def test_b200_cg_on_cpu_is_the_reference(tg, ch, kw, bip):
    torch.manual_seed(0)
    ref = tg.nn.CGConv(ch, **kw)
    mine = _b200(ref)
    f_src, f_dst = (ch, ch) if isinstance(ch, int) else ch
    x = torch.randn(10, f_src)
    x_in = (x, torch.randn(7, f_dst)) if bip else x
    ei = torch.stack([torch.randint(0, 10, (30, )), torch.randint(0, 7 if bip else 10, (30, ))])
    ea = torch.randn(30, kw["dim"]) if kw.get("dim") else None
    assert torch.equal(mine(x_in, ei, ea), ref(x_in, ei, ea))
    assert list(mine.state_dict()) == list(ref.state_dict())
    assert all(torch.equal(a, b) for a, b in zip(mine.state_dict().values(), ref.state_dict().values()))


def test_registered_hook_fires(tg):
    mine = _b200(tg.nn.CGConv(8, dim=2))
    seen = []
    mine.register_message_forward_hook(lambda mod, inp, out: seen.append(out.shape))
    mine(torch.randn(5, 8), torch.randint(0, 5, (2, 11)), torch.randn(11, 2))
    assert seen == [torch.Size([11, 8])]


def test_layer_is_registered():
    from pytorch_geometric_b200.plugin import conv as PC
    assert "CGConv" in PC.LAYERS and PC.LAYERS["CGConv"] == "B200CGConv"


def test_fusability_predicate(tg, monkeypatch):
    from pytorch_geometric_b200.plugin import conv as PC
    from pytorch_geometric_b200.plugin import routing
    monkeypatch.setattr(routing, "engine_ok", lambda t: True)       # stand in for a CUDA tensor
    x, ea = torch.randn(10, 16), torch.randn(30, 3)
    xs = (x, x)

    def layer(**kw):
        return _b200(tg.nn.CGConv(16, **{"dim": 3, **kw}))
    assert PC._cg_fusable(layer(), xs, ea)
    assert PC._cg_fusable(layer(aggr="mean"), xs, ea)
    assert PC._cg_fusable(layer(aggr=tg.nn.aggr.SumAggregation()), xs, ea)
    assert PC._cg_fusable(layer(flow="target_to_source", batch_norm=True), xs, ea)
    assert PC._cg_fusable(layer(dim=0), xs, None)
    assert not PC._cg_fusable(layer(aggr="max"), xs, ea)
    assert not PC._cg_fusable(layer(aggr=["sum", "mean"]), xs, ea)
    assert not PC._cg_fusable(layer(aggr=tg.nn.aggr.SoftmaxAggregation()), xs, ea)
    assert not PC._cg_fusable(layer(), (x, None), ea)
    assert not PC._cg_fusable(layer(), xs, None)                     # dim > 0 without edge_attr
    assert not PC._cg_fusable(layer(dim=0), xs, ea)                  # edge_attr with dim = 0
    assert not PC._cg_fusable(layer(), xs, torch.randn(30, 4))       # edge_attr of the wrong width
    m = layer()
    m.register_message_forward_hook(lambda mod, inp, out: out)
    assert not PC._cg_fusable(m, xs, ea)
    m = layer()
    m.explain = True
    assert not PC._cg_fusable(m, xs, ea)
    m = layer()
    m.decomposed_layers = 2
    assert not PC._cg_fusable(m, xs, ea)
    monkeypatch.setattr(routing, "_compiling", lambda: True)
    assert not PC._cg_fusable(layer(), xs, ea)
    monkeypatch.setattr(routing, "_compiling", lambda: False)
    m = layer()
    assert PC._cg_fusable(m, xs, ea)
    monkeypatch.setattr(torch.jit, "is_scripting", lambda: True)
    assert not PC._cg_fusable(m, xs, ea)


def test_fusability_predicate_needs_cuda_float32_or_bfloat16(tg):
    from pytorch_geometric_b200.plugin import conv as PC
    m = _b200(tg.nn.CGConv(16, dim=3))
    ea = torch.randn(30, 3)
    for dt in (torch.float32, torch.float16, torch.float64):          # CPU in any dtype; CUDA fp16 / fp64 likewise
        x = torch.randn(10, 16, dtype=dt)
        assert not PC._cg_fusable(m, (x, x), ea.to(dt))
