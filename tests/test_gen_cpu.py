"""CPU tests of the power-mean aggregation and the fused GENConv: PowerMeanAggregation's constructor errors, parameters
and repr against the reference, aggregation_resolver('powermean'), B200GENConv in plugin.conv.LAYERS and falling
through to the reference bit for bit on CPU tensors and with hooks, and the fusability predicates case by case."""
import pytest
import torch

from pytorch_geometric_b200.nn import PowerMeanAggregation, aggregation_resolver
from pytorch_geometric_b200.nn.aggr import power_mean_fusable


def test_module_errors_parameters_and_repr(tg):
    from torch_geometric.nn.aggr import PowerMeanAggregation as RefPM
    with pytest.raises(ValueError, match="Cannot set 'channels' greater than '1'"):
        PowerMeanAggregation(channels=4)
    with pytest.raises(ValueError, match="Cannot set 'channels' greater than '1'"):
        RefPM(channels=4)
    for kw in (dict(), dict(p=2.5), dict(learn=True, channels=8, p=0.7)):
        ref, ours = RefPM(**kw), PowerMeanAggregation(**kw)
        assert repr(ours) == repr(ref)
        assert [(n, tuple(v.shape)) for n, v in ours.named_parameters()] == \
            [(n, tuple(v.shape)) for n, v in ref.named_parameters()]
        assert (ours.min_value, ours.max_value) == (ref.min_value, ref.max_value)
        if kw.get("learn"):
            ours.p.data.zero_()
            ours.reset_parameters()
            assert torch.equal(ours.p.detach(), ref.p.detach())


def test_resolver():
    m = aggregation_resolver("powermean", p=2.0, learn=True)
    assert isinstance(m, PowerMeanAggregation) and m.learn and float(m.p) == 2.0


def test_gen_conv_is_a_plugin_layer(tg):
    from pytorch_geometric_b200.plugin import conv as PC
    assert PC.LAYERS["GENConv"] == "B200GENConv"
    assert issubclass(PC.B200GENConv, tg.nn.GENConv)


@pytest.mark.parametrize("kw", [dict(aggr="softmax", learn_t=True), dict(aggr="powermean", learn_p=True, edge_dim=4),
                                dict(aggr="softmax_sg", msg_norm=True), dict(aggr="mean")])
def test_subclass_falls_through_on_cpu(tg, kw):
    from pytorch_geometric_b200.plugin import conv as PC
    torch.manual_seed(0)
    ref = tg.nn.GENConv(8, 8, **kw)
    ours = PC.B200GENConv(8, 8, **kw)
    assert {k: tuple(v.shape) for k, v in ours.state_dict().items()} == \
        {k: tuple(v.shape) for k, v in ref.state_dict().items()}
    ours.load_state_dict(ref.state_dict())
    x = torch.randn(10, 8)
    ei = torch.randint(0, 10, (2, 40))
    ea = torch.randn(40, 4) if kw.get("edge_dim") else None
    assert torch.equal(ours(x, ei, ea), ref(x, ei, ea))
    seen = []
    ours.register_message_forward_hook(lambda m, i, o: seen.append(tuple(o.shape)))
    assert torch.equal(ours(x, ei, ea), ref(x, ei, ea))
    assert seen == [(40, 8)]


def _fake_cuda(t):
    """A stand-in reporting is_cuda and t's dtype (the predicate reads nothing else)."""
    class T:
        is_cuda = True
        dtype = t.dtype
    return T()


def test_power_mean_fusable_cases():
    f32, bf16 = _fake_cuda(torch.zeros(1)), _fake_cuda(torch.zeros(1, dtype=torch.bfloat16))
    f16, f64 = _fake_cuda(torch.zeros(1, dtype=torch.float16)), _fake_cuda(torch.zeros(1, dtype=torch.float64))
    assert power_mean_fusable(f32, 1.0, None, None)                       # a plain mean: no clamp needed
    assert power_mean_fusable(f32, 2.5, 1e-4, 100.0)
    assert power_mean_fusable(bf16, 2.5, 1e-4, None)
    assert power_mean_fusable(f32, torch.ones(4), 1e-4, 100.0)
    assert not power_mean_fusable(bf16, torch.ones(4), 1e-4, 100.0)       # fp32 p promotes bf16 messages
    assert power_mean_fusable(bf16, torch.ones(4, dtype=torch.bfloat16), 1e-4, 100.0)
    assert not power_mean_fusable(f16, 2.0, 1e-4, 100.0)
    assert not power_mean_fusable(f64, 2.0, 1e-4, 100.0)
    assert not power_mean_fusable(torch.zeros(1), 2.0, 1e-4, 100.0)       # CPU
    assert not power_mean_fusable(f32, 2.0, None, 100.0)                  # bases may be <= 0
    assert not power_mean_fusable(f32, 2.0, 0.0, 100.0)
    assert not power_mean_fusable(f32, 2.0, -1.0, 100.0)
    assert not power_mean_fusable(f32, 2.0, 1.0, 0.5)


def test_gen_fusable_cases(tg, monkeypatch):
    """Each branch of the predicate with `_fast` (device, hooks, explain) stubbed to pass."""
    from pytorch_geometric_b200.plugin import conv as PC
    monkeypatch.setattr(PC, "_fast", lambda self, *ts: True)
    f32, bf16 = _fake_cuda(torch.zeros(1)), _fake_cuda(torch.zeros(1, dtype=torch.bfloat16))
    for t in (f32, bf16):
        t.dim = lambda: 2
    ei = torch.randint(0, 10, (2, 40))
    ok = PC._gen_fusable
    assert ok(PC.B200GENConv(8, 8, aggr="softmax"), (f32, f32), ei, None)
    assert ok(PC.B200GENConv(8, 8, aggr="softmax_sg"), (f32, f32), ei, None)
    assert ok(PC.B200GENConv(8, 8, aggr="powermean", learn_p=True), (f32, f32), ei, None)
    assert ok(PC.B200GENConv(8, 8, aggr="softmax", learn_t=True), (f32, None), ei, None)
    for aggr in ("sum", "mean", "max", ["softmax", "mean"]):                  # not the sweep's aggregations
        assert not ok(PC.B200GENConv(8, 8, aggr=aggr), (f32, f32), ei, None)
    assert not ok(PC.B200GENConv(8, 8, aggr=["softmax", "mean"]), (f32, f32), ei, None)   # lin_aggr_out
    conv = PC.B200GENConv(8, 8, aggr="softmax", learn_t=True)
    assert not ok(conv, (f32, f32), ei.float(), None)                          # adjacency
    assert not ok(conv, (f32, f32), torch.randint(0, 10, (3, 40)), None)
    assert not ok(conv, (f32, f32), ei, torch.randn(40))                        # 1-D edge_attr
    assert not ok(conv, (f32, bf16), ei, None)                                 # mixed dtypes
    assert not ok(conv, (bf16, bf16), ei, None)                                # fp32 t with bf16 inputs promotes
    assert ok(PC.B200GENConv(8, 8, aggr="softmax", t=0.5), (bf16, bf16), ei, None)   # a Python-number t does not
    conv = PC.B200GENConv(8, 8, aggr="softmax", aggr_kwargs=dict(learn=True, channels=3))
    assert not ok(conv, (f32, f32), ei, None)                                  # t of neither 1 nor F channels
    conv = PC.B200GENConv(8, 8, aggr="powermean", aggr_kwargs=dict(p=2.0, clamp_min=None))
    assert not ok(conv, (f32, f32), ei, None)                                  # clamp bounds off the sweep


def test_mirror_constructor_errors_and_layout(tg, golden):
    from pytorch_geometric_b200.nn import GENConv
    for bad in (dict(aggr="mean"), dict(aggr="max"), dict(aggr=["softmax", "mean"])):
        with pytest.raises(ValueError, match="not on the fused path"):
            GENConv(8, 8, **bad)
    for norm in ("layer", "instance"):
        with pytest.raises(ValueError, match="norm"):
            GENConv(8, 8, norm=norm)
    z = golden("gen")
    cases = {"softmax_learn": (16, {"aggr": "softmax", "learn_t": True}),
             "softmax_sg": (16, {"aggr": "softmax_sg", "t": 0.5}),
             "pm_fixed": (16, {"aggr": "powermean", "p": 2.5}),
             "pm_learn_channels": (16, {"aggr": "powermean", "aggr_kwargs": {"p": 1.5, "learn": True, "channels": 16}}),
             "edge": (16, {"aggr": "softmax", "learn_t": True, "edge_dim": 4}),
             "bipartite": ((8, 12), {"aggr": "powermean", "learn_p": True, "norm": None}),
             "msg_norm": (16, {"aggr": "softmax", "msg_norm": True, "learn_msg_scale": True})}
    import json
    for tag, (ch, kw) in cases.items():
        conv = GENConv(ch, 16, **kw)
        assert repr(conv) == str(z[f"{tag}_repr"]), tag
        assert {n: list(p.shape) for n, p in conv.state_dict().items()} == json.loads(str(z[f"{tag}_shapes"])), tag
        ref = tg.nn.GENConv(ch, 16, **kw)
        assert [n for n, _ in conv.named_parameters()] == [n for n, _ in ref.named_parameters()], tag
    assert GENConv(8, 8, aggr="power").aggr == "powermean"
