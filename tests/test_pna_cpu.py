"""CPU checks of the PNA layers: the standalone `nn.PNAConv` mirror's layout, repr, errors and degree histogram against
the reference, `plugin.conv.B200PNAConv` falling through bit for bit on CPU tensors, and the fusability predicate."""
import copy

import pytest
import torch

from pytorch_geometric_b200.nn import PNAConv

AGGRS = ["mean", "min", "max", "std"]
SCALERS = ["identity", "amplification", "attenuation"]
DEG = torch.tensor([0, 3, 5, 2])


@pytest.mark.parametrize("kw", [dict(edge_dim=3, towers=4), dict(towers=2, divide_input=True, post_layers=2),
                                dict(train_norm=True)])
def test_mirror_state_dict_and_repr_match_the_reference(tg, kw):
    ref = tg.nn.PNAConv(16, 32, AGGRS, SCALERS, DEG, **kw)
    mine = PNAConv(16, 32, AGGRS, SCALERS, DEG, **kw)
    assert {k: v.shape for k, v in mine.state_dict().items()} == {k: v.shape for k, v in ref.state_dict().items()}
    assert repr(mine) == repr(ref)
    assert torch.equal(mine.aggr_module.avg_deg_lin, ref.aggr_module.avg_deg_lin)
    assert torch.equal(mine.aggr_module.avg_deg_log, ref.aggr_module.avg_deg_log)
    mine.load_state_dict(ref.state_dict())


def test_mirror_rejects_what_it_does_not_fuse():
    with pytest.raises(ValueError, match="pre_layers"):
        PNAConv(16, 32, AGGRS, SCALERS, DEG, pre_layers=2)
    with pytest.raises(ValueError, match="aggregator"):
        PNAConv(16, 32, ["softmax"], SCALERS, DEG)
    with pytest.raises(ValueError, match="scaler"):
        PNAConv(16, 32, AGGRS, ["cubic"], DEG)


def test_degree_histogram_matches_the_reference(tg):
    g = torch.Generator().manual_seed(0)
    graphs = []
    for n in (5, 9, 13):
        ei = torch.randint(0, n, (2, 3 * n), generator=g)
        graphs.append(tg.data.Data(edge_index=ei, num_nodes=n))
    assert torch.equal(PNAConv.get_degree_histogram(graphs), tg.nn.PNAConv.get_degree_histogram(graphs))


def test_b200_pna_on_cpu_is_the_reference(tg):
    from pytorch_geometric_b200.plugin import conv as PC
    torch.manual_seed(0)
    ref = tg.nn.PNAConv(16, 32, AGGRS, SCALERS, DEG, edge_dim=3, towers=4)
    mine = copy.deepcopy(ref)
    mine.__class__ = PC.B200PNAConv
    x = torch.randn(10, 16)
    ei = torch.randint(0, 10, (2, 30))
    ea = torch.randn(30, 3)
    assert torch.equal(mine(x, ei, ea), ref(x, ei, ea))
    assert "PNAConv" in PC.LAYERS


def test_fusability_predicate(tg, monkeypatch):
    from pytorch_geometric_b200.plugin import conv as PC
    from pytorch_geometric_b200.plugin import routing
    monkeypatch.setattr(routing, "engine_ok", lambda t: True)       # stand in for a CUDA tensor
    x, ei, ea = torch.randn(10, 16), torch.randint(0, 10, (2, 30)), torch.randn(30, 3)

    def layer(**kw):
        m = tg.nn.PNAConv(16, 32, kw.pop("aggregators", AGGRS), kw.pop("scalers", SCALERS), DEG,
                          **{"edge_dim": 3, "towers": 4, **kw})
        m.__class__ = PC.B200PNAConv
        return m
    assert PC._pna_fusable(layer(), x, ei, ea)
    assert PC._pna_fusable(layer(flow="target_to_source"), x, ei, ea)
    assert not PC._pna_fusable(layer(pre_layers=2), x, ei, ea)
    assert not PC._pna_fusable(layer(aggregators=["mean", "softmax"]), x, ei, ea)
    assert not PC._pna_fusable(layer(aggregators=["mean", "mean"]), x, ei, ea)
    assert not PC._pna_fusable(layer(), x, ei, None)                  # edge_dim without edge_attr
    assert not PC._pna_fusable(layer(), x, ei.float(), ea)
    m = layer()
    m.register_message_forward_hook(lambda mod, inp, out: out)
    assert not PC._pna_fusable(m, x, ei, ea)
    m = layer()
    m.explain = True
    assert not PC._pna_fusable(m, x, ei, ea)
    m = layer()
    m.decomposed_layers = 2
    assert not PC._pna_fusable(m, x, ei, ea)
    monkeypatch.setattr(routing, "_compiling", lambda: True)
    assert not PC._pna_fusable(layer(), x, ei, ea)
    monkeypatch.setattr(routing, "_compiling", lambda: False)
    m = layer()
    assert PC._pna_fusable(m, x, ei, ea)
    monkeypatch.setattr(torch.jit, "is_scripting", lambda: True)
    assert not PC._pna_fusable(m, x, ei, ea)


def test_fusability_predicate_needs_cuda_float32_or_bfloat16(tg):
    from pytorch_geometric_b200.plugin import conv as PC
    m = tg.nn.PNAConv(16, 32, AGGRS, SCALERS, DEG, edge_dim=3, towers=4)
    m.__class__ = PC.B200PNAConv
    ei, ea = torch.randint(0, 10, (2, 30)), torch.randn(30, 3)
    assert not PC._pna_fusable(m, torch.randn(10, 16), ei, ea)                       # CPU
    assert not PC._pna_fusable(m, torch.randn(10, 16, dtype=torch.float16), ei, ea.half())
    assert not PC._pna_fusable(m, torch.randn(10, 16, dtype=torch.float64), ei, ea.double())


GOLDEN_CASES = [("all", 16, 32, dict(aggregators=["mean", "min", "max", "std", "sum", "var"],
                                     scalers=["identity", "amplification", "attenuation", "linear", "inverse_linear"],
                                     towers=4, edge_dim=3)),
                ("divide", 16, 32, dict(aggregators=["sum", "max", "var"], scalers=["identity", "linear"], towers=2,
                                        divide_input=True, post_layers=2)),
                ("train_norm", 12, 8, dict(aggregators=AGGRS, scalers=SCALERS, edge_dim=5, train_norm=True))]


@pytest.mark.parametrize("tag,ic,oc,kw", GOLDEN_CASES)
def test_mirror_layout_matches_golden(golden, tag, ic, oc, kw):
    import json
    z = golden("pna")
    mine = PNAConv(ic, oc, deg=torch.from_numpy(z[f"{tag}_deg"]), **kw)
    assert {n: list(p.shape) for n, p in mine.state_dict().items()} == json.loads(str(z[f"{tag}_shapes"]))
    assert repr(mine) == str(z[f"{tag}_repr"])
    mine.load_state_dict({k[len(tag) + 3:]: torch.from_numpy(v) for k, v in z.items() if k.startswith(f"{tag}_p_")})
