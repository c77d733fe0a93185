"""CPU checks of the NNConv layers: the standalone `nn.NNConv` mirror's checkpoint layout, repr and constructor errors
against the golden data of the reference, `plugin.conv.B200NNConv` falling through bit for bit on CPU tensors (hooks
included), the fusability predicate, and the W' layout identity out_i = vec(P_i) W' in fp64 against the reference's
`message()` followed by sum and by mean."""
import copy
import json

import pytest
import torch
from torch.nn import Linear, ReLU, Sequential

from pytorch_geometric_b200.nn import NNConv
from pytorch_geometric_b200.nn.conv import nn_conv_split, nn_conv_weight

GOLDEN = [("qm9_add", 8, 8, 5, 16, {}), ("qm9_mean", 8, 8, 5, 16, {"aggr": "mean"}), ("bipartite", (8, 16), 32, 3, 8, {}),
          ("bare_linear", 6, 4, 3, None, {}), ("no_root_no_bias", 4, 8, 2, 6, {"root_weight": False, "bias": False}),
          ("isolated", 8, 8, 5, 16, {"aggr": "mean"})]


def _net(d, k, f_in, f_out):
    return Linear(d, f_in * f_out) if k is None else Sequential(Linear(d, k), ReLU(), Linear(k, f_in * f_out))


@pytest.mark.parametrize("tag,ch,f_out,d,k,kw", GOLDEN)
def test_mirror_layout_and_repr_match_golden(golden, tag, ch, f_out, d, k, kw):
    z = golden("nn_conv")
    f_src = ch if isinstance(ch, int) else ch[0]
    mine = NNConv(ch, f_out, _net(d, k, f_src, f_out), **kw)
    assert {n: list(p.shape) for n, p in mine.state_dict().items()} == json.loads(str(z[f"{tag}_shapes"]))
    assert list(mine.state_dict()) == list(json.loads(str(z[f"{tag}_shapes"])))
    assert repr(mine) == str(z[f"{tag}_repr"])
    mine.load_state_dict({key[len(tag) + 3:]: torch.from_numpy(v) for key, v in z.items() if key.startswith(f"{tag}_p_")})


@pytest.mark.parametrize("aggr", ["max", "min", ["sum", "mean"]])
def test_mirror_rejects_aggregations_it_does_not_fuse(aggr):
    with pytest.raises(ValueError, match="aggr"):
        NNConv(4, 4, Linear(3, 16), aggr=aggr)


@pytest.mark.parametrize("net", [Sequential(Linear(3, 16), ReLU()), Linear(3, 15), Sequential(),
                                 torch.nn.LazyLinear(16), Sequential(Linear(3, 8), ReLU(), torch.nn.LazyLinear(16)),
                                 torch.nn.Bilinear(3, 3, 16)])
def test_mirror_rejects_edge_networks_it_cannot_split(net):
    with pytest.raises(ValueError, match="edge network"):
        NNConv(4, 4, net)


def test_split_accepts_linear_sequential_and_the_reference_linear(tg):
    assert nn_conv_split(Linear(3, 16), 4, 4)[0] == []
    pre, last = nn_conv_split(Sequential(Linear(3, 8), ReLU(), Linear(8, 16)), 4, 4)
    assert len(pre) == 2 and last.out_features == 16
    assert nn_conv_split(tg.nn.Linear(3, 16), 4, 4) is not None
    assert nn_conv_split(tg.nn.Linear(-1, 16), 4, 4) is None              # lazy: not initialised yet
    hooked = Linear(3, 16)
    hooked.register_forward_hook(lambda m, i, o: o)
    assert nn_conv_split(hooked, 4, 4) is None


@pytest.mark.parametrize("where", ["net", "last"])
@pytest.mark.parametrize("hook", ["forward", "forward_pre", "forward_kwargs", "full_backward", "full_backward_pre"])
def test_split_refuses_hooks_the_fused_path_would_skip(where, hook):
    net = Sequential(Linear(3, 8), ReLU(), Linear(8, 16))
    m = net if where == "net" else net[2]
    {"forward": lambda: m.register_forward_hook(lambda mod, i, o: o),
     "forward_pre": lambda: m.register_forward_pre_hook(lambda mod, i: i),
     "forward_kwargs": lambda: m.register_forward_hook(lambda mod, a, k, o: o, with_kwargs=True),
     "full_backward": lambda: m.register_full_backward_hook(lambda mod, gi, go: gi),
     "full_backward_pre": lambda: m.register_full_backward_pre_hook(lambda mod, go: go)}[hook]()
    assert nn_conv_split(net, 4, 4) is None
    assert nn_conv_split(Sequential(Linear(3, 8), ReLU(), Linear(8, 16)), 4, 4) is not None


@pytest.mark.parametrize("kind", ["forward", "forward_pre", "backward"])
def test_split_refuses_global_module_hooks(kind):
    from torch.nn.modules import module as M
    register = {"forward": M.register_module_forward_hook, "forward_pre": M.register_module_forward_pre_hook,
                "backward": M.register_module_full_backward_hook}[kind]
    handle = register(lambda *a: None)
    try:
        assert nn_conv_split(Linear(3, 16), 4, 4) is None
    finally:
        handle.remove()
    assert nn_conv_split(Linear(3, 16), 4, 4) is not None


def test_mirror_refuses_an_edge_network_hooked_after_construction():
    conv = NNConv(4, 4, Sequential(Linear(3, 8), ReLU(), Linear(8, 16)))
    conv.nn[2].register_forward_hook(lambda m, i, o: o)
    with pytest.raises(ValueError, match="can no longer be split"):
        conv(torch.randn(5, 4), torch.randint(0, 5, (2, 7)), torch.randn(7, 3))


def test_mirror_refuses_autocast():
    conv = NNConv(4, 4, Linear(3, 16))
    with torch.autocast("cpu", dtype=torch.bfloat16), pytest.raises(ValueError, match="autocast"):
        conv(torch.randn(5, 4), torch.randint(0, 5, (2, 7)), torch.randn(7, 3))


@pytest.mark.parametrize("aggr", ["add", "mean"])
def test_w_prime_layout_reproduces_the_reference_message(tg, aggr):
    """out_i = vec(P_i) W' with P_i = REDUCE_e [h_e, 1] (x) x_j, in fp64, against the reference's message() and
    scatter: the identity the sweep and the GEMM implement."""
    torch.manual_seed(3)
    f_in, f_out, d, k, n, e = 5, 7, 4, 6, 9, 40
    conv = tg.nn.NNConv(f_in, f_out, Sequential(Linear(d, k), ReLU(), Linear(k, f_in * f_out)), aggr=aggr,
                        root_weight=False, bias=False).double()
    x = torch.randn(n, f_in, dtype=torch.float64)
    ea = torch.randn(e, d, dtype=torch.float64)
    ei = torch.stack([torch.randint(0, n, (e, )), torch.randint(1, n, (e, ))])      # node 0 has no in-edges
    want = conv(x, ei, ea)
    pre, last = nn_conv_split(conv.nn, f_in, f_out)
    h = ea
    for m in pre:
        h = m(h)
    ht = torch.cat([h, torch.ones(e, 1, dtype=h.dtype)], 1)
    outer = (ht[:, :, None] * x[ei[0]][:, None, :]).reshape(e, -1)                 # [E, (K+1) F_in]
    p = torch.zeros(n, outer.size(1), dtype=torch.float64).index_add_(0, ei[1], outer)
    if aggr == "mean":
        p = p / torch.bincount(ei[1], minlength=n).clamp(min=1).to(p.dtype)[:, None]
    got = p @ nn_conv_weight(last.weight, last.bias, f_in, f_out)
    assert (got - want).abs().max().item() <= 1e-12 * max(1.0, want.abs().max().item())


def _b200(ref):
    from pytorch_geometric_b200.plugin import conv as PC
    mine = copy.deepcopy(ref)
    mine.__class__ = PC.B200NNConv
    return mine


@pytest.mark.parametrize("tag,ch,f_out,d,k,kw", GOLDEN)
def test_b200_nn_conv_on_cpu_is_the_reference(tg, tag, ch, f_out, d, k, kw):
    torch.manual_seed(0)
    f_src, f_dst = (ch, ch) if isinstance(ch, int) else ch
    ref = tg.nn.NNConv(ch, f_out, _net(d, k, f_src, f_out), **kw)
    mine = _b200(ref)
    bip = not isinstance(ch, int)
    x = torch.randn(10, f_src)
    x_in = (x, torch.randn(7, f_dst)) if bip else x
    ei = torch.stack([torch.randint(0, 10, (30, )), torch.randint(0, 7 if bip else 10, (30, ))])
    ea = torch.randn(30, d)
    assert torch.equal(mine(x_in, ei, ea), ref(x_in, ei, ea))
    assert list(mine.state_dict()) == list(ref.state_dict())
    assert repr(mine).replace("B200NNConv", "NNConv") == repr(ref)


def test_registered_hook_fires(tg):
    mine = _b200(tg.nn.NNConv(4, 4, Linear(2, 16)))
    seen = []
    mine.register_message_forward_hook(lambda mod, inp, out: seen.append(out.shape))
    mine(torch.randn(5, 4), torch.randint(0, 5, (2, 11)), torch.randn(11, 2))
    assert seen == [torch.Size([11, 4])]


def test_layer_and_alias_are_registered():
    from pytorch_geometric_b200.plugin import conv as PC
    assert PC.LAYERS["NNConv"] == "B200NNConv" and PC.LAYERS["ECConv"] == "B200NNConv"


def test_fusability_predicate(tg, monkeypatch):
    from pytorch_geometric_b200.plugin import conv as PC
    from pytorch_geometric_b200.plugin import routing
    monkeypatch.setattr(routing, "engine_ok", lambda t: True)       # stand in for a CUDA tensor
    x, ea = torch.randn(10, 8), torch.randn(30, 3)
    ei = torch.randint(0, 10, (2, 30))
    xs = (x, x)

    def layer(net=None, **kw):
        return _b200(tg.nn.NNConv(8, 4, net if net is not None else Sequential(Linear(3, 6), ReLU(), Linear(6, 32)), **kw))
    assert PC._nn_conv_split(layer(), xs, ei, ea) is not None
    assert PC._nn_conv_split(layer(aggr="mean"), xs, ei, ea) is not None
    assert PC._nn_conv_split(layer(Linear(3, 32)), xs, ei, ea) is not None
    assert PC._nn_conv_split(layer(tg.nn.Linear(3, 32)), xs, ei, ea) is not None
    assert PC._nn_conv_split(layer(root_weight=False, bias=False), (x, None), ei, ea) is not None
    assert PC._nn_conv_split(layer(aggr="max"), xs, ei, ea) is None
    assert PC._nn_conv_split(layer(Sequential(Linear(3, 32), ReLU())), xs, ei, ea) is None
    assert PC._nn_conv_split(layer(), xs, ei, None) is None
    assert PC._nn_conv_split(layer(), xs, ei, ea.view(30, 3, 1)) is None
    assert PC._nn_conv_split(layer(), xs, torch.sparse_coo_tensor(ei, torch.ones(30), (10, 10)), ea) is None
    assert PC._nn_conv_split(layer(), xs, ei, ea.double()) is None                     # mixed dtypes
    m = layer()
    m.register_message_forward_hook(lambda mod, inp, out: out)
    assert PC._nn_conv_split(m, xs, ei, ea) is None
    m = layer()
    m.explain = True
    assert PC._nn_conv_split(m, xs, ei, ea) is None
    m = layer()
    m.decomposed_layers = 2
    assert PC._nn_conv_split(m, xs, ei, ea) is None
    monkeypatch.setattr(routing, "_compiling", lambda: True)
    assert PC._nn_conv_split(layer(), xs, ei, ea) is None
    monkeypatch.setattr(routing, "_compiling", lambda: False)
    with torch.autocast("cpu", dtype=torch.bfloat16):              # the edge network would run in bf16, x in fp32
        assert PC._nn_conv_split(layer(), xs, ei, ea) is None
    assert PC._nn_conv_split(layer(), xs, ei, ea) is not None
    m = layer()
    m.nn[2].register_full_backward_hook(lambda mod, gi, go: gi)
    assert PC._nn_conv_split(m, xs, ei, ea) is None
    big = layer(Linear(3, 8 * 4))
    assert PC._nn_conv_split(big, xs, ei, ea) is not None
    monkeypatch.setattr(PC.ops, "nn_conv_supported", lambda k, f, dt: False)
    assert PC._nn_conv_split(big, xs, ei, ea) is None


def test_supported_range():
    from pytorch_geometric_b200 import ops
    assert ops.nn_conv_supported(128, 64, torch.float32) and ops.nn_conv_supported(25, 1, torch.bfloat16)
    assert ops.nn_conv_supported(16383, 1, torch.float32) and not ops.nn_conv_supported(16384, 1, torch.float32)
    assert ops.nn_conv_supported(255, 64, torch.float32) and not ops.nn_conv_supported(256, 64, torch.float32)
    assert not ops.nn_conv_supported(8, 8, torch.float16) and not ops.nn_conv_supported(8, 0, torch.float32)
