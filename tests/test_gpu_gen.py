"""GPU tests of GENConv: the standalone `nn.GENConv` against the reference's golden vectors (tests/golden/gen.npz), and
the plug-in `B200GENConv` on bf16 inputs, with a bipartite layer's gradients, with a learnable fp32 t / p and bf16
inputs (the reference promotes: the subclass falls through), and with hooks on CUDA (falls through)."""
import json

import numpy as np
import pytest
import torch

pytestmark = pytest.mark.gpu

from pytorch_geometric_b200 import ops  # noqa: E402
from pytorch_geometric_b200.nn import GENConv  # noqa: E402

DEV = "cuda"
GOLDEN_CASES = [("softmax_learn", 16, {"aggr": "softmax", "learn_t": True}, None, False),
                ("softmax_sg", 16, {"aggr": "softmax_sg", "t": 0.5}, None, False),
                ("pm_fixed", 16, {"aggr": "powermean", "p": 2.5}, None, False),
                ("pm_learn_channels", 16, {"aggr": "powermean",
                                           "aggr_kwargs": {"p": 1.5, "learn": True, "channels": 16}}, None, False),
                ("edge", 16, {"aggr": "softmax", "learn_t": True, "edge_dim": 4}, 4, False),
                ("bipartite", (8, 12), {"aggr": "powermean", "learn_p": True, "norm": None}, None, True),
                ("msg_norm", 16, {"aggr": "softmax", "msg_norm": True, "learn_msg_scale": True}, None, False)]
FUSED = ("softmax_aggr_csr", "power_mean_csr")


def _calls():
    return {k: v["calls"] for k, v in ops.PROFILE.summary().items()}


@pytest.mark.parametrize("tag,ch,kw,edim,bip", GOLDEN_CASES, ids=[c[0] for c in GOLDEN_CASES])
def test_standalone_gen_matches_golden(golden, tag, ch, kw, edim, bip):
    z = golden("gen")
    conv = GENConv(ch, 16, **kw).to(DEV)
    assert repr(conv) == str(z[f"{tag}_repr"])
    shapes = {n: list(p.shape) for n, p in conv.state_dict().items()}
    assert shapes == json.loads(str(z[f"{tag}_shapes"]))
    conv.load_state_dict({n: torch.from_numpy(np.asarray(z[f"{tag}_p_{n}"])) for n in shapes})
    conv.train()
    x = torch.from_numpy(z[f"{tag}_x"]).to(DEV).requires_grad_()
    xd = torch.from_numpy(z[f"{tag}_x_dst"]).to(DEV).requires_grad_() if bip else None
    ea = torch.from_numpy(z[f"{tag}_ea"]).to(DEV).requires_grad_() if edim else None
    ei = torch.from_numpy(z[f"{tag}_ei"]).to(DEV)
    ops.PROFILE.reset(enabled=True)
    out = conv((x, xd) if bip else x, ei, ea)
    calls = _calls()
    ops.PROFILE.reset(enabled=False)
    assert sum(calls.get(k, 0) for k in FUSED) == 1, calls
    torch.testing.assert_close(out.cpu(), torch.from_numpy(z[f"{tag}_out"]), rtol=1e-4, atol=1e-5)
    out.backward(torch.from_numpy(z[f"{tag}_gout"]).to(DEV))
    torch.testing.assert_close(x.grad.cpu(), torch.from_numpy(z[f"{tag}_gx"]), rtol=1e-4, atol=1e-5)
    if bip:
        torch.testing.assert_close(xd.grad.cpu(), torch.from_numpy(z[f"{tag}_gx_dst"]), rtol=1e-4, atol=1e-5)
    if edim:
        torch.testing.assert_close(ea.grad.cpu(), torch.from_numpy(z[f"{tag}_gea"]), rtol=1e-4, atol=1e-5)
    for n, p in conv.named_parameters():
        if f"{tag}_g_{n}" in z:
            torch.testing.assert_close(p.grad.cpu(), torch.from_numpy(z[f"{tag}_g_{n}"]), rtol=1e-4, atol=1e-5, msg=n)


def _pair(tg, kw, dtype=torch.float32):
    from pytorch_geometric_b200.plugin import conv as PC
    torch.manual_seed(0)
    ref = tg.nn.GENConv(**kw)
    ours = PC.B200GENConv(**kw)
    ours.load_state_dict(ref.state_dict())
    return ref.to(DEV, dtype), ours.to(DEV, dtype)


@pytest.mark.parametrize("aggr,extra", [("softmax", dict(learn_t=True)), ("powermean", dict(p=2.0))])
def test_plugin_bf16_against_reference(tg, aggr, extra):
    """bf16 inputs and parameters of one dtype take the fused sweep.  Both bf16 results are compared with the reference
    run in fp32 on the same (bf16-valued) inputs and parameters: the fused layer's error may be at most twice the
    reference's own bf16 error, plus 1e-2 of the largest entry."""
    kw = dict(in_channels=16, out_channels=16, aggr=aggr, norm=None, **extra)
    ref, ours = _pair(tg, kw, torch.bfloat16)
    ref32 = _pair(tg, kw)[0]
    ref32.load_state_dict({k: v.float() for k, v in ref.state_dict().items()})
    gen = torch.Generator().manual_seed(3)
    x = torch.randn(50, 16, generator=gen).to(DEV, torch.bfloat16)
    ea = torch.randn(400, 16, generator=gen).to(DEV, torch.bfloat16)
    ei = torch.randint(0, 50, (2, 400), generator=gen).to(DEV)
    xr, xo, er, eo = (t.clone().requires_grad_() for t in (x, x, ea, ea))
    x3, e3 = x.float().requires_grad_(), ea.float().requires_grad_()
    ops.PROFILE.reset(enabled=True)
    got = ours(xo, ei, eo)
    calls = _calls()
    ops.PROFILE.reset(enabled=False)
    assert sum(calls.get(k, 0) for k in FUSED) == 1, calls
    want = ref(xr, ei, er)
    exact = ref32(x3, ei, e3)
    assert got.dtype == want.dtype == torch.bfloat16
    g = torch.randn_like(want)
    for o, gg in ((want, g), (got, g), (exact, g.float())):
        o.backward(gg)
    for u, v, w, what in ((got, want, exact, "out"), (xo.grad, xr.grad, x3.grad, "grad_x"),
                          (eo.grad, er.grad, e3.grad, "grad_edge_attr")):
        u, v, w = u.detach().float(), v.detach().float(), w.detach().float()
        assert (u - w).abs().max() <= 2 * (v - w).abs().max() + 1e-2 * w.abs().max(), what


def test_plugin_bipartite_gradients(tg):
    kw = dict(in_channels=(8, 12), out_channels=16, aggr="powermean", learn_p=True)
    ref, ours = _pair(tg, kw)
    gen = torch.Generator().manual_seed(7)
    xs = torch.randn(30, 8, generator=gen).to(DEV)
    xd = torch.randn(20, 12, generator=gen).to(DEV)
    ei = torch.stack([torch.randint(0, 30, (200, ), generator=gen), torch.randint(0, 20, (200, ), generator=gen)]).to(DEV)
    a = [t.clone().requires_grad_() for t in (xs, xd)]
    b = [t.clone().requires_grad_() for t in (xs, xd)]
    got, want = ours(tuple(a), ei), ref(tuple(b), ei)
    torch.testing.assert_close(got, want, rtol=1e-4, atol=1e-5)
    g = torch.randn_like(want)
    got.backward(g)
    want.backward(g)
    for u, v in zip(a, b):
        torch.testing.assert_close(u.grad, v.grad, rtol=1e-4, atol=1e-5)
    for (n, pr), (_, po) in zip(ref.named_parameters(), ours.named_parameters()):
        torch.testing.assert_close(po.grad, pr.grad, rtol=1e-4, atol=1e-5, msg=n)


@pytest.mark.parametrize("aggr,extra", [("softmax", dict(learn_t=True)), ("powermean", dict(learn_p=True))])
def test_plugin_fp32_parameter_with_bf16_inputs_falls_through(tg, aggr, extra):
    """A learnable fp32 t / p with bf16 features promotes in the reference; the subclass runs the reference's forward."""
    kw = dict(in_channels=16, out_channels=16, aggr=aggr, norm=None, **extra)
    ref, ours = _pair(tg, kw)
    x = torch.randn(40, 16, device=DEV).to(torch.bfloat16)
    ei = torch.randint(0, 40, (2, 300), device=DEV)
    ops.PROFILE.reset(enabled=True)
    got = ours(x, ei)
    calls = _calls()
    ops.PROFILE.reset(enabled=False)
    assert not any(k in calls for k in FUSED), calls
    want = ref(x, ei)
    assert got.dtype == want.dtype == torch.float32
    torch.testing.assert_close(got.float(), want.float(), rtol=1e-5, atol=1e-6)


def test_plugin_hooks_fall_through_on_cuda(tg):
    kw = dict(in_channels=16, out_channels=16, aggr="softmax", learn_t=True)
    ref, ours = _pair(tg, kw)
    seen = []
    ours.register_message_forward_hook(lambda m, i, o: seen.append(tuple(o.shape)))
    x = torch.randn(40, 16, device=DEV)
    ei = torch.randint(0, 40, (2, 300), device=DEV)
    ops.PROFILE.reset(enabled=True)
    got = ours(x, ei)
    calls = _calls()
    ops.PROFILE.reset(enabled=False)
    assert seen == [(300, 16)]
    assert not any(k in calls for k in FUSED), calls
    torch.testing.assert_close(got, ref(x, ei), rtol=1e-5, atol=1e-6)
