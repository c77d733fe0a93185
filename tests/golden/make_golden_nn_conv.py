"""Golden vectors for NNConv (nn_conv.py:13-126): the UNMODIFIED reference's layer on the CPU, forward and backward, for
six cases -- the QM9-style edge network Sequential(Linear(5, 16), ReLU, Linear(16, F_in F_out)) with aggr='add' and
with aggr='mean'; the bipartite NNConv((8, 16), 32) of the reference's own test; a bare Linear(3, F_in F_out) edge
network; root_weight=False, bias=False; and a graph whose destinations 0..2 have no in-edges -- plus the `state_dict`
shapes and the repr of each.  Same provenance rules as make_golden.py (needs the reference in oracle/_ref; writes
tests/golden/nn_conv.npz).

    python tests/golden/make_golden_nn_conv.py
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", "oracle", "_ref"))  # oracle/install_ref.sh
import torch_geometric.typing as tgt  # noqa: E402
from torch.nn import Linear, ReLU, Sequential  # noqa: E402
from torch_geometric.nn import NNConv  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
assert not (tgt.WITH_TORCH_SCATTER or tgt.WITH_TORCH_SPARSE or tgt.WITH_PYG_LIB)

# (tag, in_channels, out_channels, edge dim D, hidden K (None: bare Linear), constructor kwargs, isolated destinations)
CASES = [("qm9_add", 8, 8, 5, 16, {}, False),
         ("qm9_mean", 8, 8, 5, 16, {"aggr": "mean"}, False),
         ("bipartite", (8, 16), 32, 3, 8, {}, False),
         ("bare_linear", 6, 4, 3, None, {}, False),
         ("no_root_no_bias", 4, 8, 2, 6, {"root_weight": False, "bias": False}, False),
         ("isolated", 8, 8, 5, 16, {"aggr": "mean"}, True)]


def edge_net(d, k, f_in, f_out):
    if k is None:
        return Linear(d, f_in * f_out)
    return Sequential(Linear(d, k), ReLU(), Linear(k, f_in * f_out))


def main():
    g = torch.Generator().manual_seed(4242)
    N_src, N_dst, E = 12, 9, 60
    arrs = {}
    for n, (tag, ch, f_out, d, k, kw, isolated) in enumerate(CASES):
        bip = not isinstance(ch, int)
        f_src, f_dst = (ch, ch) if not bip else ch
        n_dst = N_dst if bip else N_src
        lo = 3 if isolated else 0
        ei = torch.stack([torch.randint(0, N_src, (E, ), generator=g), torch.randint(lo, n_dst, (E, ), generator=g)])
        x = torch.randn(N_src, f_src, generator=g)
        x_dst = torch.randn(n_dst, f_dst, generator=g) if bip else None
        ea = torch.randn(E, d, generator=g)
        torch.manual_seed(70 + n)
        conv = NNConv(ch, f_out, edge_net(d, k, f_src, f_out), **kw)
        if conv.bias is not None:
            with torch.no_grad():
                conv.bias.normal_()                             # the reference initialises it to 0
        for name, p in conv.state_dict().items():
            arrs[f"{tag}_p_{name}"] = p.clone()
        xr = x.clone().requires_grad_()
        xdr = x_dst.clone().requires_grad_() if bip else None
        ear = ea.clone().requires_grad_()
        out = conv((xr, xdr) if bip else xr, ei, ear)
        gout = torch.randn(out.shape, generator=g)
        out.backward(gout)
        arrs.update({f"{tag}_ei": ei, f"{tag}_x": x, f"{tag}_ea": ea, f"{tag}_out": out, f"{tag}_gout": gout,
                     f"{tag}_gx": xr.grad, f"{tag}_gea": ear.grad})
        if bip:
            arrs.update({f"{tag}_x_dst": x_dst, f"{tag}_gx_dst": xdr.grad})
        for name, p in conv.named_parameters():
            arrs[f"{tag}_g_{name}"] = p.grad
        arrs[f"{tag}_shapes"] = np.asarray(json.dumps({nm: list(p.shape) for nm, p in conv.state_dict().items()}))
        arrs[f"{tag}_repr"] = np.asarray(repr(conv))
    np_arrs = {k: (v.detach().numpy() if isinstance(v, torch.Tensor) else v) for k, v in arrs.items()}
    np.savez_compressed(os.path.join(OUT, "nn_conv.npz"), **np_arrs)
    print("wrote nn_conv", len(np_arrs), "arrays")


if __name__ == "__main__":
    main()
