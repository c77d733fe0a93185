"""Golden vectors for GINEConv (gin_conv.py:104-207): the UNMODIFIED reference's layer on the CPU, forward and backward,
for three cases -- no `edge_dim`; `edge_dim=5` with `train_eps=True`; `aggr='mean'` on a bipartite input -- plus the
`state_dict` shapes of each.  Same provenance rules as make_golden.py (needs the reference in oracle/_ref; writes
tests/golden/gine.npz).

    python tests/golden/make_golden_gine.py
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", "oracle", "_ref"))  # oracle/install_ref.sh
import torch_geometric.typing as tgt  # noqa: E402
from torch_geometric.nn import GINEConv  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
assert not (tgt.WITH_TORCH_SCATTER or tgt.WITH_TORCH_SPARSE or tgt.WITH_PYG_LIB)

F_IN, F_HID, F_OUT, EDGE_DIM = 8, 16, 8, 5
# (tag, constructor kwargs, bipartite, edge feature width)
CASES = [("plain", {}, False, F_IN),
         ("edge_dim", {"edge_dim": EDGE_DIM, "train_eps": True, "eps": 0.25}, False, EDGE_DIM),
         ("mean_bip", {"aggr": "mean", "eps": -0.5}, True, F_IN)]


def mlp():
    return torch.nn.Sequential(torch.nn.Linear(F_IN, F_HID), torch.nn.ReLU(), torch.nn.Linear(F_HID, F_OUT))


def main():
    g = torch.Generator().manual_seed(4242)
    N_src, N_dst, E = 13, 9, 70
    arrs = {}
    for k, (tag, kw, bip, fe) in enumerate(CASES):
        n_dst = N_dst if bip else N_src
        ei = torch.stack([torch.randint(0, N_src, (E, ), generator=g), torch.randint(0, n_dst - 1, (E, ), generator=g)])
        ei[:, 1] = ei[:, 0]                                    # a duplicated edge; destination n_dst-1 has no in-edge
        x = torch.randn(N_src, F_IN, generator=g)
        x_dst = torch.randn(n_dst, F_IN, generator=g) if bip else None
        ea = torch.randn(E, fe, generator=g)
        torch.manual_seed(11 + k)
        conv = GINEConv(mlp(), **kw)
        xr, ear = x.clone().requires_grad_(), ea.clone().requires_grad_()
        xdr = x_dst.clone().requires_grad_() if bip else None
        out = conv((xr, xdr) if bip else xr, ei, ear)
        gout = torch.randn(out.shape, generator=g)
        out.backward(gout)
        arrs.update({f"{tag}_ei": ei, f"{tag}_x": x, f"{tag}_ea": ea, f"{tag}_out": out, f"{tag}_gout": gout,
                     f"{tag}_gx": xr.grad, f"{tag}_gea": ear.grad})
        if bip:
            arrs.update({f"{tag}_x_dst": x_dst, f"{tag}_gx_dst": xdr.grad})
        for name, p in conv.state_dict().items():
            arrs[f"{tag}_p_{name}"] = p
        for name, p in conv.named_parameters():
            arrs[f"{tag}_g_{name}"] = p.grad
        arrs[f"{tag}_shapes"] = np.asarray(json.dumps({n: list(p.shape) for n, p in conv.state_dict().items()}))
    np_arrs = {k: (v.detach().numpy() if isinstance(v, torch.Tensor) else v) for k, v in arrs.items()}
    np.savez_compressed(os.path.join(OUT, "gine.npz"), **np_arrs)
    print("wrote gine", len(np_arrs), "arrays")


if __name__ == "__main__":
    main()
