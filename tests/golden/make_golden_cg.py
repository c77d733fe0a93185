"""Golden vectors for CGConv (cg_conv.py:12-101): the UNMODIFIED reference's layer on the CPU, forward and backward,
for three cases -- `CGConv(16)` with dim = 0; a bipartite `CGConv((8, 16), dim=5, aggr='mean', batch_norm=True)` in
training mode; `CGConv(6, dim=3, bias=False)` (rows of 24 bytes: the kernels' scalar path in fp32) -- plus the
`state_dict` shapes and the repr of each.  The graph has a duplicated edge and a destination without in-edges.  Same
provenance rules as make_golden.py (needs the reference in oracle/_ref; writes tests/golden/cg.npz).

    python tests/golden/make_golden_cg.py
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", "oracle", "_ref"))  # oracle/install_ref.sh
import torch_geometric.typing as tgt  # noqa: E402
from torch_geometric.nn import CGConv  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
assert not (tgt.WITH_TORCH_SCATTER or tgt.WITH_TORCH_SPARSE or tgt.WITH_PYG_LIB)

# (tag, channels, constructor kwargs, bipartite)
CASES = [("plain", 16, {}, False),
         ("bip_mean_bn", (8, 16), {"dim": 5, "aggr": "mean", "batch_norm": True}, True),
         ("narrow", 6, {"dim": 3, "bias": False}, False)]


def main():
    g = torch.Generator().manual_seed(8080)
    N_src, N_dst, E = 13, 9, 70
    arrs = {}
    for k, (tag, ch, kw, bip) in enumerate(CASES):
        n_dst = N_dst if bip else N_src
        f_src, f_dst = (ch, ch) if isinstance(ch, int) else ch
        dim = kw.get("dim", 0)
        ei = torch.stack([torch.randint(0, N_src, (E, ), generator=g), torch.randint(0, n_dst - 1, (E, ), generator=g)])
        ei[:, 1] = ei[:, 0]                                    # a duplicated edge; destination n_dst-1 has no in-edge
        x = torch.randn(N_src, f_src, generator=g)
        x_dst = torch.randn(n_dst, f_dst, generator=g) if bip else None
        ea = torch.randn(E, dim, generator=g) if dim else None
        torch.manual_seed(31 + k)
        conv = CGConv(ch, **kw)
        if conv.bn is not None:
            with torch.no_grad():
                conv.bn.weight.normal_()                       # the reference initialises them to 1 and 0
                conv.bn.bias.normal_()
        for name, p in conv.state_dict().items():
            arrs[f"{tag}_p_{name}"] = p.clone()
        conv.train()
        xr = x.clone().requires_grad_()
        xdr = x_dst.clone().requires_grad_() if bip else None
        ear = ea.clone().requires_grad_() if dim else None
        out = conv((xr, xdr) if bip else xr, ei, ear)
        gout = torch.randn(out.shape, generator=g)
        out.backward(gout)
        arrs.update({f"{tag}_ei": ei, f"{tag}_x": x, f"{tag}_out": out, f"{tag}_gout": gout, f"{tag}_gx": xr.grad})
        if bip:
            arrs.update({f"{tag}_x_dst": x_dst, f"{tag}_gx_dst": xdr.grad})
        if dim:
            arrs.update({f"{tag}_ea": ea, f"{tag}_gea": ear.grad})
        for name, p in conv.named_parameters():
            arrs[f"{tag}_g_{name}"] = p.grad
        arrs[f"{tag}_shapes"] = np.asarray(json.dumps({n: list(p.shape) for n, p in conv.state_dict().items()}))
        arrs[f"{tag}_repr"] = np.asarray(repr(conv))
    np_arrs = {k: (v.detach().numpy() if isinstance(v, torch.Tensor) else v) for k, v in arrs.items()}
    np.savez_compressed(os.path.join(OUT, "cg.npz"), **np_arrs)
    print("wrote cg", len(np_arrs), "arrays")


if __name__ == "__main__":
    main()
