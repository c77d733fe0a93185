"""Golden vectors for ResGatedGraphConv (res_gated_graph_conv.py:13-148): the UNMODIFIED reference's layer on the CPU,
forward and backward, for three cases -- `ResGatedGraphConv(16, 32)`; a bipartite `((16, 24), 32)` with
`aggr='mean'` and `root_weight=False`; `out_channels=6` with `bias=False` (rows of 24 bytes: the kernels' scalar path
in fp32) -- plus the `state_dict` shapes of each.  Same provenance rules as make_golden.py (needs the reference in
oracle/_ref; writes tests/golden/res_gated.npz).

    python tests/golden/make_golden_res_gated.py
"""
import json
import os
import sys

import numpy as np
import torch

sys.path.insert(0, os.path.join(os.path.dirname(os.path.abspath(__file__)), "..", "..", "oracle", "_ref"))  # oracle/install_ref.sh
import torch_geometric.typing as tgt  # noqa: E402
from torch_geometric.nn import ResGatedGraphConv  # noqa: E402

OUT = os.path.dirname(os.path.abspath(__file__))
assert not (tgt.WITH_TORCH_SCATTER or tgt.WITH_TORCH_SPARSE or tgt.WITH_PYG_LIB)

# (tag, in_channels, out_channels, constructor kwargs, bipartite)
CASES = [("plain", 16, 32, {}, False),
         ("mean_bip", (16, 24), 32, {"aggr": "mean", "root_weight": False}, True),
         ("narrow", 16, 6, {"bias": False}, False)]


def main():
    g = torch.Generator().manual_seed(5151)
    N_src, N_dst, E = 13, 9, 70
    arrs = {}
    for k, (tag, ic, oc, kw, bip) in enumerate(CASES):
        n_dst = N_dst if bip else N_src
        f_src, f_dst = (ic, ic) if isinstance(ic, int) else ic
        ei = torch.stack([torch.randint(0, N_src, (E, ), generator=g), torch.randint(0, n_dst - 1, (E, ), generator=g)])
        ei[:, 1] = ei[:, 0]                                    # a duplicated edge; destination n_dst-1 has no in-edge
        x = torch.randn(N_src, f_src, generator=g)
        x_dst = torch.randn(n_dst, f_dst, generator=g) if bip else None
        torch.manual_seed(21 + k)
        conv = ResGatedGraphConv(ic, oc, **kw)
        if conv.bias is not None:
            with torch.no_grad():
                conv.bias.normal_()                            # the reference zero-initialises it
        xr = x.clone().requires_grad_()
        xdr = x_dst.clone().requires_grad_() if bip else None
        out = conv((xr, xdr) if bip else xr, ei)
        gout = torch.randn(out.shape, generator=g)
        out.backward(gout)
        arrs.update({f"{tag}_ei": ei, f"{tag}_x": x, f"{tag}_out": out, f"{tag}_gout": gout, f"{tag}_gx": xr.grad})
        if bip:
            arrs.update({f"{tag}_x_dst": x_dst, f"{tag}_gx_dst": xdr.grad})
        for name, p in conv.state_dict().items():
            arrs[f"{tag}_p_{name}"] = p
        for name, p in conv.named_parameters():
            arrs[f"{tag}_g_{name}"] = p.grad
        arrs[f"{tag}_shapes"] = np.asarray(json.dumps({n: list(p.shape) for n, p in conv.state_dict().items()}))
        arrs[f"{tag}_repr"] = np.asarray(repr(conv))
    np_arrs = {k: (v.detach().numpy() if isinstance(v, torch.Tensor) else v) for k, v in arrs.items()}
    np.savez_compressed(os.path.join(OUT, "res_gated.npz"), **np_arrs)
    print("wrote res_gated", len(np_arrs), "arrays")


if __name__ == "__main__":
    main()
