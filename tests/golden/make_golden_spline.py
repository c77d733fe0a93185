"""Golden vectors for SplineConv (spline_conv.py:21-172): the UNMODIFIED reference's layer on the CPU, forward and
backward, with the fp64 restatement of pyg-lib's `spline_basis` / `spline_weighting` from tests/spline_oracle.py bound
into its module (pyg-lib is not installed, so the reference leaves both names None).  Six cases: FAUST-like (dim 3,
kernel 5, aggr='add'), MNIST-like (dim 2, kernel 5, aggr='mean', F_in = 1), degree 2 with mixed open / closed
dimensions and kernel sizes [3, 4], bipartite in_channels (8, 16) with `size=`, root_weight=False with bias=False,
and degree 3 at dim 1 with destinations 0..2 without in-edges -- plus the `state_dict` shapes and the repr of each.
Same provenance rules as make_golden.py (needs the reference in oracle/_ref; writes tests/golden/spline.npz).

    python tests/golden/make_golden_spline.py
"""
import json
import os
import sys

import numpy as np
import torch

HERE = os.path.dirname(os.path.abspath(__file__))
sys.path.insert(0, os.path.join(HERE, "..", "..", "oracle", "_ref"))             # oracle/install_ref.sh
sys.path.insert(0, os.path.join(HERE, ".."))
import spline_oracle as SO  # noqa: E402
import torch_geometric.nn.conv.spline_conv as tg_spline  # noqa: E402
import torch_geometric.typing as tgt  # noqa: E402

OUT = HERE
assert not (tgt.WITH_TORCH_SCATTER or tgt.WITH_TORCH_SPARSE or tgt.WITH_PYG_LIB)
assert tg_spline.spline_basis is None and tg_spline.spline_weighting is None

# (tag, in_channels, out_channels, dim, constructor kwargs, isolated destinations, bipartite size=)
CASES = [("faust_add", 8, 8, 3, {"kernel_size": 5, "aggr": "add"}, False),
         ("mnist_mean", 1, 16, 2, {"kernel_size": 5, "aggr": "mean"}, False),
         ("deg2_mixed", 6, 4, 2, {"kernel_size": [3, 4], "is_open_spline": [True, False], "degree": 2}, False),
         ("bipartite", (8, 16), 8, 2, {"kernel_size": 3, "aggr": "add"}, False),
         ("no_root_no_bias", 4, 8, 2, {"kernel_size": 4, "root_weight": False, "bias": False}, False),
         ("deg3_isolated", 4, 6, 1, {"kernel_size": 6, "degree": 3, "aggr": "mean"}, True)]


def main():
    tg_spline.spline_basis, tg_spline.spline_weighting = SO.torch_spline_basis, SO.torch_spline_weighting
    g = torch.Generator().manual_seed(5151)
    N_src, N_dst, E = 12, 9, 60
    arrs = {}
    for n, (tag, ch, f_out, dim, kw, isolated) in enumerate(CASES):
        bip = not isinstance(ch, int)
        f_src, f_dst = (ch, ch) if not bip else ch
        n_dst = N_dst if bip else N_src
        lo = 3 if isolated else 0
        ei = torch.stack([torch.randint(0, N_src, (E, ), generator=g), torch.randint(lo, n_dst, (E, ), generator=g)])
        x = torch.randn(N_src, f_src, generator=g)
        x_dst = torch.randn(n_dst, f_dst, generator=g) if bip else None
        ea = torch.rand(E, dim, generator=g)
        torch.manual_seed(90 + n)
        conv = tg_spline.SplineConv(ch, f_out, dim, **kw)
        if conv.bias is not None:
            with torch.no_grad():
                conv.bias.normal_()                             # the reference initialises it to 0
        for name, p in conv.state_dict().items():
            arrs[f"{tag}_p_{name}"] = p.clone()
        xr = x.clone().requires_grad_()
        xdr = x_dst.clone().requires_grad_() if bip else None
        ear = ea.clone().requires_grad_()
        # the bipartite case passes size= as well (the destination count of x_dst)
        out = conv((xr, xdr), ei, ear, size=(N_src, n_dst)) if bip else conv(xr, ei, ear)
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
    np.savez_compressed(os.path.join(OUT, "spline.npz"), **np_arrs)
    print("wrote spline", len(np_arrs), "arrays")


if __name__ == "__main__":
    main()
